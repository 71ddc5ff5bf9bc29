"""PSRL on the device: the posterior kernels and value iteration against the float64 restatement (oracle/oracle_psrl.py),
``update()`` and the solve against the reference's goldens, the refusals, the iteration bound, learning NChain end to end, and
the register report."""
import numpy as np
import pytest
import torch

from offpolicy_testutil import DEV, Discrete, assert_spill_free, ptxas_report
from oracle import oracle_psrl as op
from tianshou_b200.algorithm.minibatch_order import pack_numpy_state, unpack_numpy_state

pytestmark = pytest.mark.gpu

POSTERIOR = ("trans_count", "rew_mean", "rew_std", "rew_square_sum", "rew_count")
VARIANTS = ["chain", "chain_f32_done", "lake", "wide"]


def make(n_s, n_a, seed=0, gamma=0.9, eps=0.01, loop=False, zero_mean=False, **kw):
    """Random priors.  With a reward-count prior of eps, a pair seen once with a reward between 0 and twice its prior mean gets
    a NaN rew_std, as in the reference; ``zero_mean`` rules that out for tests that solve the posterior."""
    from tianshou_b200.algorithm import PSRL
    from tianshou_b200.algorithm.modelbased.psrl import PSRLPolicy
    rng = np.random.default_rng(seed)
    mean = np.zeros((n_s, n_a)) if zero_mean else rng.standard_normal((n_s, n_a))
    priors = dict(trans_count_prior=rng.random((n_s, n_a, n_s)) + 0.1, rew_mean_prior=mean, rew_std_prior=rng.random((n_s, n_a)) + 0.5)
    pol = PSRLPolicy(**priors, action_space=Discrete(n_a), discount_factor=gamma, epsilon=eps, device=DEV, **kw)
    return PSRL(policy=pol, add_done_loop=loop), priors


def rows_batch(rng, n, n_s, n_a, f32):
    """Rows skewed onto (0, 0) (thousands of rows at large n) that never visit the last state."""
    from tianshou_b200.data import Batch
    hot = rng.random(n) < 0.5
    obs = np.where(hot, 0, rng.integers(0, n_s - 1, n))
    act = np.where(hot, 0, rng.integers(0, n_a, n))
    rew = (rng.standard_normal(n) * 3).astype(np.float32 if f32 else np.float64)
    return Batch(obs=obs, act=act, obs_next=rng.integers(0, n_s - 1, n), rew=rew, done=rng.random(n) < 0.3)


def posterior(model):
    return {k: getattr(model, k) for k in POSTERIOR}


@pytest.mark.parametrize("loop", [False, True])
@pytest.mark.parametrize("f32", [False, True])
@pytest.mark.parametrize("N", [1, 31, 32, 33, 1000, 65537])
def test_posterior_kernels_bitwise(N, f32, loop):
    """ts_psrl_update (sized by ts_psrl_update_workspace_bytes) against the per-row restatement, bit for bit."""
    n_s, n_a = 7, 3
    rng = np.random.default_rng(N)
    batch = rows_batch(rng, N, n_s, n_a, f32)
    got = []
    for _ in range(2):
        algo, priors = make(n_s, n_a, loop=loop)
        np.random.seed(5)
        stats = algo._update_with_batch(batch, None, 1)
        got.append(posterior(algo.policy.model))
    np.random.seed(5)
    perm = np.random.permutation(N)
    state = op.initial_state(priors["trans_count_prior"], priors["rew_mean_prior"], priors["rew_std_prior"], 0.01)
    op.observe(state, priors["rew_std_prior"], *op.update_rows(n_s, n_a, batch.obs, batch.act, batch.obs_next, batch.rew,
                                                               batch.done, perm, loop))
    for k in POSTERIOR:
        assert np.array_equal(got[0][k], state[k], equal_nan=True), k
        assert np.array_equal(got[0][k], got[1][k], equal_nan=True), k
    for got_stat, ref in ((stats.psrl_rew_mean, state["rew_mean"].mean()), (stats.psrl_rew_std, state["rew_std"].mean())):
        assert (np.isnan(got_stat) and np.isnan(ref)) or abs(got_stat - ref) <= 1e-12 * max(1.0, abs(ref))


@pytest.mark.parametrize("bad", ["obs_high", "obs_neg", "act_high", "act_neg", "next_high", "float"])
def test_refused_indices_leave_posterior_unchanged(bad):
    n_s, n_a = 6, 2
    algo, _ = make(n_s, n_a, loop=True)
    rng = np.random.default_rng(1)
    algo._update_with_batch(rows_batch(rng, 100, n_s, n_a, False), None, 1)
    before = posterior(algo.policy.model)
    b = rows_batch(rng, 100, n_s, n_a, False)
    if bad == "float":
        b.obs = b.obs.astype(np.float32)
    else:
        key, val = {"obs_high": ("obs", n_s), "obs_neg": ("obs", -1), "act_high": ("act", n_a), "act_neg": ("act", -1),
                    "next_high": ("obs_next", n_s)}[bad]
        b[key][57] = val
    with pytest.raises(IndexError):
        algo._update_with_batch(b, None, 1)
    after = posterior(algo.policy.model)
    for k in POSTERIOR:
        assert np.array_equal(before[k], after[k], equal_nan=True), k


def test_dense_observe_matches_restatement():
    """ts_psrl_observe (PSRLModel.observe with the batch's dense arrays) == the restatement, bit for bit."""
    n_s, n_a = 9, 3
    algo, priors = make(n_s, n_a, zero_mean=True)
    rng = np.random.default_rng(7)
    dense = (rng.integers(0, 4, (n_s, n_a, n_s)).astype(float), rng.standard_normal((n_s, n_a)), rng.random((n_s, n_a)) * 5,
             rng.integers(0, 6, (n_s, n_a)).astype(float))
    algo.policy.model.observe(*dense)
    state = op.initial_state(priors["trans_count_prior"], priors["rew_mean_prior"], priors["rew_std_prior"], 0.01)
    op.observe(state, priors["rew_std_prior"], *dense)
    for k in POSTERIOR:
        assert np.array_equal(getattr(algo.policy.model, k), state[k], equal_nan=True), k
    assert not algo.policy.model.updated


def _vi_case(rng, n_s, n_a):
    P = rng.dirichlet(np.full(n_s, 0.3), (n_s, n_a))
    return P, rng.standard_normal((n_s, n_a)), rng.standard_normal((n_s, n_a))


@pytest.mark.parametrize("n_a", [1, 2, 4, 7])
@pytest.mark.parametrize("n_s", [1, 2, 5, 31, 64, 65, 200, 1024])
def test_value_iteration_vs_oracle(n_s, n_a):
    """ts_psrl_value_iteration (scratch from ts_psrl_value_iteration_scratch_bytes) against numpy float64."""
    from tianshou_b200 import ops
    from tianshou_b200.algorithm.modelbased.psrl import _solve
    rng = np.random.default_rng(n_s * 10 + n_a)
    P, R, noise = _vi_case(rng, n_s, n_a)
    t = [torch.from_numpy(x).to(DEV) for x in (P, R, noise)]
    for gamma in (0.0, 0.5, 0.99):
        for v0 in (np.zeros(n_s), rng.standard_normal(n_s) * 5):
            pol, val, sweeps, _ = op.value_iteration(P, R, gamma, 0.01, v0, noise)
            runs = []
            for _ in range(2):
                V = torch.from_numpy(v0.copy()).to(DEV)
                _, _, gpol, gsweeps = _solve(*t, gamma, 0.01, 100_000, V)
                runs.append((gpol, V.cpu().numpy(), gsweeps))
            gpol, gval, gsweeps = runs[0]
            assert gsweeps == sweeps, (gamma, gsweeps, sweeps)
            assert np.array_equal(gpol, pol), gamma
            np.testing.assert_allclose(gval, val, rtol=1e-12, atol=1e-12)
            assert np.array_equal(runs[1][0], gpol) and np.array_equal(runs[1][1], gval) and runs[1][2] == gsweeps
    assert ops.psrl_max_states() >= 1024


def test_value_iteration_exact_ties_take_the_first_action():
    from tianshou_b200.algorithm.modelbased.psrl import PSRLModel
    rng = np.random.default_rng(3)
    n_s, n_a = 65, 4
    P = np.repeat(rng.dirichlet(np.ones(n_s), n_s)[:, None, :], n_a, axis=1)
    R = np.repeat(rng.standard_normal((n_s, 1)), n_a, axis=1)
    pol, val = PSRLModel.value_iteration(P, R, 0.9, 0.01, np.zeros(n_s), noise=np.zeros((n_s, n_a)), device=DEV)
    assert pol.dtype == np.int64 and np.all(pol == 0)
    tpol, tval = PSRLModel.value_iteration(torch.from_numpy(P).to(DEV), torch.from_numpy(R).to(DEV), 0.9, 0.01,
                                           torch.zeros(n_s, dtype=torch.float64, device=DEV),
                                           noise=torch.zeros(n_s, n_a, dtype=torch.float64, device=DEV))
    assert isinstance(tval, torch.Tensor) and tval.is_cuda and np.array_equal(tval.cpu().numpy(), val)


@pytest.mark.parametrize("case", ["slow", "nan"])
def test_non_convergence_raises_and_keeps_the_policy(case):
    from tianshou_b200.data import Batch
    algo, _ = make(12, 3, gamma=0.999, eps=1e-6, zero_mean=True, max_iterations=100_000)
    pol = algo.policy
    model = pol.model
    torch.manual_seed(0)
    first = pol(Batch(obs=np.arange(12), info=Batch())).act.copy()
    value = model.value
    model.updated = False
    model.max_iterations = 5
    if case == "nan":
        model.sample_reward = lambda: torch.full((12, 3), float("nan"), dtype=torch.float64, device=DEV)
    with pytest.raises(RuntimeError, match="did not converge in 5 sweeps"):
        pol(Batch(obs=np.arange(12), info=Batch()))
    assert np.array_equal(model.policy, first) and np.array_equal(model.value, value) and not model.updated


def _buffer_from_golden(g, r, mirror):
    from tianshou_b200.data import Batch, VectorReplayBuffer
    E = int(g["cfg_E"])
    n = len(g[f"r{r}_obs"])
    T = n // E
    buf = VectorReplayBuffer(n, E, device=DEV, device_mirror=mirror)
    for t in range(T):
        idx = np.arange(E) * T + t
        d = {k: g[f"r{r}_{k}"][idx] for k in ("obs", "act", "rew", "obs_next")}
        buf.add(Batch(**d, terminated=g[f"r{r}_done"][idx], truncated=np.zeros(E, bool), info=Batch()), buffer_ids=np.arange(E))
    return buf


@pytest.mark.parametrize("mirror", [False, True])
@pytest.mark.parametrize("variant", VARIANTS)
def test_update_and_solve_match_reference(golden, variant, mirror):
    from tianshou_b200.algorithm import PSRL
    from tianshou_b200.algorithm.modelbased.psrl import PSRLPolicy
    from tianshou_b200.data import Batch
    from tianshou_b200.utils import policy_within_training_step
    g = golden(f"psrl_ref_{variant}.npz")
    n_s, n_a = int(g["cfg_n_s"]), int(g["cfg_n_a"])
    f32 = g["r0_rew"].dtype == np.float32
    if f32 and mirror:
        pytest.skip("float32 rewards reach the update in a batch of their own, not through a buffer")
    pol = PSRLPolicy(trans_count_prior=g["trans_count_prior"], rew_mean_prior=g["rew_mean_prior"],
                     rew_std_prior=g["rew_std_prior"], action_space=Discrete(n_a), discount_factor=float(g["cfg_gamma"]),
                     epsilon=float(g["cfg_eps"]), device=DEV)
    algo = PSRL(policy=pol, add_done_loop=bool(g["cfg_add_done_loop"]))
    model = pol.model
    for r in range(int(g["cfg_rounds"])):
        p = f"r{r}_"
        np.random.set_state(unpack_numpy_state("MT19937", g[p + "np_state"]))
        with policy_within_training_step(pol):
            if f32:
                stats = algo._update_with_batch(Batch(**{k: g[p + k] for k in ("obs", "act", "rew", "done", "obs_next")}), 0, 1)
            else:
                buf = _buffer_from_golden(g, r, mirror)
                if mirror:
                    assert buf.device_columns() is not None
                stats = algo.update(buffer=buf, batch_size=0, repeat=1)
        assert np.array_equal(pack_numpy_state(np.random.get_state()), g[p + "np_state_after"])
        for k in POSTERIOR:
            assert np.array_equal(getattr(model, k), g[p + k]), (r, k)
        assert abs(stats.psrl_rew_mean - g[p + "stat_mean"]) <= 1e-12 * max(1.0, abs(g[p + "stat_mean"]))
        assert abs(stats.psrl_rew_std - g[p + "stat_std"]) <= 1e-12 * max(1.0, abs(g[p + "stat_std"]))
        model.sample_trans_prob = lambda p=p: torch.from_numpy(g[p + "P"]).to(DEV)
        model.sample_reward = lambda p=p: torch.from_numpy(g[p + "R"]).to(DEV)
        model._tie_noise = lambda shape, p=p: torch.from_numpy(g[p + "noise"]).to(DEV)
        act = pol(Batch(obs=np.arange(n_s), info=Batch())).act
        assert np.array_equal(act, g[p + "policy"]), r
        np.testing.assert_allclose(model.value, g[p + "value"], rtol=1e-12, atol=1e-12)
        assert model.last_sweeps == int(g[p + "sweeps"]), (r, model.last_sweeps)
    assert sorted(algo.state_dict().keys()) == list(g["state_dict_keys"])


def test_learns_nchain():
    """Collect with the current policy -> add to the buffer -> update, seeded: PSRL reaches NChain's optimal policy."""
    from tianshou_b200.data import Batch, VectorReplayBuffer
    from tianshou_b200.utils import policy_within_training_step
    n = 5
    P_true, R_true = op.nchain_model(n)
    opt, _, _, _ = op.value_iteration(P_true, R_true, 0.99, 1e-6, np.zeros(n), np.zeros((n, 2)))
    np.random.seed(0)
    torch.manual_seed(0)
    algo, _ = make(n, 2, gamma=0.99, eps=0.01)
    from tianshou_b200.algorithm.modelbased.psrl import PSRLModel
    pol = algo.policy
    pol.model = PSRLModel(np.ones((n, 2, n)), np.zeros((n, 2)), np.ones((n, 2)), 0.99, 0.01, device=DEV)
    rng = np.random.default_rng(0)
    s = np.zeros(4, dtype=np.int64)
    for _ in range(30):
        buf = VectorReplayBuffer(400, 4, device=DEV)
        for _ in range(100):
            a = pol(Batch(obs=s, info=Batch())).act
            nxt, r = zip(*(op.nchain_step(rng, int(si), int(ai)) for si, ai in zip(s, a)))
            nxt = np.array(nxt, dtype=np.int64)
            buf.add(Batch(obs=s, act=a, rew=np.array(r), terminated=np.zeros(4, bool), truncated=np.zeros(4, bool), obs_next=nxt,
                          info=Batch()), buffer_ids=np.arange(4))
            s = nxt
        with policy_within_training_step(pol):
            algo.update(buffer=buf, batch_size=0, repeat=1)
    pol(Batch(obs=s, info=Batch()))
    assert np.array_equal(pol.model.policy, opt), (pol.model.policy, opt)


def test_one_solve_per_update_and_seeded_solves():
    from tianshou_b200 import _cabi
    from tianshou_b200.data import Batch
    algo_a, _ = make(40, 3, seed=2, zero_mean=True)
    algo_b, _ = make(40, 3, seed=2, zero_mean=True)
    batch = rows_batch(np.random.default_rng(4), 500, 40, 3, False)
    for algo in (algo_a, algo_b):
        np.random.seed(1)
        algo._update_with_batch(batch, None, 1)
    torch.manual_seed(9)
    _cabi.reset_launch_count()
    acts = [algo_a.policy(Batch(obs=np.arange(40), info=Batch())).act for _ in range(5)]
    assert _cabi.launch_count() == 1
    assert acts[0].dtype == np.int64 and all(np.array_equal(a, acts[0]) for a in acts)
    torch.manual_seed(9)
    act_b = algo_b.policy(Batch(obs=np.arange(40), info=Batch())).act
    assert np.array_equal(acts[0], act_b) and np.array_equal(algo_a.policy.model.value, algo_b.policy.model.value)


def test_refuses_states_past_shared_memory():
    """ts_psrl_max_states bounds the model size value iteration accepts."""
    from tianshou_b200 import ops
    from tianshou_b200.algorithm import UnsupportedModelError
    from tianshou_b200.algorithm.modelbased.psrl import PSRLModel
    n = ops.psrl_max_states() + 1
    with pytest.raises(UnsupportedModelError):
        PSRLModel.value_iteration(np.zeros((n, 1, 1)), np.zeros((n, 1)), 0.9, 0.01, np.zeros(n), device=DEV)


def test_kernels_have_no_stack_frame_or_spills(tmp_path):
    report = ptxas_report("psrl.cu", tmp_path)
    ours = {k: v for k, v in report.items() if "psrl" in k and "cub" not in k.lower()}
    assert len(ours) == 8
    assert_spill_free(ours)
