"""The float64 restatement of PSRL (oracle/oracle_psrl.py) against goldens from the unmodified reference, and, where the
reference is importable, against the reference itself on fresh random cases."""
import numpy as np
import pytest

from oracle import oracle_psrl as op
from oracle.ref_shim import reference_available
from tianshou_b200.algorithm.minibatch_order import pack_numpy_state, unpack_numpy_state

VARIANTS = ["chain", "chain_f32_done", "lake", "wide"]
POSTERIOR = ("trans_count", "rew_mean", "rew_std", "rew_square_sum", "rew_count")


def cfg(g):
    return int(g["cfg_n_s"]), int(g["cfg_n_a"]), float(g["cfg_gamma"]), float(g["cfg_eps"]), bool(g["cfg_add_done_loop"])


def replay(g, order=None, square_f64=False):
    """Every round of a golden through the restatement: yields (round, posterior, stats, permutation)."""
    n_s, n_a, _, eps, loop = cfg(g)
    state = op.initial_state(g["trans_count_prior"], g["rew_mean_prior"], g["rew_std_prior"], eps)
    for r in range(int(g["cfg_rounds"])):
        p = f"r{r}_"
        np.random.set_state(unpack_numpy_state("MT19937", g[p + "np_state"]))
        perm = np.random.permutation(len(g[p + "obs"]))
        rew = g[p + "rew"].astype(np.float64) if square_f64 else g[p + "rew"]
        batch = op.update_rows(n_s, n_a, g[p + "obs"], g[p + "act"], g[p + "obs_next"], rew, g[p + "done"],
                               perm if order is None else order(perm), loop)
        op.observe(state, g["rew_std_prior"], *batch)
        yield r, state, (state["rew_mean"].mean(), state["rew_std"].mean()), perm


@pytest.mark.parametrize("variant", VARIANTS)
def test_restatement_reproduces_golden(golden, variant):
    g = golden(f"psrl_ref_{variant}.npz")
    n_s, n_a, gamma, eps, _ = cfg(g)
    for r, state, stats, _ in replay(g):
        p = f"r{r}_"
        assert np.array_equal(pack_numpy_state(np.random.get_state()), g[p + "np_state_after"])
        for k in POSTERIOR:
            assert np.array_equal(state[k], g[p + k]), (variant, r, k)
        assert stats == (g[p + "stat_mean"], g[p + "stat_std"])
        pol, val, sweeps, qn = op.value_iteration(g[p + "P"], g[p + "R"], gamma, eps, g[p + "value_before"], g[p + "noise"])
        assert np.array_equal(pol, g[p + "policy"]) and np.array_equal(val, g[p + "value"]), (variant, r)
        assert sweeps == int(g[p + "sweeps"]) and op.tie_gap(qn) == g[p + "gap"]
        if r:
            assert np.array_equal(g[p + "value_before"], g[f"r{r - 1}_value"])


def test_goldens_tell_misreadings_apart(golden):
    """A float64 square of float32 rewards and a sum in buffer order both move the golden posterior."""
    g = golden("psrl_ref_chain_f32_done.npz")
    assert g["r0_rew"].dtype == np.float32
    moved = [not np.array_equal(s["rew_square_sum"], g[f"r{r}_rew_square_sum"]) for r, s, _, _ in replay(g, square_f64=True)]
    assert any(moved)
    for variant in ("wide",):     # float64 rewards with noise: float32 or small-integer rewards sum exactly in any order
        g = golden(f"psrl_ref_{variant}.npz")
        moved = [any(not np.array_equal(s[k], g[f"r{r}_{k}"]) for k in ("rew_mean", "rew_square_sum"))
                 for r, s, _, _ in replay(g, order=np.sort)]
        assert any(moved), variant


def test_unvisited_pairs_leave_the_prior(golden):
    g = golden("psrl_ref_wide.npz")
    seen = np.zeros((int(g["cfg_n_s"]), int(g["cfg_n_a"])), bool)
    seen[g["r0_obs"], g["r0_act"]] = True
    assert (~seen).sum() > 20
    assert not np.any(g["r0_rew_std"][~seen] == g["rew_std_prior"][~seen])


@pytest.mark.skipif(not reference_available(), reason="the reference is not available")
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_restatement_matches_reference(seed):
    from oracle.ref_shim import import_reference
    import_reference()
    import gymnasium as gym
    from tianshou.algorithm import PSRL
    from tianshou.algorithm.modelbased.psrl import PSRLPolicy
    from tianshou.data import Batch

    rng = np.random.default_rng(seed)
    n_s, n_a, n = int(rng.integers(2, 12)), int(rng.integers(1, 5)), int(rng.integers(1, 300))
    f32, loop = bool(seed % 2), seed != 1
    priors = (rng.random((n_s, n_a, n_s)) + 0.1, rng.standard_normal((n_s, n_a)), rng.random((n_s, n_a)) + 0.5)
    rows = dict(obs=rng.integers(0, n_s, n), act=rng.integers(0, n_a, n), obs_next=rng.integers(0, n_s, n),
                rew=rng.standard_normal(n).astype(np.float32 if f32 else np.float64), done=rng.random(n) < 0.2)
    state = op.initial_state(*priors, 0.01)
    policy = PSRLPolicy(trans_count_prior=priors[0].copy(), rew_mean_prior=priors[1].copy(), rew_std_prior=priors[2].copy(),
                        action_space=gym.spaces.Discrete(n_a), discount_factor=0.9, epsilon=0.01)
    algo = PSRL(policy=policy, add_done_loop=loop)
    np.random.seed(seed)
    algo._update_with_batch(Batch(**rows), None, 1)
    np.random.seed(seed)
    perm = np.random.permutation(n)
    op.observe(state, priors[2], *op.update_rows(n_s, n_a, rows["obs"], rows["act"], rows["obs_next"], rows["rew"], rows["done"],
                                                 perm, loop))
    for k in POSTERIOR:
        assert np.array_equal(state[k], getattr(policy.model, k), equal_nan=True), k
    P, R = rng.dirichlet(np.ones(n_s), (n_s, n_a)), rng.standard_normal((n_s, n_a))
    v0 = rng.standard_normal(n_s)
    np.random.seed(seed)
    pol, val = policy.model.value_iteration(P, R, 0.9, 0.01, v0)
    np.random.seed(seed)
    noise = np.random.randn(n_s, n_a)          # the reference draws it after the sweeps, which draw nothing
    opol, oval, _, _ = op.value_iteration(P, R, 0.9, 0.01, v0, noise)
    assert np.array_equal(pol, opol) and np.array_equal(val, oval)
