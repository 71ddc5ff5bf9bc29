"""PSRL's input checks and its device-mirror path: inputs of the wrong shape are refused on the host with ValueError before any
launch; a mirrored buffer's update reads the mirror (and refuses a bad index through it with the posterior unchanged); a buffer
whose mirror keeps uint8 indices takes the upload path and computes the same posterior."""
import numpy as np
import pytest
import torch

from offpolicy_testutil import DEV, Discrete
from oracle import oracle_psrl as op

pytestmark = pytest.mark.gpu

POSTERIOR = ("trans_count", "rew_mean", "rew_std", "rew_square_sum", "rew_count")


def make(n_s, n_a, loop=False):
    from tianshou_b200.algorithm import PSRL
    from tianshou_b200.algorithm.modelbased.psrl import PSRLPolicy
    pol = PSRLPolicy(trans_count_prior=np.ones((n_s, n_a, n_s)), rew_mean_prior=np.zeros((n_s, n_a)),
                     rew_std_prior=np.ones((n_s, n_a)), action_space=Discrete(n_a), device=DEV)
    return PSRL(policy=pol, add_done_loop=loop)


def posterior(model):
    return {k: getattr(model, k) for k in POSTERIOR}


def assert_unchanged(before, model):
    for k in POSTERIOR:
        assert np.array_equal(before[k], getattr(model, k), equal_nan=True), k


@pytest.mark.parametrize("case", ["P_states", "P_actions", "P_flat", "value_short", "value_long", "noise", "rew_1d"])
@pytest.mark.parametrize("as_tensor", [False, True])
def test_value_iteration_refuses_mismatched_shapes(case, as_tensor):
    from tianshou_b200.algorithm.modelbased.psrl import PSRLModel
    n_s, n_a = 6, 3
    rng = np.random.default_rng(0)
    P, R = rng.dirichlet(np.ones(n_s), (n_s, n_a)), rng.standard_normal((n_s, n_a))
    V, noise = np.zeros(n_s), np.zeros((n_s, n_a))
    if case == "P_states":
        P = P[:-1]
    elif case == "P_actions":
        P = P[:, :-1]
    elif case == "P_flat":
        P = P.reshape(n_s, -1)
    elif case == "value_short":
        V = V[:-2]
    elif case == "value_long":
        V = np.zeros(n_s + 5)
    elif case == "noise":
        noise = noise[:, :-1]
    else:
        R = R.reshape(-1)
    args = (P, R, 0.9, 0.01, V)
    if as_tensor:
        args = tuple(torch.from_numpy(a).to(DEV) if isinstance(a, np.ndarray) else a for a in args)
        noise = torch.from_numpy(noise).to(DEV)
    with pytest.raises(ValueError):
        PSRLModel.value_iteration(*args, noise=noise, device=DEV)


@pytest.mark.parametrize("draw", ["P", "R", "noise"])
def test_solve_refuses_draws_of_the_wrong_shape(draw):
    """A replaced draw (the seams tests use) of the wrong shape is refused before the kernel, and the model keeps its state."""
    from tianshou_b200.data import Batch
    algo = make(5, 2)
    model = algo.policy.model
    bad = torch.zeros(4, 2, dtype=torch.float64, device=DEV)
    if draw == "P":
        model.sample_trans_prob = lambda: torch.full((5, 2, 4), 0.25, dtype=torch.float64, device=DEV)
    elif draw == "R":
        model.sample_reward = lambda: bad
    else:
        model._tie_noise = lambda shape: bad
    with pytest.raises(ValueError):
        algo.policy(Batch(obs=np.arange(5), info=Batch()))
    assert not model.updated and np.array_equal(model.value, np.zeros(5))


@pytest.mark.parametrize("short", ["rew", "done", "act", "obs_next"])
def test_update_refuses_short_columns(short):
    from tianshou_b200.data import Batch
    algo = make(5, 2, loop=True)
    rng = np.random.default_rng(1)
    n = 40
    cols = dict(obs=rng.integers(0, 5, n), act=rng.integers(0, 2, n), obs_next=rng.integers(0, 5, n), rew=rng.standard_normal(n),
                done=rng.random(n) < 0.3)
    cols[short] = cols[short][:-3]
    before = posterior(algo.policy.model)
    np.random.seed(0)
    with pytest.raises(ValueError):
        algo._update_with_batch(Batch(**cols), None, 1)
    assert_unchanged(before, algo.policy.model)


def test_dense_observe_refuses_mismatched_shapes():
    algo = make(4, 2)
    model = algo.policy.model
    before = posterior(model)
    z = np.zeros((4, 2))
    with pytest.raises(ValueError):
        model.observe(np.zeros((4, 2, 3)), z, z, z)
    with pytest.raises(ValueError):
        model.observe(np.zeros((4, 2, 4)), z, np.zeros(8), z)
    assert_unchanged(before, model)


def _fill(buf, rng, n_s, n_a, E, T, obs_dtype=np.int64, bad=None):
    from tianshou_b200.data import Batch
    for t in range(T):
        obs = rng.integers(0, n_s, E).astype(obs_dtype)
        if bad is not None and t == T // 2:
            obs[0] = bad
        buf.add(Batch(obs=obs, act=rng.integers(0, n_a, E), rew=rng.standard_normal(E), terminated=rng.random(E) < 0.1,
                      truncated=np.zeros(E, bool), obs_next=rng.integers(0, n_s, E).astype(obs_dtype), info=Batch()),
                buffer_ids=np.arange(E))


def _update(algo, buf, monkeypatch):
    """One update; returns what ``_Rows.from_mirror`` returned (None: the upload path)."""
    from tianshou_b200.algorithm.modelbased import psrl
    from tianshou_b200.utils import policy_within_training_step
    seen = []
    orig = psrl._Rows.from_mirror

    def spy(*a, **k):
        seen.append(orig(*a, **k))
        return seen[-1]
    monkeypatch.setattr(psrl._Rows, "from_mirror", staticmethod(spy))
    np.random.seed(3)
    try:
        with policy_within_training_step(algo.policy):
            algo.update(buffer=buf, batch_size=0, repeat=1)
    finally:
        monkeypatch.undo()
    assert len(seen) == 1
    return seen[0]


@pytest.mark.parametrize("obs_dtype", [np.int64, np.uint8])
def test_mirror_path_is_taken_and_matches_the_restatement(obs_dtype, monkeypatch):
    from tianshou_b200.data import VectorReplayBuffer
    n_s, n_a, E, T = 9, 3, 4, 50
    buf = VectorReplayBuffer(E * T, E, device=DEV, device_mirror=True)
    _fill(buf, np.random.default_rng(2), n_s, n_a, E, T, obs_dtype)
    assert buf.device_columns() is not None
    algo = make(n_s, n_a, loop=True)
    rows = _update(algo, buf, monkeypatch)
    if obs_dtype == np.int64:
        assert rows is not None and rows.obs.dtype == torch.float32       # the mirror's float32 index columns
    else:
        assert rows is None                                              # uint8 indices: the upload path
    b, _ = buf.sample(0)
    np.random.seed(3)
    perm = np.random.permutation(len(b))
    state = op.initial_state(np.ones((n_s, n_a, n_s)), np.zeros((n_s, n_a)), np.ones((n_s, n_a)), 0.01)
    op.observe(state, np.ones((n_s, n_a)), *op.update_rows(n_s, n_a, b.obs.astype(np.int64), b.act, b.obs_next.astype(np.int64),
                                                           b.rew, b.done, perm, True))
    for k in POSTERIOR:
        assert np.array_equal(getattr(algo.policy.model, k), state[k], equal_nan=True), k


@pytest.mark.parametrize("bad", [9, -1])
def test_mirror_path_refuses_a_bad_index(bad, monkeypatch):
    from tianshou_b200.data import VectorReplayBuffer
    n_s, n_a, E, T = 9, 3, 4, 50
    algo = make(n_s, n_a, loop=True)
    good = VectorReplayBuffer(E * T, E, device=DEV, device_mirror=True)
    _fill(good, np.random.default_rng(4), n_s, n_a, E, T)
    assert _update(algo, good, monkeypatch) is not None
    before = posterior(algo.policy.model)
    buf = VectorReplayBuffer(E * T, E, device=DEV, device_mirror=True)
    _fill(buf, np.random.default_rng(5), n_s, n_a, E, T, bad=bad)
    with pytest.raises(IndexError):
        _update(algo, buf, monkeypatch)
    assert_unchanged(before, algo.policy.model)
