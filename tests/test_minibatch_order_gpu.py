"""``MinibatchOrder`` (algorithm/minibatch_order.py): the rows each source delivers, numpy's global state afterwards, that
``update()`` and a direct ``_sample`` / ``_preprocess_batch`` / ``_update_with_batch`` compute the same update on every
on-policy path, and the clean-up when a pass raises."""
import warnings

import numpy as np
import pytest
import torch

from ts_testutil import Box, build_actor_critic, gaussian_dist, synth_rollout

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
O, A = 17, 6


def _buffer(E=16, T=64, obs=O, seed=0):
    from tianshou_b200.data import Batch, VectorReplayBuffer
    buf = VectorReplayBuffer(E * T, E, device=DEV)
    for s in synth_rollout(np.random.default_rng(seed), E, T, obs, A, p_term=0.01, trunc_len=200):
        buf.add(Batch(**s), buffer_ids=np.arange(E))
    return buf


def _policy(actor):
    from tianshou_b200.algorithm import ProbabilisticActorPolicy
    return ProbabilisticActorPolicy(actor=actor, dist_fn=gaussian_dist, action_scaling=True, action_bound_method="clip",
                                    action_space=Box(A))


def _ppo(obs=O, **kw):
    from tianshou_b200.algorithm import PPO, AdamOptimizerFactory
    actor, critic = build_actor_critic(obs, A, DEV)
    return PPO(policy=_policy(actor), critic=critic, optim=AdamOptimizerFactory(lr=1e-3), max_grad_norm=0.5, **kw)


def _a2c_rmsprop():
    from tianshou_b200.algorithm import A2C
    from tianshou_b200.algorithm.optim import RMSpropOptimizerFactory
    actor, critic = build_actor_critic(O, A, DEV)
    return A2C(policy=_policy(actor), critic=critic, optim=RMSpropOptimizerFactory(lr=7e-4, eps=1e-5, alpha=0.99),
               max_grad_norm=0.5)


def _natural(name):
    from tianshou_b200.algorithm import NPG, TRPO, AdamOptimizerFactory
    actor, critic = build_actor_critic(O, A, DEV)
    return {"npg": NPG, "trpo": TRPO}[name](policy=_policy(actor), critic=critic, optim=AdamOptimizerFactory(lr=1e-3),
                                            trust_region_size=0.01)


def _gail():
    from tianshou_b200.algorithm import GAIL, AdamOptimizerFactory
    from tianshou_b200.data import ReplayBuffer
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.continuous import ContinuousCritic
    actor, critic = build_actor_critic(O, A, DEV)
    disc = ContinuousCritic(preprocess_net=Net(state_shape=(O,), action_shape=(A,), hidden_sizes=(64, 64),
                                               activation=torch.nn.Tanh, concat=True)).to(DEV)
    rng = np.random.default_rng(5)
    n = 256
    expert = ReplayBuffer.from_data(rng.standard_normal((n, O)).astype(np.float32), rng.standard_normal((n, A)).astype(np.float32),
                                    np.zeros(n), np.zeros(n, bool), np.zeros(n, bool), np.zeros(n, bool),
                                    rng.standard_normal((n, O)).astype(np.float32))
    return GAIL(policy=_policy(actor), critic=critic, optim=AdamOptimizerFactory(lr=1e-3), expert_buffer=expert, disc_net=disc,
                disc_optim=AdamOptimizerFactory(lr=5e-4))


PATHS = {      # name -> (constructor, obs width, layer-wise forced)
    "ppo_tc": (lambda: _ppo(), O, False),
    "ppo_tc_device_order": (lambda: _ppo(minibatch_shuffle="device", shuffle_seed=7), O, False),
    "ppo_simt": (lambda: _ppo(40), 40, False),
    "ppo_layered": (lambda: _ppo(), O, True),
    "ppo_layered_device_order": (lambda: _ppo(minibatch_shuffle="device", shuffle_seed=7), O, True),
    "a2c_rmsprop": (_a2c_rmsprop, O, False),
    "npg": (lambda: _natural("npg"), O, False),
    "trpo": (lambda: _natural("trpo"), O, False),
    "gail": (_gail, O, False),
}


def _groups(algo):
    groups = [algo._flat]
    if algo._layered is not None and algo._layered.group is not algo._flat:
        groups.append(algo._layered.group)
    if hasattr(algo, "_g_disc"):
        groups.append(algo._g_disc)
    return groups


def _outcome(algo):
    out = {}
    for i, g in enumerate(_groups(algo)):
        for k in ("flat", "exp_avg", "exp_avg_sq", "step_dev"):
            t = getattr(g, k, None)
            if t is not None:
                out[f"{i}.{k}"] = t.detach().clone()
        out[f"{i}._step"] = getattr(g, "_step", None)
    for k in ("last_loss_table", "last_stats_table", "last_disc_table"):
        if getattr(algo, k, None) is not None:
            out[k] = torch.from_numpy(np.asarray(getattr(algo, k)).copy())
    return out


def _two_updates(path, via_update, monkeypatch):
    from tianshou_b200.utils import policy_within_training_step
    make, obs, layered = PATHS[path]
    if layered:
        monkeypatch.setenv("TS_B200_FORCE_LAYERED", "1")
    algo = make()
    monkeypatch.delenv("TS_B200_FORCE_LAYERED", raising=False)
    assert (algo._layered is not None) == (layered or path in ("npg", "trpo"))
    buf = _buffer(obs=obs)
    batch_size, repeat = (512, 2) if path in ("npg", "trpo") else (256, 3)
    np.random.seed(1234)
    with policy_within_training_step(algo.policy):
        for _ in range(2):
            if via_update:
                algo.update(buffer=buf, batch_size=batch_size, repeat=repeat)
            else:
                batch, idx = algo._sample(buf, 0)
                algo._update_with_batch(algo._preprocess_batch(batch, buf, idx), batch_size, repeat)
    torch.cuda.synchronize()
    return _outcome(algo), np.random.get_state()


def _permutations(state, n, count):
    np.random.set_state(state)
    return [np.random.permutation(n) for _ in range(count)]


@pytest.mark.parametrize("source", ["numpy", "device"])
def test_rows_and_numpy_state_per_source(source, monkeypatch):
    """The rows on the device after ``ready(r)`` are bit for bit numpy's ``repeat`` draws (numpy source; numpy's state then
    equals the reference's) or ``make_permutation(seed, epoch, repeat, N)`` (device source; numpy untouched), and two
    consecutive device-order updates take epochs 0..R-1 and R..2R-1."""
    from tianshou_b200 import ops
    from tianshou_b200.algorithm import minibatch_order
    from tianshou_b200.utils import policy_within_training_step
    R, N = 3, 16 * 64
    algo = _ppo(minibatch_shuffle=source, shuffle_seed=11)
    np.random.seed(99)
    start = np.random.get_state()
    ref = _permutations(start, N, R)
    ref_state = np.random.get_state()
    np.random.set_state(start)
    for k in range(2):
        with algo._minibatch_order(R, N) as order:
            got = []
            for r in range(R):
                order.ready(r)
                got.append(order.rows[r].cpu())
        if source == "numpy":
            assert all(np.array_equal(g.numpy(), p) for g, p in zip(got, ref, strict=True))
            st = np.random.get_state()
            assert np.array_equal(st[1], ref_state[1]) and st[2:] == ref_state[2:]
            np.random.set_state(start)
        else:
            assert torch.equal(torch.stack(got), ops.make_permutation(11, k * R, R, N, torch.device(DEV)).cpu())
            st = np.random.get_state()
            assert np.array_equal(st[1], start[1]) and st[2:] == start[2:]
    if source == "device":
        algo = _ppo(minibatch_shuffle="device", shuffle_seed=11)
        epochs = []
        real = ops.make_permutation

        def spy(seed, first_epoch, n_epochs, n, device):
            epochs.append((first_epoch, n_epochs))
            return real(seed, first_epoch, n_epochs, n, device)
        monkeypatch.setattr(minibatch_order.ops, "make_permutation", spy)
        buf = _buffer()
        with policy_within_training_step(algo.policy):
            for _ in range(2):
                algo.update(buffer=buf, batch_size=256, repeat=R)
        assert epochs == [(0, R), (R, R)]


@pytest.mark.parametrize("path", list(PATHS))
def test_update_matches_direct_calls(path, monkeypatch):
    """``update()`` (order opened before ``_sample``) and direct ``_sample`` / ``_preprocess_batch`` / ``_update_with_batch``
    (order opened by ``_update_with_batch``) from the same seed: identical parameters, optimiser moments, step counters, loss
    tables and numpy state after two updates."""
    a, st_a = _two_updates(path, True, monkeypatch)
    b, st_b = _two_updates(path, False, monkeypatch)
    assert a.keys() == b.keys()
    for k in a:
        if isinstance(a[k], torch.Tensor):
            assert torch.isfinite(a[k].double()).all() and torch.equal(a[k], b[k]), k
        else:
            assert a[k] == b[k], k
    assert np.array_equal(st_a[1], st_b[1]) and st_a[2:] == st_b[2:]


@pytest.mark.parametrize("where", ["fused", "layered"])
def test_exception_in_a_pass_leaves_numpy_state_advanced(where, monkeypatch):
    """A Python exception raised after the first pass's work is enqueued propagates; the feed and the job are finished in
    order, numpy's state is the start state advanced by exactly ``repeat`` permutations (no warning), and the next
    ``update()`` draws the following rows and completes."""
    from tianshou_b200.algorithm.layered import LayeredActorCritic
    from tianshou_b200.algorithm.modelfree.ppo import FusedActorCriticUpdate
    from tianshou_b200.utils import policy_within_training_step
    if where == "layered":
        monkeypatch.setenv("TS_B200_FORCE_LAYERED", "1")
    algo = _ppo()
    assert (algo._layered is not None) == (where == "layered")
    buf = _buffer()
    R, N = 3, len(buf)
    cls, name = (LayeredActorCritic, "minibatch_step") if where == "layered" else (FusedActorCriticUpdate, "_device_passes")
    real = getattr(cls, name)

    def failing(self, *args, **kwargs):
        real(self, *args, **kwargs)
        raise RuntimeError("injected failure")
    monkeypatch.setattr(cls, name, failing)
    np.random.seed(4321)
    start = np.random.get_state()
    _permutations(start, N, R)
    after_first = np.random.get_state()
    ref = _permutations(start, N, 2 * R)
    np.random.set_state(start)
    with policy_within_training_step(algo.policy), warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        with pytest.raises(RuntimeError, match="injected failure"):
            algo.update(buffer=buf, batch_size=256, repeat=R)
        st = np.random.get_state()
        assert np.array_equal(st[1], after_first[1]) and st[2:] == after_first[2:]
        monkeypatch.setattr(cls, name, real)
        algo.update(buffer=buf, batch_size=256, repeat=R)
    torch.cuda.synchronize()
    assert not [w for w in caught if "numpy's global RNG" in str(w.message)]
    rows = algo._scratch["perms_dev"].cpu().numpy()
    assert all(np.array_equal(rows[r], ref[R + r]) for r in range(R))
    assert np.isfinite(algo.last_loss_table).all() and algo.last_loss_table.shape[0] == R * (N // 256)
