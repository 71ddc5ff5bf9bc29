"""Imitation learning on the GPU: both rows kernels against float64 (the restatement pinned to autograd in
test_oracle_imitation), ``update()`` against outputs of the imported reference (tests/golden/il_ref_*.npz from
oracle/gen_golden_imitation.py) with the device mirror on and off, the flat gradient of one update against float64 autograd, a
second batch size, the ``state_dict()`` round trip, the torch forward between updates, the priorities written back, the
refusals, the reference's four constructions and the register report."""
import copy

import numpy as np
import pytest
import torch

from oracle import oracle_imitation as oim
from offpolicy_testutil import (DEV, EPS, Box, Discrete, assert_spill_free, capture_batches, capture_grads, check_second_batch_size,
                                grid_caps, ptxas_report, rng_state, set_rng_state, stream, vector_buffer_from_golden)
from test_oracle_imitation import VARIANTS, b200_actor, b200_policy
from ts_testutil import load_golden, record_parity

gpu = pytest.mark.gpu
A_CASES = [1, 2, 6, 33, 70]


# ------------------------------------------------------------------------------------------------------------ rows kernels
def _mse(z, act, m):
    from tianshou_b200._cabi import call, ptr
    dz, loss = torch.empty_like(z), torch.empty(1, device=DEV)
    call("ts_imitation_mse_rows", ptr(z), ptr(act), z.shape[0], z.shape[1], m, ptr(dz), ptr(loss), stream())
    torch.cuda.synchronize()
    return float(loss.item()), dz.cpu().numpy()


def _nll(z, act, softmax):
    from tianshou_b200._cabi import call, ptr
    B, A = z.shape
    dz, rows, loss = torch.empty_like(z), torch.empty(B, device=DEV), torch.empty(1, device=DEV)
    call("ts_imitation_nll_rows", ptr(z), ptr(act), B, A, int(softmax), ptr(dz), ptr(rows), ptr(loss), stream())
    torch.cuda.synchronize()
    return float(loss.item()), dz.cpu().numpy(), rows.cpu().numpy()


def _batch_sizes(A, per_row):
    """1, 301, and past the launch's grid: more elements than the grid-stride kernel's threads, or more rows than the per-row
    kernel's warps."""
    caps = grid_caps()
    past = caps["warp_per_row"] + 37 if per_row else caps["offpolicy_1d"] // A + 37
    return [1, 301, past]


@gpu
@pytest.mark.parametrize("A", A_CASES)
def test_mse_rows_kernel_vs_fp64(A):
    """Saturated tanh (|z| >> 1) and targets outside +-max_action.  Each dz element is a few roundings of its float64 value; the
    loss is a fixed-order sum of B A non-negative terms."""
    m = 2.0
    for B in _batch_sizes(A, per_row=False):
        g = torch.Generator().manual_seed(B + A)
        z = torch.randn(B, A, generator=g) * 2
        z[: max(1, B // 5)] *= 30.0
        act = torch.randn(B, A, generator=g) * 3
        loss, dz = _mse(z.to(DEV), act.to(DEV), m)
        ref, rdz = oim.mse_rows(z.numpy(), act.numpy(), m)
        if B > 1:
            assert (np.abs(act.numpy()) > m).any() and (np.abs(z.numpy()) > 20).any()
        # tanh(z) carries a few ulps, which 1 - t^2 turns into an absolute error of the same size: bound each element by the scale of
        # 2 (pi - act) / n * max_action
        d64 = m * np.tanh(z.double().numpy()) - act.double().numpy()
        scale = float(np.abs(2.0 * d64 / (B * A) * m).max())
        record_parity(f"il_mse/A{A}_B{B}/loss", np.array([loss]), np.array([ref]), rtol=(np.ceil(B * A / 1024) + 16) * EPS * 4, atol=0.0)
        record_parity(f"il_mse/A{A}_B{B}/dz", dz, rdz, rtol=16 * EPS, atol=16 * EPS * scale)
        again = _mse(z.to(DEV), act.to(DEV), m)
        assert again[0] == loss and np.array_equal(again[1], dz), "two calls must be bit-identical"


@gpu
@pytest.mark.parametrize("softmax", [False, True], ids=["logits", "softmax_output"])
@pytest.mark.parametrize("A", A_CASES)
def test_nll_rows_kernel_vs_fp64(A, softmax):
    """Logit spreads that underflow the probabilities (a quarter of the rows times 40), with ``softmax_output`` on and off."""
    for B in _batch_sizes(A, per_row=True):
        g = torch.Generator().manual_seed(7 * B + A)
        z = torch.randn(B, A, generator=g) * 3
        z[: max(1, B // 4)] *= 40.0
        act = torch.randint(0, A, (B,), generator=g)
        loss, dz, rows = _nll(z.to(DEV), act.to(DEV), softmax)
        ref, rdz, rrows = oim.nll_rows(z.numpy(), act.numpy(), softmax)
        if B > 1 and A > 1:
            assert (np.exp(z.numpy() - z.numpy().max(1, keepdims=True)) == 0).any(), "some probabilities must underflow in fp32"
        k = (np.ceil(A / 32) + 10) * EPS
        tag = f"il_nll/A{A}_B{B}_{'sm' if softmax else 'logits'}"
        record_parity(f"{tag}/rows", rows, rrows, rtol=0.0, atol=float(8 * k * (np.abs(rrows).max() + np.abs(z.numpy()).max() + 1)))
        record_parity(f"{tag}/loss", np.array([loss]), np.array([ref]), rtol=(np.ceil(B / 1024) + 12) * EPS * 4,
                      atol=float(8 * k * (np.abs(z.numpy()).max() + 1)))
        record_parity(f"{tag}/dz", dz * B, rdz * B, rtol=0.0, atol=float(16 * k))
        again = _nll(z.to(DEV), act.to(DEV), softmax)
        assert again[0] == loss and np.array_equal(again[1], dz) and np.array_equal(again[2], rows), "two calls must be bit-identical"


# ------------------------------------------------------------------------------------------------------------ update vs goldens
def build_from_golden(g):
    from tianshou_b200.algorithm import AdamOptimizerFactory
    from tianshou_b200.algorithm.imitation import OfflineImitationLearning, OffPolicyImitationLearning
    policy = b200_policy(g, b200_actor(g).to(DEV))
    Algo = OffPolicyImitationLearning if str(g["cfg_algo"]) == "offpolicy" else OfflineImitationLearning
    return Algo(policy=policy, optim=AdamOptimizerFactory(lr=float(g["cfg_lr"])))


def check_final(tag, g, algo):
    """Final parameters and Adam moments within DESIGN.md section 4's bars: Adam normalises a step to ~lr per element, so the
    absolute term is stated in units of one step."""
    from oracle.oracle_discrete_sac import golden_view
    view = golden_view if bool(g["cfg_compact"]) else (lambda t: t.detach().cpu().numpy())
    lr, grp = float(g["cfg_lr"]), algo._group
    assert [id(p) for p in grp.params] == [id(p) for p in algo.policy.parameters()]
    for i, p in enumerate(grp.params):
        record_parity(f"{tag}/pf_{i}", view(p), g[f"pf_{i}"], rtol=1e-3, atol=0.1 * lr)
        m, v = g[f"m_{i}"], g[f"v_{i}"]
        record_parity(f"{tag}/m_{i}", view(grp.view(grp.exp_avg, p).view(p.shape)), m, rtol=2e-3, atol=2e-3 * float(np.abs(m).max()) + 1e-12)
        record_parity(f"{tag}/v_{i}", view(grp.view(grp.exp_avg_sq, p).view(p.shape)), v, rtol=4e-3, atol=4e-3 * float(np.abs(v).max()) + 1e-20)
    assert grp.sync_step_from_device() == int(g["adam_step"])


@gpu
@pytest.mark.parametrize("mirror", [False, True], ids=["host", "mirror"])
@pytest.mark.parametrize("variant", VARIANTS)
def test_update_matches_reference(variant, mirror):
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden(f"il_ref_{variant}.npz")
    algo, buf = build_from_golden(g), vector_buffer_from_golden(g, mirror)
    assert list(algo.state_dict().keys()) == [str(k) for k in g["state_dict_keys"]]
    with capture_batches(algo) as cap:
        for u in range(int(g["cfg_updates"])):
            np.random.seed(500 + u)
            with policy_within_training_step(algo.policy):
                stats = algo.update(buffer=buf, sample_size=int(g["cfg_bs"]))
            assert np.array_equal(cap["indices"], g[f"u{u}_indices"]), "sampled indices differ from the reference's"
            record_parity(f"il_{variant}_m{int(mirror)}_u{u}/loss", np.array([stats.loss]), np.array([float(g[f"u{u}_loss"])]),
                          rtol=2e-5, atol=2e-6)
            if variant == "per":        # the importance weight of the sample, written back untouched as the new priorities
                record_parity(f"il_per_m{int(mirror)}_u{u}/prio", cap["prio"].cpu().numpy(), g[f"u{u}_prio"], rtol=1e-6, atol=0.0)
            else:
                assert cap["prio"] is None
    check_final(f"il_{variant}_m{int(mirror)}", g, algo)
    if variant == "per":
        record_parity(f"il_per_m{int(mirror)}/leaves", np.asarray(buf.weight[np.arange(buf.maxsize)]), g["prio_leaves"], rtol=1e-6,
                      atol=0.0)


# ------------------------------------------------------------------------------------------------------------ gradient
GRAD_CASES = {    # a variant's layout on a synthetic buffer
    "cont": dict(kind="cont", obs=5, A=3, hidden=(48, 40), net_action=False, max_action=1.5, act_scale=2.5),
    "d4rl": dict(kind="cont", obs=17, A=6, hidden=(64,), net_action=True, max_action=1.0, act_scale=0.6),
    "disc_sm": dict(kind="mlp", obs=4, A=2, hidden=(64, 64), actor="discrete", softmax=True),
    "disc_logits": dict(kind="mlp", obs=9, A=40, hidden=(48,), actor="discrete", softmax=False),
    "net": dict(kind="mlp", obs=6, A=5, hidden=(32,), actor="net", softmax=False),
    "cnn": dict(kind="cnn", H=44, W=44, A=6, actor="dqnet", softmax=False),
}


def synthetic(cfg, B_max=256, seed=0, mirror=False):
    """A tianshou_b200 actor, ImitationPolicy and buffer of one layout (a stack_num=4 uint8 frame buffer for the CNN)."""
    from tianshou_b200.data import Batch, VectorReplayBuffer
    from tianshou_b200.env.atari.atari_network import DQNet
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.continuous import ContinuousActorDeterministic
    from tianshou_b200.utils.net.discrete import DiscreteActor
    from tianshou_b200.algorithm.imitation import ImitationPolicy
    actor = oim.make_actor(cfg, (Net, ContinuousActorDeterministic, DiscreteActor, DQNet)).to(DEV)
    cont, cnn = cfg["kind"] == "cont", cfg["kind"] == "cnn"
    space = Box(cfg["A"], cfg["max_action"]) if cont else Discrete(cfg["A"])
    policy = ImitationPolicy(actor=actor, action_space=space)
    rng = np.random.default_rng(seed)
    E, T = 4, max(B_max // 4, 16)
    kw = dict(stack_num=4, ignore_obs_next=True, save_only_last_obs=True) if cnn else {}
    buf = VectorReplayBuffer(E * T, E, device=DEV, device_mirror=mirror, **kw)
    for _ in range(T):
        if cnn:
            obs = np.repeat(rng.integers(0, 256, (E, cfg["H"], cfg["W"]), dtype=np.uint8)[:, None], 4, axis=1)
        else:
            obs = rng.standard_normal((E, cfg["obs"])).astype(np.float32)
        act = (rng.standard_normal((E, cfg["A"])) * cfg["act_scale"]).astype(np.float32) if cont else rng.integers(0, cfg["A"], E)
        term = rng.random(E) < 0.05
        buf.add(Batch(obs=obs, act=act, rew=rng.standard_normal(E), terminated=term, truncated=np.zeros(E, bool) & ~term,
                      obs_next=obs), buffer_ids=np.arange(E))
    return policy, buf


def _algo(policy, lr=1e-3):
    from tianshou_b200.algorithm import AdamOptimizerFactory
    from tianshou_b200.algorithm.imitation import OffPolicyImitationLearning
    return OffPolicyImitationLearning(policy=policy, optim=AdamOptimizerFactory(lr=lr))


@gpu
@pytest.mark.parametrize("B", [1, 64, 65, 200])
@pytest.mark.parametrize("case", list(GRAD_CASES))
def test_update_gradient_vs_fp64_autograd(case, B):
    """The flat gradient before the Adam step against float64 autograd of the reference loss on a copy of the actor.  The GEMMs
    are fp32-faithful (bf16x3) and a weight gradient sums B products per element: 2e-4 relative plus 1e-4 of the tensor's
    largest value, as in test_discrete_bcq_gpu."""
    from tianshou_b200.utils import policy_within_training_step
    cfg = GRAD_CASES[case]
    policy, buf = synthetic(cfg, seed=B)
    algo = _algo(policy)
    ref = oim.ImitationState(copy.deepcopy(policy.actor).cpu(), 1e-3)
    np.random.seed(B)
    with capture_batches(algo) as cap, capture_grads(algo._group) as grads, policy_within_training_step(algo.policy):
        stats = algo.update(buffer=buf, sample_size=B)
    idx = cap["indices"]
    assert len(idx) == B
    r = oim.imitation_update(ref, np.asarray(buf[idx].obs), np.asarray(buf.act)[idx], cfg["kind"],
                             cfg.get("max_action", 1.0), cfg.get("softmax", False))
    grp = algo._group
    for i, (p, gr) in enumerate(zip(grp.params, r["grads"], strict=True)):
        want = gr.numpy()
        got = grp.view(grads[-1], p).view(p.shape).cpu().numpy()
        record_parity(f"il_grad/{case}_B{B}/grad_{i}", got, want, rtol=2e-4, atol=1e-4 * float(np.abs(want).max()) + 1e-12)
    record_parity(f"il_grad/{case}_B{B}/loss", np.array([stats.loss]), np.array([r["loss"]]), rtol=5e-5, atol=5e-6)


@gpu
@pytest.mark.parametrize("case", ["d4rl", "disc_logits", "cnn"])
def test_second_batch_size_is_independent_of_the_first(case):
    cfg = GRAD_CASES[case]
    policy, buf = synthetic(cfg, seed=3)

    def build():
        return _algo(copy.deepcopy(policy))

    check_second_batch_size(build, buf, 200, 65, name=case)


@gpu
@pytest.mark.parametrize("case", ["cont", "disc_sm"])
def test_state_dict_round_trip_continues_identically(case):
    from tianshou_b200.utils import policy_within_training_step
    cfg = GRAD_CASES[case]
    policy, buf = synthetic(cfg, seed=5)
    a = _algo(copy.deepcopy(policy))
    for u in range(3):
        np.random.seed(u)
        with policy_within_training_step(a.policy):
            a.update(buffer=buf, sample_size=64)
    b = _algo(copy.deepcopy(policy))
    with torch.no_grad():
        for p in b.parameters():
            p.add_(0.01)
    b.load_state_dict(copy.deepcopy(a.state_dict()))
    rng = rng_state(buf)          # the buffer draws indices from its own streams: both continue from the same state
    for algo in (a, b):
        set_rng_state(buf, rng)
        for u in range(3):
            np.random.seed(10 + u)
            with policy_within_training_step(algo.policy):
                algo.update(buffer=buf, sample_size=64)
    ga, gb = a._group, b._group
    assert torch.equal(ga.flat, gb.flat) and torch.equal(ga.exp_avg, gb.exp_avg) and torch.equal(ga.exp_avg_sq, gb.exp_avg_sq)
    assert ga.sync_step_from_device() == gb.sync_step_from_device() == 6


@gpu
@pytest.mark.parametrize("case", ["cont", "disc_sm", "cnn"])
def test_torch_forward_between_updates(case):
    """The Collector's path, ``ImitationPolicy.forward``, between two updates: it reads the device parameters, leaves the Adam
    state alone, and the next update is bit-identical to one without that forward."""
    from tianshou_b200.data import Batch
    from tianshou_b200.utils import policy_within_training_step
    cfg = GRAD_CASES[case]
    policy, buf = synthetic(cfg, seed=11)
    a, b = _algo(copy.deepcopy(policy)), _algo(copy.deepcopy(policy))
    obs = np.asarray(buf[np.arange(8)].obs)
    rng = rng_state(buf)          # the buffer draws indices from its own streams: both instances take the same draws
    for algo in (a, b):
        set_rng_state(buf, rng)
        np.random.seed(1)
        with policy_within_training_step(algo.policy):
            algo.update(buffer=buf, sample_size=64)
    state = [t.clone() for t in (a._group.exp_avg, a._group.exp_avg_sq)]
    with torch.no_grad():
        out = a.policy(Batch(obs=obs, info=Batch()))
        y, _ = b.policy.actor(obs)          # the same parameters, read through the other instance's modules
    assert torch.equal(out.logits, y)
    assert torch.equal(out.act, y.argmax(1) if cfg["kind"] != "cont" else y)
    ref = copy.deepcopy(policy.actor)      # the updated parameters, read by plain torch from the flat buffer
    with torch.no_grad():
        for p, q in zip(ref.parameters(), a._group.params, strict=True):
            p.copy_(a._group.view(a._group.flat, q).view(q.shape))
        assert torch.equal(ref(obs)[0], out.logits)
    assert all(torch.equal(s, t) for s, t in zip(state, (a._group.exp_avg, a._group.exp_avg_sq)))
    rng = rng_state(buf)
    for algo in (a, b):
        set_rng_state(buf, rng)
        np.random.seed(2)
        with policy_within_training_step(algo.policy):
            algo.update(buffer=buf, sample_size=64)
    assert torch.equal(a._group.flat, b._group.flat) and torch.equal(a._group.exp_avg_sq, b._group.exp_avg_sq)


# ------------------------------------------------------------------------------------------------------------ refusals
@gpu
def test_refusals():
    from tianshou_b200.algorithm import AdamOptimizerFactory, RMSpropOptimizerFactory, UnsupportedModelError
    from tianshou_b200.algorithm.imitation import ImitationPolicy, OffPolicyImitationLearning
    from tianshou_b200.data import Batch, VectorReplayBuffer
    from tianshou_b200.utils import policy_within_training_step
    from tianshou_b200.utils.net.common import Net, Recurrent
    from tianshou_b200.utils.net.continuous import ContinuousActorDeterministic, ContinuousActorProbabilistic
    from tianshou_b200.utils.net.discrete import DiscreteActor

    def make(actor, space, optim=None):
        return OffPolicyImitationLearning(policy=ImitationPolicy(actor=actor, action_space=space),
                                          optim=optim or AdamOptimizerFactory(lr=1e-3))

    cont = ContinuousActorDeterministic(preprocess_net=Net(state_shape=(5,), hidden_sizes=(16,)), action_shape=3, max_action=1.0)
    make(cont.to(DEV), Box(3, 1.0))
    with pytest.raises(UnsupportedModelError, match="probabilistic actor"):
        make(ContinuousActorProbabilistic(preprocess_net=Net(state_shape=(5,), hidden_sizes=(16,)), action_shape=3).to(DEV), Box(3, 1.0))
    with pytest.raises(UnsupportedModelError, match="3 outputs for an action of dimension 2"):
        make(copy.deepcopy(cont).to(DEV), Box(2, 1.0))
    with pytest.raises(UnsupportedModelError, match="no CPU path"):
        make(copy.deepcopy(cont).cpu(), Box(3, 1.0))
    with pytest.raises(UnsupportedModelError, match="supports torch.optim.Adam only, got RMSprop"):
        make(copy.deepcopy(cont).to(DEV), Box(3, 1.0), RMSpropOptimizerFactory(lr=1e-3))
    with pytest.raises(UnsupportedModelError, match="DQN"):
        make(Recurrent(layer_num=1, state_shape=(4,), action_shape=3).to(DEV), Discrete(3))
    with pytest.raises(UnsupportedModelError, match="5 outputs for 3 actions"):
        make(Net(state_shape=(4,), action_shape=5, hidden_sizes=(16,)).to(DEV), Discrete(3))
    with pytest.raises(UnsupportedModelError, match="4 outputs for 3 actions"):
        make(DiscreteActor(preprocess_net=Net(state_shape=(4,), hidden_sizes=(16,)), action_shape=4).to(DEV), Discrete(3))
    with pytest.raises(UnsupportedModelError, match="linear layer"):
        make(Net(state_shape=(4,), hidden_sizes=(16, 3)).to(DEV), Discrete(3))
    # a continuous buffer whose action rows have another width
    algo = make(copy.deepcopy(cont).to(DEV), Box(3, 1.0))
    buf = VectorReplayBuffer(64, 2, device=DEV)
    for _ in range(8):
        buf.add(Batch(obs=np.zeros((2, 5), np.float32), act=np.zeros((2, 2), np.float32), rew=np.zeros(2),
                      terminated=np.zeros(2, bool), truncated=np.zeros(2, bool), obs_next=np.zeros((2, 5), np.float32)),
                buffer_ids=np.arange(2))
    with pytest.raises(UnsupportedModelError, match="action rows of width 2"), policy_within_training_step(algo.policy):
        algo.update(buffer=buf, sample_size=8)


# ------------------------------------------------------------------------------------------------------------ constructions
@gpu
def test_reference_constructions_take_a_device_update():
    """The model and policy code of the imitation halves of test_sac_with_il.py and test_a2c_with_il.py, of d4rl_il.py and of
    atari_il.py, each taking one device ``update()`` on a synthetic buffer."""
    from tianshou_b200.algorithm import AdamOptimizerFactory, OffPolicyImitationLearning
    from tianshou_b200.algorithm.imitation.imitation_base import ImitationPolicy, OfflineImitationLearning
    from tianshou_b200.data import Batch, VectorReplayBuffer
    from tianshou_b200.env.atari.atari_network import DQNet
    from tianshou_b200.utils import policy_within_training_step
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.continuous import ContinuousActorDeterministic
    from tianshou_b200.utils.net.discrete import DiscreteActor

    def run(algo, obs_fn, act_fn, stack=False):
        rng = np.random.default_rng(0)
        kw = dict(stack_num=4, ignore_obs_next=True, save_only_last_obs=True) if stack else {}
        buf = VectorReplayBuffer(256, 4, device=DEV, **kw)
        for _ in range(40):
            o = obs_fn(rng)
            buf.add(Batch(obs=o, act=act_fn(rng), rew=np.zeros(4), terminated=np.zeros(4, bool), truncated=np.zeros(4, bool),
                          obs_next=o), buffer_ids=np.arange(4))
        with policy_within_training_step(algo.policy):
            stats = algo.update(buffer=buf, sample_size=32)
        assert np.isfinite(stats.loss) and stats.loss > 0
        return stats

    # test/continuous/test_sac_with_il.py (Pendulum: obs 3, action 1, max_action 2)
    il_net = Net(state_shape=(3,), hidden_sizes=[128, 128])
    il_actor = ContinuousActorDeterministic(preprocess_net=il_net, action_shape=(1,), max_action=2.0).to(DEV)
    il_policy = ImitationPolicy(actor=il_actor, action_space=Box(1, 2.0), action_scaling=True, action_bound_method="clip")
    run(OffPolicyImitationLearning(policy=il_policy, optim=AdamOptimizerFactory(lr=1e-3)),
        lambda r: r.standard_normal((4, 3)).astype(np.float32), lambda r: (r.standard_normal((4, 1)) * 3).astype(np.float32))
    # test/discrete/test_a2c_with_il.py (CartPole: obs 4, 2 actions)
    net = Net(state_shape=(4,), hidden_sizes=[64, 64])
    actor = DiscreteActor(preprocess_net=net, action_shape=2).to(DEV)
    il_policy = ImitationPolicy(actor=actor, action_space=Discrete(2))
    run(OffPolicyImitationLearning(policy=il_policy, optim=AdamOptimizerFactory(lr=1e-3)),
        lambda r: r.standard_normal((4, 4)).astype(np.float32), lambda r: r.integers(0, 2, 4))
    # examples/offline/d4rl_il.py (halfcheetah: obs 17, action 6)
    net = Net(state_shape=(17,), action_shape=(6,), hidden_sizes=[256, 256])
    actor = ContinuousActorDeterministic(preprocess_net=net, action_shape=(6,), max_action=1.0).to(DEV)
    policy = ImitationPolicy(actor=actor, action_space=Box(6, 1.0), action_scaling=True, action_bound_method="clip")
    run(OfflineImitationLearning(policy=policy, optim=AdamOptimizerFactory(lr=1e-4)),
        lambda r: r.standard_normal((4, 17)).astype(np.float32), lambda r: r.uniform(-1, 1, (4, 6)).astype(np.float32))
    # examples/offline/atari_il.py (4 x 84 x 84 frames, 6 actions)
    net = DQNet(c=4, h=84, w=84, action_shape=6).to(DEV)
    policy = ImitationPolicy(actor=net, action_space=Discrete(6))
    run(OfflineImitationLearning(policy=policy, optim=AdamOptimizerFactory(lr=1e-4)),
        lambda r: np.repeat(r.integers(0, 256, (4, 84, 84), dtype=np.uint8)[:, None], 4, axis=1), lambda r: r.integers(0, 6, 4),
        stack=True)


# ------------------------------------------------------------------------------------------------------------ resources
def test_kernels_have_no_stack_frame_or_spills(tmp_path):
    report = ptxas_report("imitation.cu", tmp_path)
    ours = {e: v for e, v in report.items() if "imitation_" in e}      # row_sums.cuh's shared kernel is compiled in as well
    assert len(ours) == 4, report
    assert_spill_free(ours)
