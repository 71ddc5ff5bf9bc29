"""TD3 / TD3+BC on the GPU: the td3.cu kernels against float64 references, ``update()`` against outputs of the imported reference
(tests/golden/td3_ref_*.npz from oracle/gen_golden_td3.py) with the buffer mirror on and off, the gradients of every optimiser
step against float64 autograd of the eager restatement, the delayed actor and lagged networks, the absence of host
synchronisation inside the update, ``state_dict()`` round trips, the refusals and the kernels' register report."""
import copy
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from ts_testutil import load_golden, record_parity

DEV = "cuda:0"
gpu = pytest.mark.gpu
KEYS = ("obs", "act", "rew", "terminated", "truncated", "obs_next")


class _Box:
    def __init__(self, dim, m=1.0):
        self.shape = (dim,)
        self.low = -m * np.ones(dim, np.float32)
        self.high = m * np.ones(dim, np.float32)


def _st():
    from tianshou_b200._cabi import stream_ptr
    return stream_ptr(torch.device(DEV))


# ------------------------------------------------------------------------------------------------------------ kernels
ACT_CASES = [(7, 5, 3, 1.0, 0.5, True), (300000, 17, 6, 2.5, 0.5, True), (1000, 11, 4, 2.0, 0.0, True), (300000, 4, 3, 1.0, 0.5, False)]


@gpu
@pytest.mark.parametrize("B,O,A,m,clip,noisy", ACT_CASES, ids=[f"B{c[0]}-O{c[1]}-A{c[2]}-m{c[3]}-clip{c[4]}-noise{int(c[5])}" for c in ACT_CASES])
def test_act_rows_kernel_vs_fp64(B, O, A, m, clip, noisy):
    """[s | max_action * tanh(z) (+ clamp(noise * policy_noise))], every row written past the grid cap, no clamp at noise_clip 0,
    and no clip back to the action bounds."""
    from tianshou_b200._cabi import call, ptr
    g = torch.Generator().manual_seed(B + O)
    z, obs, noise = torch.randn(B, A, generator=g) * 2, torch.randn(B, O, generator=g), torch.randn(B, A, generator=g)
    pn = 0.7
    d = [t.to(DEV).contiguous() for t in (z, obs, noise)]
    x = torch.full((B, O + A), float("nan"), device=DEV)
    call("ts_td3_act_rows", ptr(d[0]), ptr(d[2]) if noisy else None, B, A, m, pn, clip, ptr(d[1]), O, ptr(x), _st())
    torch.cuda.synchronize()
    a = m * torch.tanh(z.double())
    if noisy:
        n = noise.double() * np.float32(pn)
        a = a + (n.clamp(-clip, clip) if clip > 0 else n)
    ref = torch.cat([obs.double(), a], dim=1)
    tag = f"td3_act_rows/B{B}_A{A}_m{m}_clip{clip}_n{int(noisy)}"
    record_parity(tag, x.cpu().numpy(), ref.numpy(), rtol=1e-6, atol=1e-6)
    assert torch.equal(x[:, :O].cpu(), obs)
    if noisy and clip == 0.0:
        assert float(x[:, O:].abs().max()) > m, "the smoothed action is not clipped back to the bounds"


@gpu
@pytest.mark.parametrize("B", [5, 300000])
def test_target_min_kernel(B):
    from tianshou_b200._cabi import call, ptr
    g = torch.Generator().manual_seed(B)
    q1, q2 = torch.randn(B, generator=g), torch.randn(B, generator=g)
    q1[0] = float("nan")
    d = [t.to(DEV) for t in (q1, q2)]
    out = torch.empty(B, device=DEV)
    call("ts_td3_target_min", ptr(d[0]), ptr(d[1]), B, ptr(out), _st())
    torch.cuda.synchronize()
    assert torch.equal(out.cpu().nan_to_num(-7.0), torch.min(q1, q2).nan_to_num(-7.0))


def _actor_kernels(q, z, act, dact, B, A, m, alpha):
    from tianshou_b200._cabi import call, ptr
    dq, loss, dz = torch.full((B,), float("nan"), device=DEV), torch.full((1,), float("nan"), device=DEV), torch.empty(B, A, device=DEV)
    call("ts_td3_actor_rows", ptr(q), ptr(z), ptr(act), B, A, m, alpha, ptr(dq), ptr(loss), _st())
    call("ts_td3_actor_head_bwd", ptr(z), ptr(dact), ptr(act), B, A, m, ptr(dz), _st())
    torch.cuda.synchronize()
    return dq, loss, dz


ROW_CASES = [(256, 6, 1.0, False), (256, 6, 1.0, True), (70000, 17, 2.0, True), (3000, 3, 1.5, False)]


@gpu
@pytest.mark.parametrize("B,A,m,bc", ROW_CASES, ids=[f"B{c[0]}-A{c[1]}-m{c[2]}-{'bc' if c[3] else 'td3'}" for c in ROW_CASES])
def test_actor_rows_and_head_backward_vs_fp64_autograd(B, A, m, bc):
    """TD3's -mean(q) and TD3+BC's -lmbda mean(q) + mse(pi, a) with lmbda = alpha / mean|q| detached, |q| spanning 1e4; dq, the
    loss and dz = d loss / dz (through dact from critic 1 and the BC term) against float64 autograd; two runs bit-identical."""
    g = torch.Generator().manual_seed(B + A)
    q = torch.randn(B, generator=g) * torch.pow(10.0, torch.empty(B).uniform_(-2.0, 2.0, generator=g))
    z, dact = torch.randn(B, A, generator=g) * 1.5, torch.randn(B, A, generator=g) / B
    act = (m * torch.tanh(torch.randn(B, A, generator=g))) if bc else None
    alpha = 2.5
    d = lambda t: None if t is None else t.to(DEV).contiguous()
    args = (d(q), d(z), d(act), d(dact), B, A, m, alpha)
    dq, loss, dz = _actor_kernels(*args)
    qq, zz = q.double().requires_grad_(True), z.double().requires_grad_(True)
    pi = m * torch.tanh(zz)
    if bc:
        lmbda = alpha / qq.abs().mean().detach()
        ref_loss = -lmbda * qq.mean() + torch.nn.functional.mse_loss(pi, act.double())
    else:
        ref_loss = -qq.mean()
    (ref_loss + (pi * dact.double()).sum()).backward()
    tag = f"td3_actor_rows/B{B}_A{A}_m{m}_{'bc' if bc else 'td3'}"
    record_parity(f"{tag}/loss", loss.cpu().numpy(), np.array([ref_loss.item()]), rtol=1e-5, atol=1e-6)
    record_parity(f"{tag}/dq", dq.cpu().numpy(), qq.grad.numpy(), rtol=1e-5, atol=1e-12)
    record_parity(f"{tag}/dz", dz.cpu().numpy(), zz.grad.numpy(), rtol=1e-5, atol=1e-6 * float(zz.grad.abs().max()))
    again = _actor_kernels(*args)
    for a, b in zip((dq, loss, dz), again, strict=True):
        assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------------------ goldens
def _cfg(g):
    return {k[4:]: g[k] for k in g.files if k.startswith("cfg_")}


def _load(mod, g, prefix):
    with torch.no_grad():
        for i, p in enumerate(mod.parameters()):
            p.copy_(torch.as_tensor(g[f"{prefix}{i}"]).reshape(p.shape))


def _check_params(tag, mod, g, prefix, lr):
    for i, p in enumerate(mod.parameters()):
        record_parity(f"{tag}/{prefix}{i}", p.detach().cpu().numpy(), g[f"{prefix}{i}"], rtol=1e-3, atol=0.1 * lr)


def _nets(O, A, H, m=1.0, last_hidden=()):
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.continuous import ContinuousActorDeterministic, ContinuousCritic
    actor = ContinuousActorDeterministic(preprocess_net=Net(state_shape=(O,), hidden_sizes=H), action_shape=(A,), hidden_sizes=last_hidden,
                                         max_action=m).to(DEV)
    crit = lambda: ContinuousCritic(preprocess_net=Net(state_shape=(O,), action_shape=(A,), hidden_sizes=H, concat=True)).to(DEV)
    return actor, crit


def _build(cfg, g=None, **over):
    from tianshou_b200.algorithm import TD3, TD3BC, AdamOptimizerFactory
    from tianshou_b200.algorithm.modelfree.ddpg import ContinuousDeterministicPolicy
    O, A, H, m = int(cfg["obs"]), int(cfg["act"]), tuple(int(x) for x in cfg["hidden"]), float(cfg["max_action"])
    actor, crit = _nets(O, A, H, m)
    c1 = crit()
    c2 = crit() if bool(cfg["critic2"]) else None
    if g is not None:
        _load(actor, g, "p0_actor_"); _load(c1, g, "p0_c1_")
        if c2 is not None:
            _load(c2, g, "p0_c2_")
    policy = ContinuousDeterministicPolicy(actor=actor, action_space=_Box(A, m), action_scaling=bool(cfg["action_scaling"]))
    kw = dict(policy=policy, policy_optim=AdamOptimizerFactory(lr=float(cfg["actor_lr"])), critic=c1,
              critic_optim=AdamOptimizerFactory(lr=float(cfg["critic_lr"])), critic2=c2,
              critic2_optim=AdamOptimizerFactory(lr=float(cfg["critic2_lr"])) if c2 is not None else None, tau=float(cfg["tau"]),
              gamma=float(cfg["gamma"]), policy_noise=float(cfg["policy_noise"]), update_actor_freq=int(cfg["freq"]),
              noise_clip=float(cfg["noise_clip"]), n_step_return_horizon=int(cfg["n_step"]))
    kw.update(over)
    if str(cfg["algo"]) == "bc":
        return TD3BC(alpha=float(cfg["alpha"]), **kw)
    return TD3(**kw)


def _buffer(g, mirror):
    from tianshou_b200.data import Batch, PrioritizedReplayBuffer, ReplayBuffer
    cfg = _cfg(g)
    if int(cfg["adds"]) == 0:
        buf = ReplayBuffer.from_data(*(g["buf_" + k].copy() for k in ("obs", "act", "rew", "terminated", "truncated", "done", "obs_next")))
    else:
        size = int(cfg["size"])
        buf = (PrioritizedReplayBuffer(size, alpha=float(cfg["per_alpha"]), beta=float(cfg["per_beta"]), device=DEV) if bool(cfg["per"])
               else ReplayBuffer(size, device=DEV))
        for i in range(int(cfg["adds"])):
            buf.add(Batch(**{k: g["add_" + k][i] for k in KEYS}, info={}))
    for k in (*KEYS, "done"):
        assert np.array_equal(np.asarray(buf._meta[k]), g["buf_" + k]), f"rebuilt buffer differs in {k}"
    if mirror:
        buf.enable_device_mirror()
        buf.sync_device_mirror()
        assert buf.device_columns() is not None
    return buf


def _cpu_noise(shape):
    """The reference ran on the CPU: torch.randn on the CPU generator, uploaded."""
    return torch.randn(shape).to(DEV)


@gpu
@pytest.mark.parametrize("mirror", [False, True])
@pytest.mark.parametrize("variant", ["mujoco", "per_nstep", "bc", "bc_freq1"])
def test_update_matches_reference(variant, mirror):
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden(f"td3_ref_{variant}.npz")
    cfg = _cfg(g)
    algo = _build(cfg, g)
    assert sorted(algo.state_dict().keys()) == list(g["state_dict_keys"]), "state_dict() keys differ from the reference's"
    buf = _buffer(g, mirror)
    algo._noise_fn = _cpu_noise
    captured = {}
    orig = algo._preprocess_batch

    def hook(batch, buffer, indices):
        captured["indices"] = np.asarray(indices).copy()
        if bool(cfg["per"]):
            captured["is_weight"] = batch.weight.detach().cpu().numpy().copy()
        return orig(batch, buffer, indices)

    algo._preprocess_batch = hook
    lr, a_lr = float(cfg["critic_lr"]), float(cfg["actor_lr"])
    c2_lr = float(cfg["critic2_lr"]) if bool(cfg["critic2"]) else lr
    for u in range(int(cfg["updates"])):
        np.random.seed(500 + u)
        torch.manual_seed(100 + u)
        with policy_within_training_step(algo.policy):
            stats = algo.update(buf, int(cfg["bs"]))
        o, tag = f"u{u}_", f"td3/{variant}_m{int(mirror)}_u{u}"
        assert np.array_equal(captured["indices"], g[o + "indices"]), "sampled indices differ from the reference's"
        assert np.array_equal(torch.get_rng_state().numpy(), g[o + "torch_rng"]), "CPU generator differs from the reference's"
        record_parity(f"{tag}/losses", np.array([stats.actor_loss, stats.critic1_loss, stats.critic2_loss]), g[o + "losses"],
                      rtol=2e-5, atol=2e-6)
        if bool(cfg["per"]):
            record_parity(f"{tag}/is_weight", captured["is_weight"], g[o + "is_weight"], rtol=1e-6, atol=1e-7)
            record_parity(f"{tag}/priorities", np.asarray(buf.weight[np.arange(len(buf))]), g[o + "priorities"], rtol=1e-3, atol=1e-6)
        _check_params(tag, algo.policy.actor, g, o + "actor_", a_lr)
        _check_params(tag, algo.critic, g, o + "c1_", lr); _check_params(tag, algo.critic2, g, o + "c2_", c2_lr)
        _check_params(tag, algo.critic_old, g, o + "c1old_", lr); _check_params(tag, algo.critic2_old, g, o + "c2old_", c2_lr)
        _check_params(tag, algo.actor_old, g, o + "aold_", a_lr)


@gpu
def test_delayed_actor_and_lagged_networks():
    """update_actor_freq=2: the actor and all three lagged networks move on updates 0, 2, ...; on the others the lagged networks
    are bit-unchanged, the actor too, and actor_loss repeats the last actor step's loss."""
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden("td3_ref_mujoco.npz")
    algo = _build(_cfg(g), g)
    buf = _buffer(g, mirror=True)
    assert algo._cnt == 0 and algo._last == 0
    groups = lambda: [t.flat.clone() for t in (algo._g_actor, *algo._g_ct, algo._g_at)]
    last = None
    for u in range(4):
        before = groups()
        with policy_within_training_step(algo.policy):
            stats = algo.update(buf, 32)
        after = groups()
        moved = [not torch.equal(a, b) for a, b in zip(before, after, strict=True)]
        if u % 2 == 0:
            assert all(moved), moved
            last = stats.actor_loss
        else:
            assert not any(moved), moved
            assert stats.actor_loss == last
    assert algo._cnt == 4
    assert not any(k.startswith("_cnt") or k.startswith("_last") for k in algo.state_dict())


# ------------------------------------------------------------------------------------------------------------ gradients
class _Recorder(torch.optim.Adam):
    """Adam that keeps the gradient it is about to apply."""

    def step(self, closure=None):
        self.seen = [p.grad.detach().clone() for g in self.param_groups for p in g["params"]]
        return super().step(closure)


def _random_buffer(O, A, n, seed, m=1.0):
    from tianshou_b200.data import ReplayBuffer
    rng = np.random.default_rng(seed)
    term = rng.random(n) < 0.05
    term[[0, -1]] = True                      # episode ends at both ends (see oracle/gen_golden_td3.py)
    trunc = (rng.random(n) < 0.03) & ~term
    return ReplayBuffer.from_data(rng.standard_normal((n, O)).astype(np.float32), (m * np.tanh(rng.standard_normal((n, A)))).astype(np.float32),
                                  rng.standard_normal(n), term, trunc, term | trunc, rng.standard_normal((n, O)).astype(np.float32))


GRAD_CASES = [(17, 6, (256, 256), "td3"), (17, 6, (256, 256), "bc"), (376, 17, (64, 64), "td3"), (376, 17, (64, 64), "bc")]


@gpu
@pytest.mark.parametrize("O,A,H,algo_kind", GRAD_CASES, ids=[f"O{c[0]}-A{c[1]}-{c[3]}" for c in GRAD_CASES])
def test_update_gradients_vs_fp64_autograd(O, A, H, algo_kind):
    """Two updates at batch 256 with n = 3 and max_action 2: an actor step, then a critic-only step.  Each critic step's
    gradient, taken before its Adam step, against float64 autograd of the eager restatement on copies of the modules with the same
    batch and target noise; the actor step's against float64 autograd of the actor loss on the pre-update actor and the critic 1
    the update stepped (the actor step runs against the updated critic, whose Adam step is lr * sign(g) and so moves a weight by
    2 lr where a tiny gradient's sign differs).  This is the check that sees a gradient off by a factor."""
    from oracle.oracle_td3 import Td3Nets, actor_objective, td3_update
    from tianshou_b200.algorithm.flat_params import FlatGroup
    from tianshou_b200.utils import policy_within_training_step
    m, B = 2.0, 256
    cfg = dict(obs=O, act=A, hidden=H, max_action=m, critic2=True, critic2_lr=1e-3, action_scaling=False, actor_lr=1e-4,
               critic_lr=3e-4, tau=0.005, gamma=0.99, policy_noise=0.2, freq=2, noise_clip=0.5, n_step=3, algo=algo_kind, alpha=2.5)
    torch.manual_seed(3)
    algo = _build(cfg)
    buf = _random_buffer(O, A, 700, seed=O + A, m=m)
    noises = []

    def noise(shape):
        noises.append(torch.randn(shape, device=DEV))
        return noises[-1]

    algo._noise_fn = noise
    names = {id(algo._g_actor): "actor", id(algo._g_c[0]): "c1", id(algo._g_c[1]): "c2"}
    cap = {}

    def adam(group, optimizer, mgn):
        cap[names[id(group)]] = group.grad[:group.n].detach().cpu().double().clone()
        FlatGroup.adam_step(group, optimizer, mgn)

    algo._adam = adam
    orig = algo._preprocess_batch
    algo._preprocess_batch = lambda b, buffer, idx: (cap.update(indices=np.asarray(idx).copy()), orig(b, buffer, idx))[1]
    d = {k: np.asarray(buf._meta[k]) for k in ("obs", "act", "rew", "done", "terminated", "obs_next")}
    d.update(offset=np.array([0, len(buf)]), last_index=np.asarray(buf.last_index), lengths=np.array([len(buf)]),
             unfinished=[] if d["done"][len(buf) - 1] else [len(buf) - 1])
    for u, actor_step in enumerate((True, False)):
        nets = Td3Nets(O, A, H, m)
        with torch.no_grad():
            for dst, src in ((nets.a, algo.policy.actor), (nets.c[0], algo.critic), (nets.c[1], algo.critic2),
                             (nets.a_old, algo.actor_old), (nets.c_old[0], algo.critic_old), (nets.c_old[1], algo.critic2_old)):
                for p, q in zip(dst.parameters(), src.parameters(), strict=True):
                    p.copy_(q.detach().cpu())
        for mod in nets.modules():
            mod.double()
        actor_before = [p.detach().clone() for p in algo.policy.actor.parameters()]
        cap.clear(); noises.clear()
        with policy_within_training_step(algo.policy):
            stats = algo.update(buf, B)
        torch.cuda.synchronize()
        if actor_step:                        # the actor loss on the pre-update actor and the stepped critic 1, float64
            anets = Td3Nets(O, A, H, m)
            with torch.no_grad():
                for p, q in zip(anets.a.parameters(), actor_before, strict=True):
                    p.copy_(q.cpu())
                for p, q in zip(anets.c[0].parameters(), algo.critic.parameters(), strict=True):
                    p.copy_(q.detach().cpu())
            anets.a.double(); anets.c[0].double()
            f64 = lambda k: torch.as_tensor(d[k][cap["indices"]]).double()
            loss = actor_objective(anets, f64("obs"), f64("act"), 2.5 if algo_kind == "bc" else None)
            grads = torch.autograd.grad(loss, list(anets.a.parameters()))
            want = torch.cat([x.reshape(-1) for x in grads]).numpy()
            record_parity(f"td3_grad/O{O}_A{A}_{algo_kind}_u{u}/grad_actor", cap["actor"].numpy(), want, rtol=2e-4,
                          atol=1e-4 * float(np.abs(want).max()) + 1e-12)
            record_parity(f"td3_grad/O{O}_A{A}_{algo_kind}_u{u}/actor_loss", np.array([stats.actor_loss]), np.array([loss.item()]),
                          rtol=2e-5, atol=1e-5)
        assert set(cap) == ({"indices", "actor", "c1", "c2"} if actor_step else {"indices", "c1", "c2"})
        it = iter(noises)
        opts = [_Recorder(nets.a.parameters(), lr=1e-4), _Recorder(nets.c[0].parameters(), lr=3e-4), _Recorder(nets.c[1].parameters(), lr=1e-3)]
        ref = td3_update(nets, opts, d, cap["indices"], lambda shape: next(it).double().cpu(), gamma=0.99, n_step=3, tau=0.005,
                         policy_noise=0.2, noise_clip=0.5, actor_step=actor_step, bc_alpha=2.5 if algo_kind == "bc" else None)
        tag = f"td3_grad/O{O}_A{A}_{algo_kind}_u{u}"
        for name, opt in (("c1", opts[1]), ("c2", opts[2])):
            want = torch.cat([x.reshape(-1) for x in opt.seen]).numpy()
            record_parity(f"{tag}/grad_{name}", cap[name].numpy(), want, rtol=2e-4, atol=1e-4 * float(np.abs(want).max()) + 1e-12)
        record_parity(f"{tag}/losses", np.array([stats.critic1_loss, stats.critic2_loss]),
                      np.array([ref["critic1_loss"], ref["critic2_loss"]]), rtol=2e-5, atol=1e-5)


# ------------------------------------------------------------------------------------------------------------ host sync
@gpu
@pytest.mark.parametrize("variant", ["mujoco", "bc"])
def test_device_update_has_no_torch_host_sync(variant):
    """The critic steps, the actor step (TD3+BC's lmbda included) and Polyak run under torch.cuda.set_sync_debug_mode("error")."""
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden(f"td3_ref_{variant}.npz")
    algo = _build(_cfg(g), g)
    buf = _buffer(g, mirror=True)
    with policy_within_training_step(algo.policy):
        algo.update(buf, 32)                      # first update: scratch buffers exist afterwards
        for cnt in (0, 1):                        # an actor step, then a critic-only step
            algo._cnt = cnt
            batch, indices = algo._sample(buf, 32)
            batch = algo._preprocess_batch(batch, buf, indices)
            torch.cuda.synchronize()
            torch.cuda.set_sync_debug_mode("error")
            try:
                losses, actor_step = algo._device_update(batch)
            finally:
                torch.cuda.set_sync_debug_mode("default")
            assert actor_step == (cnt == 0) and bool(torch.isfinite(losses[:3 if actor_step else 2]).all())


# ------------------------------------------------------------------------------------------------------------ state_dict
@gpu
@pytest.mark.parametrize("variant", ["mujoco", "bc"])
def test_state_dict_round_trip_continues_identically(variant):
    """A fresh algorithm loaded from another's ``state_dict()`` after two updates (update_actor_freq=2, so both are at the same
    point of the actor schedule) continues bit for bit."""
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden(f"td3_ref_{variant}.npz")
    cfg = _cfg(g)
    a = _build(cfg, g)
    a._noise_fn = _cpu_noise
    buf_a = _buffer(g, mirror=False)
    for u in range(2):
        torch.manual_seed(1 + u)
        with policy_within_training_step(a.policy):
            a.update(buf_a, int(cfg["bs"]))
    b = _build(cfg, g)
    b._noise_fn = _cpu_noise
    with torch.no_grad():
        for p in b.parameters():
            p.add_(0.01)
    b.load_state_dict(copy.deepcopy(a.state_dict()))
    for algo in (a, b):
        buf = _buffer(g, mirror=False)
        for u in range(3):
            torch.manual_seed(10 + u)
            with policy_within_training_step(algo.policy):
                algo.update(buf, int(cfg["bs"]))
    for ga, gb in zip([a._g_actor, *a._g_c, *a._g_ct, a._g_at], [b._g_actor, *b._g_c, *b._g_ct, b._g_at], strict=True):
        assert torch.equal(ga.flat, gb.flat) and torch.equal(ga.exp_avg, gb.exp_avg) and torch.equal(ga.exp_avg_sq, gb.exp_avg_sq)
    for ga, gb in zip([a._g_actor, *a._g_c], [b._g_actor, *b._g_c], strict=True):
        assert ga.step == gb.step


# ------------------------------------------------------------------------------------------------------------ refusals
@gpu
def test_refusals_and_accepted_actors():
    from torch import nn

    from tianshou_b200.algorithm import TD3, TD3BC, AdamOptimizerFactory, UnsupportedModelError
    from tianshou_b200.algorithm.modelfree.ddpg import ContinuousDeterministicPolicy
    from tianshou_b200.utils import policy_within_training_step
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.continuous import ContinuousActorDeterministic, ContinuousCritic
    O, A = 4, 2

    class _Discrete:
        n = 3
        shape = ()

    def make(cls=TD3, dev=DEV, space=None, actor=None, critic=None, m=1.0, last_hidden=(), **kw):
        actor = actor or ContinuousActorDeterministic(preprocess_net=Net(state_shape=(O,), hidden_sizes=(8,)), action_shape=(A,),
                                                      hidden_sizes=last_hidden, max_action=m)
        critic = critic or ContinuousCritic(preprocess_net=Net(state_shape=(O,), action_shape=(A,), hidden_sizes=(8,), concat=True))
        pol = ContinuousDeterministicPolicy(actor=actor.to(dev), action_space=space or _Box(A, m), action_scaling=space is None and m == 1.0,
                                            action_bound_method=None if space is not None else "clip")
        return cls(policy=pol, policy_optim=AdamOptimizerFactory(lr=1e-3), critic=critic.to(dev), critic_optim=AdamOptimizerFactory(lr=1e-3),
                   **kw)

    make()
    with pytest.raises(ValueError, match="Box"):
        make(space=_Discrete())
    with pytest.raises(UnsupportedModelError, match="no CPU path"):
        make(dev="cpu")
    with pytest.raises(UnsupportedModelError, match="no CPU path"):
        make(critic=ContinuousCritic(preprocess_net=Net(state_shape=(O,), action_shape=(A,), hidden_sizes=(8,), concat=True)).cpu(),
             critic2=ContinuousCritic(preprocess_net=Net(state_shape=(O,), action_shape=(A,), hidden_sizes=(8,), concat=True)).cpu())
    with pytest.raises(UnsupportedModelError):
        make(actor=ContinuousActorDeterministic(preprocess_net=Net(state_shape=(O,), hidden_sizes=(8,), norm_layer=nn.LayerNorm),
                                                action_shape=(A,)))
    with pytest.raises(UnsupportedModelError):
        make(critic=ContinuousCritic(preprocess_net=Net(state_shape=(O,), action_shape=(A,), hidden_sizes=(8,), concat=True,
                                                        norm_layer=nn.LayerNorm)))
    with pytest.raises(UnsupportedModelError, match="apply_preprocess_net_to_obs_only"):
        make(critic=ContinuousCritic(preprocess_net=Net(state_shape=(O,), hidden_sizes=(8,)), apply_preprocess_net_to_obs_only=True))
    for cls in (TD3, TD3BC):                      # hidden layers in `last` and any max_action are accepted and train
        for last_hidden, m in (((), 1.0), ((6,), 3.0)):
            algo = make(cls=cls, m=m, last_hidden=last_hidden, update_actor_freq=1)
            buf = _random_buffer(O, A, 40, seed=2, m=m)
            with policy_within_training_step(algo.policy):
                stats = algo.update(buf, 8)
            assert np.isfinite([stats.actor_loss, stats.critic1_loss, stats.critic2_loss]).all()


# ------------------------------------------------------------------------------------------------------------ resources
def test_td3_kernels_have_no_stack_frame_or_spills(tmp_path):
    from tianshou_b200.csrc import build as B
    if shutil.which(B.NVCC) is None and not os.path.exists(B.NVCC):
        pytest.skip("nvcc not available")
    r = subprocess.run([B.NVCC, *B.FLAGS, "-c", os.path.join(B.HERE, "td3.cu"), "-o", str(tmp_path / "t.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    hits = re.findall(r"Compiling entry function '(\S+)' for 'sm_90a'\n(?:.*\n)*?\s*(\d+) bytes stack frame, (\d+) bytes spill "
                      r"stores, (\d+) bytes spill loads", r.stdout + r.stderr)
    names = sorted(re.search(r"td3_(act_rows|target_min|actor_rows|actor_head_bwd)_kernel", h[0]).group(1) for h in hits)
    assert names == ["act_rows", "actor_head_bwd", "actor_rows", "target_min"], hits
    assert all(tuple(map(int, h[1:])) == (0, 0, 0) for h in hits), hits
