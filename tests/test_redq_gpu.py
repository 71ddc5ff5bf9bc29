"""REDQ on the GPU: the batched GEMM (``ts_net_gemm_batched``) against float64 and against ``ts_net_gemm`` bit for bit, the
ensemble layers of ``FusedStack`` against float64 autograd, the redq.cu kernels against float64, ``update()`` against outputs
of the imported reference (tests/golden/redq_ref_*.npz from oracle/gen_golden_redq.py) with the buffer mirror on and off, the
gradient of every optimiser step against float64 autograd of the eager restatement at mujoco_redq.py's width, bit-identical
repeats, the absence of host synchronisation inside the update, ``state_dict()`` round trips, the refusals and the register
report."""
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


# ------------------------------------------------------------------------------------------------------------ batched GEMM
SHAPES = [(1, 1, 1), (127, 128, 129), (129, 300, 128), (300, 127, 300), (128, 129, 127)]
LAYOUTS = [(0, 0), (0, 1), (1, 0), (1, 1)]
MEMBERS = [1, 2, 10, 17]


def _batched(E, M, N, K, a_mn, b_mn, *, share_a, bias, act, mask_kind, accumulate, ws, seed):
    """One ts_net_gemm_batched launch on random operands; returns (result, float64 reference, |A||B| + |bias| bound)."""
    from tianshou_b200._cabi import ABI, call, load_library, ptr
    g = torch.Generator().manual_seed(seed)
    Ea = 1 if share_a else E
    A, B = torch.randn(Ea, M, K, generator=g), torch.randn(E, N, K, generator=g)
    a_st = (A.transpose(1, 2) if a_mn else A).contiguous().to(DEV)
    b_st = (B.transpose(1, 2) if b_mn else B).contiguous().to(DEV)
    C0 = torch.randn(E, M, N, generator=g)
    c = C0.clone().to(DEV)
    bv = torch.randn(E, N, generator=g) if bias else None
    y = torch.tanh(torch.randn(E, M, N, generator=g)) if mask_kind else None
    if y is not None and mask_kind == ABI.consts["TS_ACT_RELU"]:
        y = torch.relu(y)
    ws_n = int(load_library().ts_net_gemm_batched_workspace_floats(E, M, N, K)) if ws else 0
    w = torch.full((max(ws_n, 1),), float("nan"), device=DEV)
    bv_d = bv.to(DEV) if bias else None
    y_d = y.to(DEV) if y is not None else None
    call("ts_net_gemm_batched", E, ptr(a_st), M if a_mn else K, a_mn, 0 if share_a else M * K, ptr(b_st), N if b_mn else K, b_mn,
         N * K, ptr(c), N, M * N, M, N, K, ptr(bv_d), N, act, ptr(y_d), N, M * N, mask_kind or 1, int(accumulate),
         ptr(w) if ws_n else None, ws_n, _st())
    torch.cuda.synchronize()
    ref = torch.matmul(A.double(), B.double().transpose(1, 2)).expand(E, M, N)
    bound = torch.matmul(A.double().abs(), B.double().abs().transpose(1, 2)).expand(E, M, N).clone()
    if bias:
        ref = ref + bv.double()[:, None, :]
        bound = bound + bv.double().abs()[:, None, :]
    if act == 1:
        ref = torch.relu(ref)
    elif act == 2:
        ref = torch.tanh(ref)
    if y is not None:
        yd = y.double()
        ref = ref * (1 - yd * yd) if mask_kind == 2 else ref * (yd > 0)
    if accumulate:
        ref = ref + C0.double()
        bound = bound + C0.double().abs()
    return c.cpu().double(), ref, bound


@gpu
@pytest.mark.parametrize("layout", LAYOUTS, ids=[f"a{a}b{b}" for a, b in LAYOUTS])
@pytest.mark.parametrize("shape", SHAPES, ids=[f"M{s[0]}-N{s[1]}-K{s[2]}" for s in SHAPES])
@pytest.mark.parametrize("E", MEMBERS)
def test_batched_gemm_vs_fp64(E, shape, layout):
    """Every operand arrangement at the tile edges, with and without a shared A, bias, activation, mask, accumulation and a
    split-K workspace (the options rotate with the case so each appears at every member count)."""
    M, N, K = shape
    i = MEMBERS.index(E) * 20 + SHAPES.index(shape) * 4 + LAYOUTS.index(layout)
    opts = dict(share_a=i % 2 == 0, bias=i % 3 != 0, act=i % 3, mask_kind=(0, 1, 2)[(i // 3) % 3], accumulate=i % 4 == 1,
                ws=i % 5 != 0)
    got, ref, bound = _batched(E, M, N, K, *layout, seed=i, **opts)
    tol = 2e-6 * bound + 1e-6
    err = (got - ref).abs()
    assert bool((err <= tol).all()), (opts, float((err / tol).max()))
    record_parity(f"redq_gemm/E{E}_M{M}_N{N}_K{K}_a{layout[0]}b{layout[1]}", got.numpy(), ref.numpy(), rtol=0, atol=float(tol.max()))


@gpu
@pytest.mark.parametrize("ws", [False, True])
def test_batched_gemm_splitk_and_shared_operand(ws):
    """A batch-256 ensemble weight gradient (K = rows) splits when given a workspace and not without one; both agree with float64."""
    from tianshou_b200._cabi import load_library
    assert load_library().ts_net_gemm_batched_workspace_floats(10, 256, 256, 256) > 0
    for E in (1, 10):
        got, ref, bound = _batched(E, 256, 256, 256, 1, 1, share_a=True, bias=False, act=0, mask_kind=0, accumulate=False, ws=ws,
                                   seed=E)
        assert bool(((got - ref).abs() <= 2e-6 * bound + 1e-6).all())


@gpu
@pytest.mark.parametrize("shape", [(256, 256, 256), (300, 129, 1000), (64, 8, 33), (1, 1, 1)])
def test_one_member_batched_gemm_equals_net_gemm_bitwise(shape):
    """ts_net_gemm is the one-member case of ts_net_gemm_batched: same tiles, split choice and reduction order, so the outputs are
    bitwise equal, with every epilogue option."""
    from tianshou_b200._cabi import call, load_library, ptr
    M, N, K = shape
    lib = load_library()
    assert lib.ts_net_gemm_workspace_floats(M, N, K) == lib.ts_net_gemm_batched_workspace_floats(1, M, N, K)
    g = torch.Generator().manual_seed(M + N + K)
    for a_mn, b_mn in LAYOUTS:
        a = torch.randn(M * K, generator=g).to(DEV)
        b = torch.randn(N * K, generator=g).to(DEV)
        bias, y = torch.randn(N, generator=g).to(DEV), torch.relu(torch.randn(M * N, generator=g)).to(DEV)
        c0 = torch.randn(M * N, generator=g).to(DEV)
        ws_n = int(lib.ts_net_gemm_workspace_floats(M, N, K))
        ws = torch.empty(max(ws_n, 1), device=DEV)
        lda, ldb = (M if a_mn else K), (N if b_mn else K)
        c1, c2 = c0.clone(), c0.clone()
        call("ts_net_gemm", ptr(a), lda, a_mn, ptr(b), ldb, b_mn, ptr(c1), N, M, N, K, ptr(bias), 2, ptr(y), N, 1, 1,
             ptr(ws) if ws_n else None, ws_n, _st())
        call("ts_net_gemm_batched", 1, ptr(a), lda, a_mn, 0, ptr(b), ldb, b_mn, 0, ptr(c2), N, 0, M, N, K, ptr(bias), 0, 2, ptr(y),
             N, 0, 1, 1, ptr(ws) if ws_n else None, ws_n, _st())
        torch.cuda.synchronize()
        assert torch.equal(c1, c2), (a_mn, b_mn)


@gpu
def test_batched_colsum_and_member_sum():
    from tianshou_b200._cabi import call, ptr
    g = torch.Generator().manual_seed(5)
    E, M, N = 7, 300, 45
    x = torch.randn(E, M, N, generator=g)
    out = torch.full((E, 1, N), float("nan"), device=DEV)
    xd = x.to(DEV)
    call("ts_net_colsum_batched", E, ptr(xd), N, M * N, M, N, ptr(out), N, 0, _st())
    s = torch.zeros(M, N, device=DEV)
    call("ts_net_member_sum", ptr(xd), E, M * N, M * N, ptr(s), 0, _st())
    torch.cuda.synchronize()
    record_parity("redq_colsum", out.cpu().reshape(E, N).numpy(), x.double().sum(1).numpy(), rtol=1e-5, atol=1e-4)
    ref = x[0].clone()
    for e in range(1, E):
        ref = ref + x[e]
    assert torch.equal(s.cpu(), ref), "the members are summed in index order"


# ------------------------------------------------------------------------------------------------------------ ensemble stack
def _ensemble_critic(O, A, H, E, act=torch.nn.ReLU):
    from tianshou_b200.utils.net.common import EnsembleLinear, Net
    from tianshou_b200.utils.net.continuous import ContinuousCritic
    lin = lambda x, y: EnsembleLinear(E, x, y)
    net_c = Net(state_shape=(O,), action_shape=(A,), hidden_sizes=H, concat=True, linear_layer=lin, activation=act)
    return ContinuousCritic(preprocess_net=net_c, linear_layer=lin, flatten_input=False).to(DEV)


@gpu
@pytest.mark.parametrize("B,E,act", [(1, 3, "relu"), (257, 10, "relu"), (64, 4, "tanh")])
def test_fused_stack_ensemble_vs_fp64_autograd(B, E, act):
    """Forward, the parameter gradients and the input gradient over the action columns summed over the members."""
    from tianshou_b200.algorithm.flat_params import FlatGroup
    from tianshou_b200.algorithm.modelfree.redq import describe_ensemble_critic
    from tianshou_b200.algorithm.netgraph import FusedStack
    O, A, H = 11, 3, (64, 48)
    torch.manual_seed(B + E)
    critic = _ensemble_critic(O, A, H, E, torch.nn.ReLU if act == "relu" else torch.nn.Tanh)
    ref = copy.deepcopy(critic).cpu().double()
    layers, params = describe_ensemble_critic(critic, O, A, E)
    grp = FlatGroup(params, torch.device(DEV))
    stack = FusedStack(layers, grp, "critic")
    x = torch.randn(B, O + A)
    dy = torch.randn(E, B, 1)
    xd = x.to(DEV)
    acts = stack.forward(xd, B, "t")
    dx = torch.full((B, A), float("nan"), device=DEV)
    stack.backward(acts, dy.to(DEV), B, "t", input_grad=True, input_cols=(O, O + A), dx_out=dx)
    torch.cuda.synchronize()
    xr = x.double().requires_grad_(True)
    q = ref.last.model(ref.preprocess.model.model(xr))      # the Sequentials: MLP.forward casts its input to float32
    (q * dy.double()).sum().backward()
    tag = f"redq_stack/B{B}_E{E}_{act}"
    record_parity(f"{tag}/q", acts[-1].cpu().numpy(), q.detach().numpy(), rtol=1e-5, atol=1e-5)
    want = torch.cat([p.grad.reshape(-1) for p in ref.parameters()]).numpy()
    record_parity(f"{tag}/grad", grp.grad[:grp.n].cpu().numpy(), want, rtol=1e-4, atol=1e-5 * float(np.abs(want).max()))
    want_dx = xr.grad[:, O:].numpy()
    record_parity(f"{tag}/dx", dx.cpu().numpy(), want_dx, rtol=1e-4, atol=1e-5 * float(np.abs(want_dx).max()))


@gpu
def test_ensemble_chain_refusals():
    from torch import nn

    from tianshou_b200.algorithm import UnsupportedModelError
    from tianshou_b200.algorithm.modelfree.redq import describe_ensemble_critic
    from tianshou_b200.algorithm.netgraph import FusedStack, compile_sequential
    from tianshou_b200.algorithm.flat_params import FlatGroup
    from tianshou_b200.utils.net.common import EnsembleLinear
    with pytest.raises(UnsupportedModelError, match="mixes"):
        compile_sequential([EnsembleLinear(3, 4, 8), nn.ReLU(), nn.Linear(8, 1)], (4,), ensemble=True)
    with pytest.raises(UnsupportedModelError, match="different ensemble sizes"):
        compile_sequential([EnsembleLinear(3, 4, 8), nn.ReLU(), EnsembleLinear(4, 8, 1)], (4,), ensemble=True)
    with pytest.raises(UnsupportedModelError, match="bias"):
        compile_sequential([EnsembleLinear(3, 4, 8, bias=False)], (4,), ensemble=True)
    with pytest.raises(UnsupportedModelError, match="outside"):        # the twin-critic algorithms do not read ensembles
        compile_sequential([EnsembleLinear(3, 4, 8)], (4,))
    with pytest.raises(UnsupportedModelError, match="ensemble_size"):
        describe_ensemble_critic(_ensemble_critic(3, 1, (8,), 4), 3, 1, 5)
    layers = compile_sequential([EnsembleLinear(3, 4, 8).to(DEV), nn.ReLU(), EnsembleLinear(3, 8, 1).to(DEV)], (4,), ensemble=True)
    from tianshou_b200.algorithm.netgraph import layer_params
    stack = FusedStack(layers, FlatGroup(layer_params(layers), torch.device(DEV)))
    x = torch.randn(2, 4, device=DEV)
    acts = stack.forward(x, 2)
    with pytest.raises(UnsupportedModelError, match="ensemble"):
        stack.jvp(acts, stack.group.flat, 2)


# ------------------------------------------------------------------------------------------------------------ loss kernels
@gpu
@pytest.mark.parametrize("B", [1, 255, 256, 257, 300000])
@pytest.mark.parametrize("mode", ["min", "mean"])
def test_redq_kernels_vs_fp64(B, mode):
    from tianshou_b200._cabi import ABI, call, ptr
    E = 10
    g = torch.Generator().manual_seed(B)
    q, target, w, logp = (torch.randn(E, B, generator=g) * 3, torch.randn(B, generator=g), torch.rand(B, generator=g) + 0.1,
                          torch.randn(B, generator=g))
    subset = [7, 2, 4]
    mask = sum(1 << e for e in subset)
    alpha = 0.3
    q_d, t_d, w_d, lp_d = (t.to(DEV).contiguous() for t in (q, target, w, logp))     # held: the launches are asynchronous
    d = {id(q): q_d, id(target): t_d, id(w): w_d, id(logp): lp_d}.get
    d = (lambda f: lambda t: f(id(t)))(d)
    out = torch.full((B,), float("nan"), device=DEV)
    code = ABI.consts["TS_REDQ_MIN" if mode == "min" else "TS_REDQ_MEAN"]
    call("ts_redq_target", ptr(d(q)), E, B, mask, code, alpha, ptr(d(logp)), ptr(out), _st())
    td, dq = torch.full((E, B), float("nan"), device=DEV), torch.full((E, B), float("nan"), device=DEV)
    rmean, rows, loss = torch.empty(B, device=DEV), torch.empty(B, device=DEV), torch.full((1,), float("nan"), device=DEV)
    call("ts_redq_critic_rows", ptr(d(q)), ptr(d(target)), ptr(d(w)), E, B, ptr(td), ptr(dq), ptr(rmean), ptr(rows), ptr(loss), _st())
    adq, arows, aloss = torch.full((E, B), float("nan"), device=DEV), torch.empty(B, device=DEV), torch.full((1,), float("nan"), device=DEV)
    call("ts_redq_actor_rows", ptr(d(q)), ptr(d(logp)), E, B, alpha, ptr(adq), ptr(arows), ptr(aloss), _st())
    torch.cuda.synchronize()
    qd = q.double()
    sub = qd[subset]
    want = (sub.min(0)[0] if mode == "min" else sub.mean(0)) - np.float32(alpha) * logp.double()
    tag = f"redq_kernels/B{B}_{mode}"
    record_parity(f"{tag}/target", out.cpu().numpy(), want.numpy(), rtol=2e-6, atol=2e-6)
    qq = qd.clone().requires_grad_(True)
    tdr = qq - target.double()
    lref = (tdr.pow(2) * w.double()).mean()
    lref.backward()
    record_parity(f"{tag}/td", td.cpu().numpy(), tdr.detach().numpy(), rtol=1e-6, atol=1e-6)
    record_parity(f"{tag}/critic_loss", loss.cpu().numpy(), np.array([lref.item()]), rtol=1e-5, atol=1e-7)
    record_parity(f"{tag}/dq", dq.cpu().numpy(), qq.grad.numpy(), rtol=1e-5, atol=1e-12)
    record_parity(f"{tag}/row_mean", rmean.cpu().numpy(), tdr.detach().mean(0).numpy(), rtol=1e-5, atol=1e-6)
    qa = qd.clone().requires_grad_(True)
    aref = (alpha * logp.double() - qa.mean(0)).mean()
    aref.backward()
    record_parity(f"{tag}/actor_loss", aloss.cpu().numpy(), np.array([aref.item()]), rtol=1e-5, atol=1e-6)
    record_parity(f"{tag}/actor_dq", adq.cpu().numpy(), qa.grad.numpy(), rtol=1e-6, atol=0)
    again = torch.empty(1, device=DEV)
    call("ts_redq_critic_rows", ptr(d(q)), ptr(d(target)), ptr(d(w)), E, B, ptr(td), ptr(dq), ptr(rmean), ptr(rows), ptr(again), _st())
    torch.cuda.synchronize()
    assert torch.equal(again, loss)


@gpu
def test_redq_target_refuses_bad_masks():
    from tianshou_b200._cabi import call, ptr
    q, logp, out = torch.zeros(3, 4, device=DEV), torch.zeros(4, device=DEV), torch.zeros(4, device=DEV)
    for E, mask in ((65, 1), (3, 0), (3, 8)):
        with pytest.raises(RuntimeError):
            call("ts_redq_target", ptr(q), E, 4, mask, 0, 0.1, ptr(logp), ptr(out), _st())


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


def _build(cfg, g=None, **over):
    from tianshou_b200.algorithm import REDQ, AdamOptimizerFactory, REDQPolicy
    from tianshou_b200.algorithm.modelfree.sac import AutoAlpha
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.continuous import ContinuousActorProbabilistic
    O, A, H, E = int(cfg["obs"]), int(cfg["act"]), tuple(int(x) for x in cfg["hidden"]), int(cfg["E"])
    actor = ContinuousActorProbabilistic(preprocess_net=Net(state_shape=(O,), hidden_sizes=H), action_shape=(A,), unbounded=True,
                                         conditioned_sigma=True).to(DEV)
    critic = _ensemble_critic(O, A, H, E)
    if g is not None:
        _load(actor, g, "p0_actor_"); _load(critic, g, "p0_critic_")
    alpha = (AutoAlpha(-A, 0.0, AdamOptimizerFactory(lr=float(cfg["alpha_lr"]))).to(DEV) if bool(cfg["auto_alpha"])
             else float(cfg["alpha"]))
    policy = REDQPolicy(actor=actor, action_space=_Box(A))
    kw = dict(policy=policy, policy_optim=AdamOptimizerFactory(lr=float(cfg["actor_lr"])), critic=critic,
              critic_optim=AdamOptimizerFactory(lr=float(cfg["critic_lr"])), ensemble_size=E, subset_size=int(cfg["M"]),
              tau=float(cfg["tau"]), gamma=float(cfg["gamma"]), alpha=alpha, n_step_return_horizon=int(cfg["n_step"]),
              actor_delay=int(cfg["delay"]), target_mode=str(cfg["target_mode"]))
    kw.update(over)
    return REDQ(**kw)


def _buffer(g, mirror):
    from tianshou_b200.data import Batch, PrioritizedReplayBuffer, ReplayBuffer
    cfg = _cfg(g)
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
    """The reference ran on the CPU: Normal.rsample's draw on the CPU generator, uploaded."""
    return torch.empty(shape).normal_().to(DEV)


class _SubsetSpy:
    """Records the subset REDQ draws with numpy's own ``np.random.choice`` (the stream is untouched)."""

    def __init__(self, monkeypatch):
        self.seen = []
        orig = np.random.choice

        def choice(*args, **kwargs):
            r = orig(*args, **kwargs)
            if kwargs.get("replace", True) is False:
                self.seen.append(np.asarray(r).copy())
            return r

        monkeypatch.setattr(np.random, "choice", choice)


@gpu
@pytest.mark.parametrize("mirror", [False, True])
@pytest.mark.parametrize("variant", ["mujoco", "per_mean", "full"])
def test_update_matches_reference(variant, mirror, monkeypatch):
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden(f"redq_ref_{variant}.npz")
    cfg = _cfg(g)
    algo = _build(cfg, g)
    assert sorted(algo.state_dict().keys()) == list(g["state_dict_keys"]), "state_dict() keys differ from the reference's"
    buf = _buffer(g, mirror)
    algo._noise_fn = _cpu_noise
    spy = _SubsetSpy(monkeypatch)
    captured = {}
    orig = algo._preprocess_batch

    def hook(batch, buffer, indices):
        captured["indices"] = np.asarray(indices).copy()
        if bool(cfg["per"]):
            captured["is_weight"] = batch.weight.detach().cpu().numpy().copy()
        return orig(batch, buffer, indices)

    algo._preprocess_batch = hook
    lr, a_lr = float(cfg["critic_lr"]), float(cfg["actor_lr"])
    delay = int(cfg["delay"])
    for u in range(int(cfg["updates"])):
        np.random.seed(500 + u)
        torch.manual_seed(100 + u)
        actor_before = algo._g_actor.flat.clone()
        with policy_within_training_step(algo.policy):
            stats = algo.update(buf, int(cfg["bs"]))
        o, tag = f"u{u}_", f"redq/{variant}_m{int(mirror)}_u{u}"
        assert np.array_equal(captured["indices"], g[o + "indices"]), "sampled indices differ from the reference's"
        assert np.array_equal(spy.seen[-1], g[o + "subset"]), "the ensemble subset differs from the reference's"
        record_parity(f"{tag}/losses", np.array([stats.actor_loss, stats.critic_loss]), g[o + "losses"], rtol=2e-5, atol=2e-6)
        record_parity(f"{tag}/alpha", np.array([stats.alpha]), np.array([g[o + "alpha"]]), rtol=1e-5, atol=0)
        assert (stats.alpha_loss is None) == bool(np.isnan(g[o + "alpha_loss"]))
        assert torch.equal(actor_before, algo._g_actor.flat) == ((u + 1) % delay != 0), "the actor steps on delay multiples only"
        if bool(cfg["per"]):
            record_parity(f"{tag}/is_weight", captured["is_weight"], g[o + "is_weight"], rtol=1e-6, atol=1e-7)
            record_parity(f"{tag}/priorities", np.asarray(buf.weight[np.arange(len(buf))]), g[o + "priorities"], rtol=1e-3, atol=1e-6)
        _check_params(tag, algo.policy.actor, g, o + "actor_", a_lr)
        _check_params(tag, algo.critic, g, o + "critic_", lr)
        _check_params(tag, algo.critic_old, g, o + "cold_", lr)
    assert algo.critic_gradient_step == int(cfg["updates"])


# ------------------------------------------------------------------------------------------------------------ gradients
class _Recorder(torch.optim.Adam):
    """Adam that keeps the gradient it is about to apply."""

    def step(self, closure=None):
        self.seen = [p.grad.detach().clone() for g in self.param_groups for p in g["params"]]
        return super().step(closure)


def _random_buffer(O, A, n, seed):
    from tianshou_b200.data import ReplayBuffer
    rng = np.random.default_rng(seed)
    term = rng.random(n) < 0.05
    term[[0, -1]] = True
    trunc = (rng.random(n) < 0.03) & ~term
    return ReplayBuffer.from_data(rng.standard_normal((n, O)).astype(np.float32), np.tanh(rng.standard_normal((n, A))).astype(np.float32),
                                  rng.standard_normal(n), term, trunc, term | trunc, rng.standard_normal((n, O)).astype(np.float32))


@gpu
@pytest.mark.parametrize("mode", ["min", "mean"])
def test_update_gradients_vs_fp64_autograd(mode, monkeypatch):
    """mujoco_redq.py's width (Ant-v4's 27 observations and 8 actions, hidden [256, 256], E 10, subset 2, batch 256), n = 3: an
    actor step, then a critic-only step.  The ensemble step's gradient, taken before its Adam step, against float64 autograd of the
    eager restatement on copies of the modules with the same batch, noise and subset; the actor step's against float64 autograd
    of the actor loss on the pre-update actor and the ensemble the update stepped."""
    from oracle.oracle_redq import FixedAlpha, RedqNets, actor_objective, redq_update
    from tianshou_b200.algorithm.flat_params import FlatGroup
    from tianshou_b200.utils import policy_within_training_step
    O, A, H, E, B = 27, 8, (256, 256), 10, 256
    cfg = dict(obs=O, act=A, hidden=H, E=E, M=2, delay=2, actor_lr=3e-4, critic_lr=3e-4, tau=0.005, gamma=0.99, n_step=3,
               alpha=0.2, auto_alpha=False, target_mode=mode)
    torch.manual_seed(3)
    algo = _build(cfg)
    algo.critic_gradient_step = 1                 # the first update is an actor step
    buf = _random_buffer(O, A, 900, seed=11)
    spy = _SubsetSpy(monkeypatch)
    noises = []

    def noise(shape):
        noises.append(torch.randn(shape, device=DEV))
        return noises[-1]

    algo._noise_fn = noise
    # the gradient in the modules' parameter order (the actor's flat buffer keeps mu / sigma weights adjacent)
    names = {id(algo._g_actor): ("actor", algo.policy.actor), id(algo._g_c): ("critic", algo.critic)}
    cap = {}

    def adam(group, optimizer, mgn):
        name, mod = names[id(group)]
        cap[name] = torch.cat([group.view(group.grad, p).reshape(-1) for p in mod.parameters()]).detach().cpu().double()
        FlatGroup.adam_step(group, optimizer, mgn)

    algo._adam = adam
    orig = algo._preprocess_batch
    algo._preprocess_batch = lambda b, buffer, idx: (cap.update(indices=np.asarray(idx).copy()), orig(b, buffer, idx))[1]
    d = {k: np.asarray(buf._meta[k]) for k in ("obs", "act", "rew", "done", "terminated", "obs_next")}
    d.update(offset=np.array([0, len(buf)]), last_index=np.asarray(buf.last_index), lengths=np.array([len(buf)]),
             unfinished=[] if d["done"][len(buf) - 1] else [len(buf) - 1])
    for u, actor_step in enumerate((True, False)):
        nets = RedqNets(O, A, H, E)
        with torch.no_grad():
            for dst, src in ((nets.actor, algo.policy.actor), (nets.critic, algo.critic), (nets.critic_old, algo.critic_old)):
                for p, q in zip(dst.parameters(), src.parameters(), strict=True):
                    p.copy_(q.detach().cpu())
        for mod in nets.modules():
            mod.double()
        actor_before = [p.detach().clone() for p in algo.policy.actor.parameters()]
        cap.clear(); noises.clear()
        with policy_within_training_step(algo.policy):
            stats = algo.update(buf, B)
        torch.cuda.synchronize()
        tag = f"redq_grad/{mode}_u{u}"
        assert set(cap) == ({"indices", "actor", "critic"} if actor_step else {"indices", "critic"})
        if actor_step:
            anets = RedqNets(O, A, H, E)
            with torch.no_grad():
                for p, q in zip(anets.actor.parameters(), actor_before, strict=True):
                    p.copy_(q.cpu())
                for p, q in zip(anets.critic.parameters(), algo.critic.parameters(), strict=True):
                    p.copy_(q.detach().cpu())
            anets.actor.double(); anets.critic.double()
            obs = torch.as_tensor(d["obs"][cap["indices"]]).double()
            loss, _ = actor_objective(anets, obs, noises[1].double().cpu(), 0.2)
            grads = torch.autograd.grad(loss, list(anets.actor.parameters()))
            want = torch.cat([x.reshape(-1) for x in grads]).numpy()
            record_parity(f"{tag}/grad_actor", cap["actor"].numpy(), want, rtol=2e-4, atol=1e-4 * float(np.abs(want).max()) + 1e-12)
            record_parity(f"{tag}/actor_loss", np.array([stats.actor_loss]), np.array([loss.item()]), rtol=2e-5, atol=1e-5)
        it = iter(noises)
        opts = [_Recorder(nets.actor.parameters(), lr=3e-4), _Recorder(nets.critic.parameters(), lr=3e-4)]
        ref = redq_update(nets, opts, FixedAlpha(0.2), d, cap["indices"], lambda shape: next(it).double().cpu(), spy.seen[-1],
                          gamma=0.99, n_step=3, tau=0.005, target_mode=mode, actor_step=False)
        want = torch.cat([x.reshape(-1) for x in opts[1].seen]).numpy()
        record_parity(f"{tag}/grad_critic", cap["critic"].numpy(), want, rtol=2e-4, atol=1e-4 * float(np.abs(want).max()) + 1e-12)
        record_parity(f"{tag}/critic_loss", np.array([stats.critic_loss]), np.array([ref["critic_loss"]]), rtol=2e-5, atol=1e-5)
        assert len(cap["indices"]) == B and all(x.shape[0] == B for x in noises)


# ------------------------------------------------------------------------------------------------------------ determinism, sync, state
@gpu
def test_identical_updates_are_bit_identical():
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden("redq_ref_mujoco.npz")
    cfg = _cfg(g)
    flats = []
    for _ in range(2):
        algo = _build(cfg, g)
        algo._noise_fn = _cpu_noise
        buf = _buffer(g, mirror=True)
        for u in range(4):
            np.random.seed(500 + u)
            torch.manual_seed(100 + u)
            with policy_within_training_step(algo.policy):
                algo.update(buf, int(cfg["bs"]))
        flats.append([t.flat.clone() for t in (algo._g_actor, algo._g_c, algo._g_ct)])
    assert all(torch.equal(a, b) for a, b in zip(*flats, strict=True))


@gpu
def test_device_update_has_no_torch_host_sync():
    """With a fixed alpha the ensemble step, the actor step and Polyak run under torch.cuda.set_sync_debug_mode("error"); the
    losses are read at the end."""
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden("redq_ref_mujoco.npz")
    algo = _build(_cfg(g), g)
    buf = _buffer(g, mirror=True)
    seen = []
    orig_cpu = torch.Tensor.cpu
    with policy_within_training_step(algo.policy):
        algo.update(buf, 32)
        for step in (2, 0):                       # critic_gradient_step -> 3 (an actor step), then -> 1 (critic only)
            algo.critic_gradient_step = step
            batch, indices = algo._sample(buf, 32)
            batch = algo._preprocess_batch(batch, buf, indices)
            torch.cuda.synchronize()

            def cpu(t, *a, **k):                  # the final read of the losses is allowed: it happens outside the checked span
                torch.cuda.set_sync_debug_mode("default")
                seen.append(tuple(t.shape))
                return orig_cpu(t, *a, **k)

            torch.Tensor.cpu = cpu
            torch.cuda.set_sync_debug_mode("error")
            try:
                stats = algo._update_with_batch(batch)
            finally:
                torch.cuda.set_sync_debug_mode("default")
                torch.Tensor.cpu = orig_cpu
            assert np.isfinite(stats.critic_loss) and stats.alpha_loss is None
    assert seen == [(2,), (1,)], seen


@gpu
def test_state_dict_round_trip_continues_identically():
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden("redq_ref_mujoco.npz")        # actor_delay 3: the continuation takes an actor step
    cfg = _cfg(g)
    a = _build(cfg, g)
    a._noise_fn = _cpu_noise
    buf_a = _buffer(g, mirror=False)
    for u in range(2):
        torch.manual_seed(1 + u)
        np.random.seed(1 + u)
        with policy_within_training_step(a.policy):
            a.update(buf_a, int(cfg["bs"]))
    b = _build(cfg, g)
    b._noise_fn = _cpu_noise
    with torch.no_grad():
        for p in b.parameters():
            p.add_(0.01)
    b.load_state_dict(copy.deepcopy(a.state_dict()))
    b.critic_gradient_step = a.critic_gradient_step
    for algo in (a, b):
        buf = _buffer(g, mirror=False)
        for u in range(3):
            torch.manual_seed(10 + u)
            np.random.seed(10 + u)
            with policy_within_training_step(algo.policy):
                algo.update(buf, int(cfg["bs"]))
    for ga, gb in zip([a._g_actor, a._g_c, a._g_ct], [b._g_actor, b._g_c, b._g_ct], strict=True):
        assert torch.equal(ga.flat, gb.flat) and torch.equal(ga.exp_avg, gb.exp_avg) and torch.equal(ga.exp_avg_sq, gb.exp_avg_sq)


# ------------------------------------------------------------------------------------------------------------ refusals
@gpu
def test_refusals():
    from tianshou_b200.algorithm import REDQ, AdamOptimizerFactory, REDQPolicy, UnsupportedModelError
    from tianshou_b200.utils.net.common import EnsembleLinear, Net
    from tianshou_b200.utils.net.continuous import ContinuousActorProbabilistic, ContinuousCritic
    O, A, E = 4, 2, 3

    def make(dev=DEV, critic=None, unbounded=True, c_sigma=True, **kw):
        actor = ContinuousActorProbabilistic(preprocess_net=Net(state_shape=(O,), hidden_sizes=(8,)), action_shape=(A,),
                                             unbounded=unbounded, conditioned_sigma=c_sigma).to(dev)
        critic = critic if critic is not None else _ensemble_critic(O, A, (8,), E).to(dev)
        return REDQ(policy=REDQPolicy(actor=actor, action_space=_Box(A)), policy_optim=AdamOptimizerFactory(lr=1e-3), critic=critic,
                    critic_optim=AdamOptimizerFactory(lr=1e-3), ensemble_size=kw.pop("ensemble_size", E), subset_size=2, **kw)

    make()
    with pytest.raises(UnsupportedModelError, match="no CPU path"):
        make(dev="cpu")
    with pytest.raises(UnsupportedModelError, match="unbounded"):
        make(unbounded=False)
    with pytest.raises(UnsupportedModelError, match="conditioned_sigma"):
        make(c_sigma=False)
    lin = lambda x, y: EnsembleLinear(E, x, y)
    mixed = ContinuousCritic(preprocess_net=Net(state_shape=(O,), action_shape=(A,), hidden_sizes=(8,), concat=True),
                             linear_layer=lin, flatten_input=False).to(DEV)
    with pytest.raises(UnsupportedModelError):
        make(critic=mixed)
    mismatched = ContinuousCritic(preprocess_net=Net(state_shape=(O,), action_shape=(A,), hidden_sizes=(8,), concat=True,
                                                     linear_layer=lin), linear_layer=lambda x, y: EnsembleLinear(E + 1, x, y),
                                  flatten_input=False).to(DEV)
    with pytest.raises(UnsupportedModelError, match="different ensemble sizes"):
        make(critic=mismatched)
    with pytest.raises(UnsupportedModelError, match="ensemble_size"):
        make(ensemble_size=E + 1)
    obs_only = ContinuousCritic(preprocess_net=Net(state_shape=(O,), hidden_sizes=(8,), linear_layer=lin), linear_layer=lin,
                                flatten_input=False, apply_preprocess_net_to_obs_only=True).to(DEV)
    with pytest.raises(UnsupportedModelError, match="apply_preprocess_net_to_obs_only"):
        make(critic=obs_only)


# ------------------------------------------------------------------------------------------------------------ resources
def _ptxas(src, tmp_path):
    from tianshou_b200.csrc import build as B
    if shutil.which(B.NVCC) is None and not os.path.exists(B.NVCC):
        pytest.skip("nvcc not available")
    r = subprocess.run([B.NVCC, *B.FLAGS, "-c", os.path.join(B.HERE, src), "-o", str(tmp_path / "t.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    return re.findall(r"Compiling entry function '(\S+)' for 'sm_90a'\n(?:.*\n)*?\s*(\d+) bytes stack frame, (\d+) bytes spill "
                      r"stores, (\d+) bytes spill loads", r.stdout + r.stderr)


def test_redq_kernels_have_no_stack_frame_or_spills(tmp_path):
    hits = _ptxas("redq.cu", tmp_path)
    names = sorted(re.search(r"redq_(target|critic_rows|actor_rows|sum)_kernel", h[0]).group(1) for h in hits)
    assert names == ["actor_rows", "critic_rows", "sum", "target"], hits
    assert all(tuple(map(int, h[1:])) == (0, 0, 0) for h in hits), hits


def test_net_gemm_kernels_have_no_stack_frame_or_spills(tmp_path):
    hits = _ptxas("net_gemm.cu", tmp_path)
    gemm = [h for h in hits if "net_gemm_kernel" in h[0]]
    assert len(gemm) == 4 and len(hits) == 7, hits
    assert all(tuple(map(int, h[1:])) == (0, 0, 0) for h in hits), hits
