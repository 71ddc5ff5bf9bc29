"""CQL on the GPU: ``ts_cql_rows`` / ``ts_cql_losses`` / ``ts_cql_target`` against float64 autograd, ``CQL.update()`` against
outputs of the imported reference (tests/golden/cql_ref_*.npz from oracle/gen_golden_cql.py) with the buffer mirror on and off,
the gradients of the actor, both critics and the Lagrange multiplier against float64 autograd of the eager restatement, the
absence of host synchronisation inside the update, ``state_dict()`` round trips, the refusals and the kernels' register report."""
import copy
import re

import numpy as np
import pytest
import torch

from offpolicy_testutil import DEV, Box, assert_spill_free, check_params, golden_cfg, load_params, ptxas_report, stream
from ts_testutil import load_golden, record_parity, set_buffer_state

gpu = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------------------ kernels
def _kernels(q1, q2, y, B, R, lp_c, lp_x, rand_logp, cal, T, w, log_alpha, amin, amax, thr):
    from tianshou_b200._cabi import call, ptr
    N = B * R
    dq1, dq2 = torch.empty(B + 3 * N, device=DEV), torch.empty(B + 3 * N, device=DEV)
    sq, lse = torch.empty(2 * B, device=DEV), torch.empty(2 * N, device=DEV)
    grad, out = torch.full((1,), float("nan"), device=DEV), torch.full((4,), float("nan"), device=DEV)
    st = stream()
    call("ts_cql_rows", ptr(q1), ptr(q2), ptr(y), B, R, ptr(lp_c), ptr(lp_x), rand_logp, ptr(cal), T, w, ptr(log_alpha), amin, amax,
         ptr(dq1), ptr(dq2), ptr(sq), ptr(lse), st)
    call("ts_cql_losses", ptr(q1), ptr(q2), ptr(sq), ptr(lse), B, N, T, w, ptr(log_alpha), amin, amax, thr,
         ptr(grad) if log_alpha is not None else None, ptr(out), st)
    torch.cuda.synchronize()
    return dq1, dq2, lse, grad, out


def _fp64(q1, q2, y, B, R, lp_c, lp_x, rand_logp, cal, T, w, log_alpha, amin, amax, thr):
    """cql.py:295-381 in float64 autograd on the same values."""
    N = B * R
    q = [t.detach().cpu().double().requires_grad_(True) for t in (q1, q2)]
    la = None if log_alpha is None else log_alpha.detach().cpu().double().requires_grad_(True)
    yy, lc, lx = (t.detach().cpu().double() for t in (y, lp_c, lp_x))
    ret = None if cal is None else cal.detach().cpu().double().unsqueeze(1).repeat(1, R).view(-1, 1)
    losses, lses = [], []
    a = None if la is None else torch.clamp(la.exp(), amin, amax)
    for k in range(2):
        d, blk = q[k][:B], q[k][B:].view(3, N, 1)
        vals = [blk[0] - np.float32(rand_logp), blk[1] - lc.view(-1, 1), blk[2] - lx.view(-1, 1)]
        if ret is not None:
            vals = [torch.max(v, ret) for v in vals]
        lse = torch.logsumexp(torch.cat(vals, 1) / T, dim=1)
        lses.append(lse)
        pen = lse.mean() * w * T - d.mean() * w
        if a is not None:
            pen = a * (pen - thr)
        losses.append(((d - yy) ** 2).mean() + pen)
    (losses[0] + losses[1]).backward()
    g_la = None
    if la is not None:
        la2 = log_alpha.detach().cpu().double().requires_grad_(True)
        a2 = torch.clamp(la2.exp(), amin, amax)
        pens = [lses[k].detach().mean() * w * T - q[k].detach()[:B].mean() * w for k in range(2)]
        aloss = -(a2 * (pens[0] - thr) + a2 * (pens[1] - thr)) * 0.5
        aloss.backward()
        g_la = la2.grad
        return q[0].grad, q[1].grad, torch.cat(lses).detach(), g_la, [l.item() for l in losses] + [a2.item(), aloss.item()]
    return q[0].grad, q[1].grad, torch.cat(lses).detach(), g_la, [l.item() for l in losses]


KERNEL_CASES = [
    # (B, R, A, T, calibrated, lagrange, kind)
    (64, 1, 1, 1.0, True, True, "plain"),
    (32, 10, 6, 0.5, True, True, "ties"),
    (16, 33, 17, 3.0, False, False, "plain"),
    (40, 10, 6, 1.0, True, False, "spread"),
    (48, 10, 3, 1.0, True, True, "clamped"),
    (20000, 33, 6, 1.0, True, True, "past_grid_cap"),
]


@gpu
@pytest.mark.parametrize("B,R,A,T,calibrated,lagrange,kind", KERNEL_CASES, ids=[f"B{c[0]}-R{c[1]}-A{c[2]}-T{c[3]}-{c[6]}" for c in KERNEL_CASES])
def test_rows_and_losses_kernels_vs_fp64(B, R, A, T, calibrated, lagrange, kind):
    g = torch.Generator().manual_seed(B + R + A)
    N = B * R
    q1, q2 = (torch.randn(B + 3 * N, generator=g) * 3 for _ in range(2))
    if kind == "spread":              # values 1e4 apart inside one row: the shifted log-sum-exp must stay finite
        q1[B:B + N] += 1e4
        q2[B + 2 * N:] -= 1e4
    y = torch.randn(B, generator=g)
    lp_c, lp_x = torch.randn(N, generator=g), torch.randn(N, generator=g)
    rand_logp = float(np.log(0.5 ** A))
    cal = torch.randn(B, generator=g) if calibrated else None
    if kind == "ties":                # exact ties between a block value and its calibration return: half the gradient
        lp_c[: N // 2] = 0.0
        q1[B + N: B + N + N // 2] = cal.repeat_interleave(R)[: N // 2]
        q2[B + N: B + N + N // 2] = cal.repeat_interleave(R)[: N // 2]
    log_alpha = torch.tensor([0.3 if kind != "clamped" else 2.0]) if lagrange else None
    amin, amax, thr, w = 0.0, (1e6 if kind != "clamped" else 2.0), 5.0, 1.7
    dev = lambda t: None if t is None else t.to(DEV).contiguous()
    args = (dev(q1), dev(q2), dev(y), B, R, dev(lp_c), dev(lp_x), rand_logp, dev(cal), T, w, dev(log_alpha), amin, amax, thr)
    dq1, dq2, lse, grad, out = _kernels(*args)
    r1, r2, rlse, rga, rl = _fp64(q1, q2, y, B, R, lp_c, lp_x, rand_logp, cal, T, w, log_alpha, amin, amax, thr)
    tag = f"cql_rows/B{B}_R{R}_A{A}_{kind}"
    scale = lambda r: 1e-6 * float(r.abs().max())
    record_parity(f"{tag}/dq1", dq1.cpu().numpy(), r1.numpy(), rtol=1e-5, atol=scale(r1))
    record_parity(f"{tag}/dq2", dq2.cpu().numpy(), r2.numpy(), rtol=1e-5, atol=scale(r2))
    record_parity(f"{tag}/lse", lse.cpu().numpy(), rlse.numpy(), rtol=1e-6, atol=1e-6)
    n = 4 if lagrange else 2
    record_parity(f"{tag}/losses", out[:n].cpu().numpy(), np.array(rl[:n]), rtol=1e-5, atol=1e-6)
    if lagrange:
        record_parity(f"{tag}/grad_log_alpha", grad.cpu().numpy(), rga.numpy(), rtol=1e-5, atol=1e-7)
        if kind == "clamped":
            assert grad.item() == 0.0 and out[2].item() == 2.0
    if kind == "ties":
        assert int((r1[B + N: B + N + N // 2] != 0).sum()) > 0
    again = _kernels(*args)           # fixed-order reductions: bit-identical from run to run
    for a, b in zip((dq1, dq2, lse, out), (again[0], again[1], again[2], again[4]), strict=True):
        assert torch.equal(a.nan_to_num(-7.0), b.nan_to_num(-7.0))


@gpu
@pytest.mark.parametrize("B", [5, 300000])
def test_target_kernel_vs_fp32_reference_order(B):
    from tianshou_b200._cabi import call, ptr
    g = torch.Generator().manual_seed(B)
    q1, q2, lp, rew = (torch.randn(B, generator=g) for _ in range(4))
    done = (torch.rand(B, generator=g) < 0.3).float()
    alpha, gamma = 0.2, 0.99
    out = torch.empty(B, device=DEV)
    d = [t.to(DEV) for t in (q1, q2, lp, rew, done)]          # kept alive until the kernel has run
    call("ts_cql_target", ptr(d[0]), ptr(d[1]), ptr(d[2]), alpha, ptr(d[3]), ptr(d[4]), gamma, B, ptr(out), stream())
    torch.cuda.synchronize()
    ref = rew.double() + (1.0 - done.double()) * np.float64(np.float32(gamma)) * (torch.min(q1, q2).double() - np.float32(alpha) * lp.double())
    record_parity(f"cql_target/B{B}", out.cpu().numpy(), ref.numpy(), rtol=1e-6, atol=1e-6)
    assert bool((out.cpu()[done > 0] == rew[done > 0]).all()), "done rows carry the reward alone"


# ------------------------------------------------------------------------------------------------------------ goldens
def build_from_cfg(cfg, g=None, **over):
    from tianshou_b200.algorithm import CQL, AdamOptimizerFactory
    from tianshou_b200.algorithm.modelfree.sac import AutoAlpha, SACPolicy
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.continuous import ContinuousActorProbabilistic, ContinuousCritic
    O, A, H = int(cfg["obs"]), int(cfg["act"]), tuple(int(x) for x in cfg["hidden"])
    actor = ContinuousActorProbabilistic(preprocess_net=Net(state_shape=(O,), hidden_sizes=H), action_shape=(A,), unbounded=True,
                                         conditioned_sigma=True).to(DEV)
    crit = lambda: ContinuousCritic(preprocess_net=Net(state_shape=(O,), action_shape=(A,), hidden_sizes=H, concat=True)).to(DEV)
    c1 = crit()
    c2 = crit() if bool(cfg["critic2"]) else None
    if g is not None:
        load_params(actor, g, "p0_actor_"); load_params(c1, g, "p0_c1_")
        if c2 is not None:
            load_params(c2, g, "p0_c2_")
    alpha = AutoAlpha(-float(A), 0.0, AdamOptimizerFactory(lr=float(cfg["alpha_lr"]))).to(DEV) if bool(cfg["auto"]) else float(cfg["alpha"])
    kw = dict(cql_alpha_lr=float(cfg["cql_alpha_lr"]), cql_weight=float(cfg["cql_weight"]), tau=float(cfg["tau"]), gamma=float(cfg["gamma"]),
              alpha=alpha, temperature=float(cfg["temperature"]), with_lagrange=bool(cfg["with_lagrange"]),
              lagrange_threshold=float(cfg["lagrange_threshold"]), min_action=float(cfg["min_action"]), max_action=float(cfg["max_action"]),
              num_repeat_actions=int(cfg["R"]), alpha_min=float(cfg["alpha_min"]), alpha_max=float(cfg["alpha_max"]),
              max_grad_norm=float(cfg["max_grad_norm"]), calibrated=bool(cfg["calibrated"]))
    kw.update(over)
    return CQL(policy=SACPolicy(actor=actor, action_space=Box(A)), policy_optim=AdamOptimizerFactory(lr=float(cfg["actor_lr"])),
               critic=c1, critic_optim=AdamOptimizerFactory(lr=float(cfg["critic_lr"])), critic2=c2,
               critic2_optim=AdamOptimizerFactory(lr=float(cfg["critic2_lr"])) if c2 is not None else None, **kw)


def buffer_from_golden(g, mirror):
    from tianshou_b200.data import Batch, ReplayBuffer
    keys = ("obs", "act", "rew", "terminated", "truncated", "done", "obs_next")
    if int(golden_cfg(g)["adds"]) == 0:
        buf = ReplayBuffer.from_data(*(g["buf_" + k].copy() for k in keys))
    else:
        buf = ReplayBuffer(int(golden_cfg(g)["size"]), device=DEV)
        buf.set_batch(Batch(**{k: g["buf_" + k].copy() for k in keys}))
        ins, size = int(g["buf_insertion_idx"]), int(g["buf_size"])
        set_buffer_state(buf, np.array([(ins - 1) % size]), np.array([size]))
    if mirror:
        buf.enable_device_mirror()
        buf.sync_device_mirror()
        assert buf.device_columns() is not None
    return buf


@gpu
@pytest.mark.parametrize("mirror", [False, True])
@pytest.mark.parametrize("variant", ["d4rl", "nolag", "wrap"])
def test_update_matches_reference(variant, mirror):
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden(f"cql_ref_{variant}.npz")
    cfg = golden_cfg(g)
    algo = build_from_cfg(cfg, g)
    assert sorted(algo.state_dict().keys()) == list(g["state_dict_keys"]), "state_dict() keys differ from the reference's"
    buf = algo.process_buffer(buffer_from_golden(g, mirror))
    if bool(cfg["calibrated"]):
        record_parity(f"cql/{variant}/calibration_returns", np.asarray(buf._meta["calibration_returns"]), g["calibration_returns"],
                      rtol=1e-12, atol=1e-12)
    if mirror:
        assert buf.device_columns() is not None, "process_buffer must keep the device mirror"
    # the reference drew its rsample noise from torch's CPU generator (it ran on the CPU): same draws, uploaded
    algo._noise_fn = lambda shape: torch.normal(torch.zeros(shape), torch.ones(shape)).to(DEV)
    captured = {}
    orig = algo._preprocess_batch

    def hook(batch, buffer, indices):
        captured["indices"] = np.asarray(indices).copy()
        return orig(batch, buffer, indices)

    algo._preprocess_batch = hook
    c2_lr = float(cfg["critic2_lr"]) if bool(cfg["critic2"]) else float(cfg["critic_lr"])
    for u in range(int(cfg["updates"])):
        torch.manual_seed(100 + u)
        with policy_within_training_step(algo.policy):
            stats = algo.update(buf, int(cfg["bs"]))
        o, tag = f"u{u}_", f"cql/{variant}_m{int(mirror)}_u{u}"
        assert np.array_equal(captured["indices"], g[o + "indices"]), "sampled indices differ from the reference's"
        assert np.array_equal(torch.get_rng_state().numpy(), g[o + "torch_rng"]), "CPU generator differs from the reference's"
        got = np.array([stats.actor_loss, stats.critic1_loss, stats.critic2_loss])
        record_parity(f"{tag}/losses", got, g[o + "losses"], rtol=2e-5, atol=2e-6)
        if bool(cfg["with_lagrange"]):
            record_parity(f"{tag}/cql_alpha", np.array([stats.cql_alpha, stats.cql_alpha_loss, algo.cql_log_alpha.item()]),
                          np.array([g[o + "cql_alpha"], g[o + "cql_alpha_loss"], g[o + "cql_log_alpha"]]), rtol=2e-5, atol=1e-7)
        else:
            assert stats.cql_alpha is None and stats.cql_alpha_loss is None
        record_parity(f"{tag}/alpha", np.array([stats.alpha]), np.array([g[o + "alpha"]]), rtol=1e-6, atol=0)
        if bool(cfg["auto"]):
            record_parity(f"{tag}/alpha_loss", np.array([stats.alpha_loss]), np.array([g[o + "alpha_loss"]]), rtol=2e-5, atol=1e-7)
        check_params(tag, algo.policy.actor, g, o + "actor_", float(cfg["actor_lr"]))
        check_params(tag, algo.critic, g, o + "c1_", float(cfg["critic_lr"])); check_params(tag, algo.critic2, g, o + "c2_", c2_lr)
        check_params(tag, algo.critic_old, g, o + "c1old_", float(cfg["critic_lr"]))
        check_params(tag, algo.critic2_old, g, o + "c2old_", c2_lr)


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
    trunc = (rng.random(n) < 0.02) & ~term
    return ReplayBuffer.from_data(rng.standard_normal((n, O)).astype(np.float32), np.tanh(rng.standard_normal((n, A))).astype(np.float32),
                                  rng.standard_normal(n), term, trunc, term | trunc, rng.standard_normal((n, O)).astype(np.float32))


GRAD_CASES = [(11, 3, (256, 256), 10), (376, 17, (64, 64), 3)]


@gpu
@pytest.mark.parametrize("O,A,H,R", GRAD_CASES, ids=["hopper", "obs376-act17"])
def test_update_gradients_vs_fp64_autograd(O, A, H, R):
    grad_case(O, A, H, R)


def grad_case(O, A, H, R, B=128, edge=""):
    """One update at batch ``B`` (128 in the suite's own cases): the gradient of each of the four optimiser steps (actor,
    Lagrange multiplier, critic 1, critic 2), taken
    before its Adam step, against float64 autograd of the eager restatement on copies of the modules with the same batch,
    noise and random actions.  Adam's first step is lr * sign(g); this is the check that sees a gradient off by a factor."""
    from oracle.oracle_cql import cql_nets, cql_update
    from tianshou_b200.algorithm.flat_params import FlatGroup
    from tianshou_b200.utils import policy_within_training_step
    cfg = dict(obs=O, act=A, hidden=H, critic2=True, critic2_lr=1e-3, auto=False, alpha=0.2, cql_alpha_lr=1e-3, cql_weight=1.0,
               tau=0.005, gamma=0.99, temperature=1.0, with_lagrange=True, lagrange_threshold=10.0, min_action=-0.5, max_action=1.0,
               R=R, alpha_min=0.0, alpha_max=1e6, max_grad_norm=1e9, calibrated=True, actor_lr=1e-4, critic_lr=3e-4)
    torch.manual_seed(3)
    algo = build_from_cfg(cfg)
    with torch.no_grad():
        algo.cql_log_alpha.fill_(0.4)
    nets = cql_nets(O, A, H)
    src_actor = [*algo.policy.actor.preprocess.parameters(), *algo.policy.actor.mu.parameters(), *algo.policy.actor.sigma.parameters()]
    with torch.no_grad():
        for p, q in zip(nets.actor_params(), src_actor, strict=True):
            p.copy_(q.detach().cpu())
        for k, (c, co) in enumerate(((algo.critic, algo.critic_old), (algo.critic2, algo.critic2_old))):
            for p, q in zip(nets.c[k].parameters(), c.parameters(), strict=True):
                p.copy_(q.detach().cpu())
            for p, q in zip(nets.c_old[k].parameters(), co.parameters(), strict=True):
                p.copy_(q.detach().cpu())
    for m in (nets.a_trunk, nets.a_mu, nets.a_sigma, *nets.c, *nets.c_old):
        m.double()
    buf = algo.process_buffer(_random_buffer(O, A, 600, seed=O))
    noises = []

    def noise(shape):
        noises.append(torch.randn(shape, device=DEV))
        return noises[-1]

    algo._noise_fn = noise
    names = {id(algo._g_actor): "actor", id(algo._g_c[0]): "c1", id(algo._g_c[1]): "c2", id(algo._g_la): "la"}
    cap = {}

    def adam(group, optimizer, mgn):
        cap[names[id(group)]] = group.grad[:group.n].detach().cpu().double().clone()
        FlatGroup.adam_step(group, optimizer, mgn)

    algo._adam = adam
    orig = algo._preprocess_batch
    algo._preprocess_batch = lambda b, buffer, idx: (cap.update(indices=np.asarray(idx).copy()), orig(b, buffer, idx))[1]
    torch.manual_seed(9)
    with policy_within_training_step(algo.policy):
        stats = algo.update(buf, B)
    torch.cuda.synchronize()
    idx = cap["indices"]
    f64 = lambda k: torch.as_tensor(np.asarray(buf._meta[k])[idx]).to(torch.float64)
    batch = dict(obs=f64("obs"), act=f64("act"), rew=torch.as_tensor(np.asarray(buf._meta["rew"])[idx]).float().double(),
                 done=f64("done"), obs_next=f64("obs_next"),
                 calibration_returns=torch.as_tensor(np.asarray(buf._meta["calibration_returns"])[idx]).float().double())
    it = iter(noises)
    la = torch.tensor([0.4], dtype=torch.float64, requires_grad=True)
    opts = [_Recorder(nets.actor_params(), lr=1e-4), _Recorder(nets.c[0].parameters(), lr=3e-4), _Recorder(nets.c[1].parameters(), lr=1e-3)]
    la_opt = _Recorder([la], lr=1e-3)
    torch.manual_seed(9)
    ref = cql_update(nets, opts, 0.2, (la, la_opt), batch, lambda shape: next(it).double().cpu(), gamma=0.99, tau=0.005, temperature=1.0,
                     cql_weight=1.0, num_repeat_actions=R, lagrange_threshold=10.0, min_action=-0.5, max_action=1.0, alpha_min=0.0,
                     alpha_max=1e6, max_grad_norm=1e9)
    tag = f"cql_grad{edge}/O{O}_A{A}"
    for name, opt in (("actor", opts[0]), ("c1", opts[1]), ("c2", opts[2]), ("la", la_opt)):
        want = torch.cat([g.reshape(-1) for g in opt.seen]).numpy()
        got = cap[name].numpy()
        if name == "actor":        # the flat layout is trunk, (mu ; sigma) weights, (mu ; sigma) biases
            grp = algo._g_actor
            got = np.concatenate([grp.view(cap[name], p).numpy() for p in src_actor])
        record_parity(f"{tag}/grad_{name}", got, want, rtol=2e-4, atol=1e-4 * float(np.abs(want).max()) + 1e-12)
    record_parity(f"{tag}/losses", np.array([stats.actor_loss, stats.critic1_loss, stats.critic2_loss, stats.cql_alpha_loss]),
                  np.array([ref["actor_loss"], ref["critic1_loss"], ref["critic2_loss"], ref["cql_alpha_loss"]]), rtol=2e-5, atol=1e-5)
    assert len(idx) == B and algo._scratch["rep_idx"].numel() == B * R, "the repeated-action rows must be B x R"


# ------------------------------------------------------------------------------------------------------------ host sync
@gpu
def test_device_update_has_no_torch_host_sync():
    """Everything after the sampling runs under torch.cuda.set_sync_debug_mode("error") (fixed alpha, mirrored buffer)."""
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden("cql_ref_d4rl.npz")
    algo = build_from_cfg(golden_cfg(g), g)
    buf = algo.process_buffer(buffer_from_golden(g, mirror=True))
    with policy_within_training_step(algo.policy):
        algo.update(buf, 32)                      # first update: scratch buffers exist afterwards
        batch, indices = algo._sample(buf, 32)
        batch = algo._preprocess_batch(batch, buf, indices)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            losses, alpha_loss = algo._device_update(batch)
        finally:
            torch.cuda.set_sync_debug_mode("default")
    assert alpha_loss is None and bool(torch.isfinite(losses).all())


# ------------------------------------------------------------------------------------------------------------ state_dict
@gpu
@pytest.mark.parametrize("variant", ["d4rl", "nolag"])
def test_state_dict_round_trip_continues_identically(variant):
    """A fresh algorithm loaded from another's ``state_dict()`` after one update continues bit for bit; the multiplier and its
    Adam (not in state_dict(), as in the reference) and AutoAlpha's Adam are carried over by hand."""
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden(f"cql_ref_{variant}.npz")
    cfg = golden_cfg(g)
    a = build_from_cfg(cfg, g)
    buf_a = a.process_buffer(buffer_from_golden(g, mirror=False))
    torch.manual_seed(1)
    with policy_within_training_step(a.policy):
        a.update(buf_a, int(cfg["bs"]))
    b = build_from_cfg(cfg, g)
    with torch.no_grad():
        for p in b.parameters():
            p.add_(0.01)
    b.load_state_dict(copy.deepcopy(a.state_dict()))
    with torch.no_grad():
        b.cql_log_alpha.copy_(a.cql_log_alpha)
    b.cql_alpha_optim.load_state_dict(copy.deepcopy(a.cql_alpha_optim.state_dict()))
    if bool(cfg["auto"]):
        b.alpha._optim.load_state_dict(copy.deepcopy(a.alpha._optim.state_dict()))
    for algo in (a, b):
        buf = algo.process_buffer(buffer_from_golden(g, mirror=False))
        for u in range(2):
            torch.manual_seed(10 + u)
            with policy_within_training_step(algo.policy):
                algo.update(buf, int(cfg["bs"]))
    for ga, gb in zip([a._g_actor, *a._g_c, *a._g_ct, a._g_la], [b._g_actor, *b._g_c, *b._g_ct, b._g_la], strict=True):
        assert torch.equal(ga.flat, gb.flat) and torch.equal(ga.exp_avg, gb.exp_avg) and torch.equal(ga.exp_avg_sq, gb.exp_avg_sq)
        assert ga.step == gb.step
    if bool(cfg["with_lagrange"]):
        assert a.cql_log_alpha.item() != 0.0


# ------------------------------------------------------------------------------------------------------------ refusals
@gpu
def test_refusals():
    from tianshou_b200.algorithm import CQL, AdamOptimizerFactory, RMSpropOptimizerFactory, UnsupportedModelError
    from tianshou_b200.algorithm.modelfree.sac import SACPolicy
    from tianshou_b200.utils import policy_within_training_step
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.continuous import ContinuousActorProbabilistic, ContinuousCritic
    O, A = 4, 2

    def make(dev=DEV, opt=AdamOptimizerFactory, c_sigma=True, **kw):
        actor = ContinuousActorProbabilistic(preprocess_net=Net(state_shape=(O,), hidden_sizes=(8,)), action_shape=(A,), unbounded=True,
                                             conditioned_sigma=c_sigma).to(dev)
        c = ContinuousCritic(preprocess_net=Net(state_shape=(O,), action_shape=(A,), hidden_sizes=(8,), concat=True)).to(dev)
        return CQL(policy=SACPolicy(actor=actor, action_space=Box(A)), policy_optim=opt(lr=1e-3), critic=c, critic_optim=opt(lr=1e-3), **kw)

    make()
    with pytest.raises(UnsupportedModelError, match="no CPU path"):
        make(dev="cpu")
    with pytest.raises(UnsupportedModelError, match="Adam"):
        make(opt=RMSpropOptimizerFactory)
    with pytest.raises(UnsupportedModelError, match="conditioned_sigma"):
        make(c_sigma=False)
    with pytest.raises(ValueError, match="num_repeat_actions"):
        make(num_repeat_actions=0)
    with pytest.raises(ValueError):
        make(alpha=1)                 # Alpha.from_float_or_instance, as in the reference
    algo = make()
    buf = _random_buffer(O, A, 50, seed=1)
    with pytest.raises(AttributeError, match="process_buffer"), policy_within_training_step(algo.policy):
        algo.update(buf, 8)


# ------------------------------------------------------------------------------------------------------------ resources
def test_cql_kernels_have_no_stack_frame_or_spills(tmp_path):
    report = ptxas_report("cql.cu", tmp_path)
    names = sorted(re.search(r"cql_(rows|losses|target)_kernel", e).group(1) for e in report)
    assert names == ["losses", "rows", "target"], report
    assert_spill_free(report)
