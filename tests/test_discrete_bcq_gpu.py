"""Discrete BCQ on the GPU: the target and rows kernels against float64, two heads on one trunk against float64 autograd,
``DiscreteBCQ.update()`` against outputs of the imported reference (tests/golden/dbcq_ref_*.npz from
oracle/gen_golden_discrete_bcq.py), ``state_dict()`` keys and round trip, the policy's torch path, the refusals and the kernels'
register report."""
import copy
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from oracle import oracle_discrete_bcq as odb
from oracle import oracle_discrete_sac as ods
from ts_testutil import load_golden, record_parity

DEV = "cuda:0"
gpu = pytest.mark.gpu
EPS = float(np.finfo(np.float32).eps)
A_CASES = (1, 2, 6, 18, 33, 64, 1000)


class _Discrete:
    def __init__(self, n):
        self.n = n
        self.shape = ()


def past_grid_rows():
    """More rows than the per-row kernels' grid has warps, and not a multiple of anything."""
    return torch.cuda.get_device_properties(0).multi_processor_count * 16 * 8 + 37


def row_bound(A, terms):
    """A warp's row sum: each lane adds ceil(A / 32) terms in order, then five butterfly levels, every term a few roundings off:
    ~(A / 32 + 10) eps times the sum of the magnitudes of the terms."""
    return (np.ceil(A / 32) + 10) * EPS * terms


def block_bound(B, terms):
    """The closing one-block sum over B rows: B / 1024 terms per thread in order, then a ten-level tree."""
    return (np.ceil(B / 1024) + 12) * EPS * terms


# ------------------------------------------------------------------------------------------------------------ kernels
@gpu
@pytest.mark.parametrize("A", A_CASES)
def test_target_kernel_matches_torch_expression(A):
    """Exact: the kernel forms the masked values in fp32 as torch does, so the chosen action is torch's, ties included."""
    from tianshou_b200._cabi import call, ptr, stream_ptr
    g = torch.Generator().manual_seed(A)
    B = past_grid_rows() if A == 6 else 301
    q = torch.randint(-2, 3, (B, A), generator=g).float()          # exact ties, also under the mask
    z = torch.randn(B, A, generator=g) * 2
    q_old = torch.randn(B, A, generator=g)
    z[:7] = 0.0                                                     # every logit equal: nothing masked at any threshold
    for log_tau in (float(np.log(0.6)), float(np.log(0.05)), -1e-9, -np.inf):
        ref_a = (q - torch.finfo(torch.float32).max * ((z - z.max(-1, keepdim=True).values) < log_tau).float()).argmax(-1)
        out, act = torch.empty(B, device=DEV), torch.empty(B, dtype=torch.int64, device=DEV)
        qd, zd, od = q.to(DEV), z.to(DEV), q_old.to(DEV)
        call("ts_discrete_bcq_target", ptr(qd), ptr(zd), ptr(od), log_tau, B, A, ptr(out), ptr(act), stream_ptr(torch.device(DEV)))
        torch.cuda.synchronize()
        assert torch.equal(act.cpu(), ref_a), f"A={A} log_tau={log_tau}"
        assert torch.equal(out.cpu(), q_old[torch.arange(B), ref_a])
        assert np.array_equal(odb.bcq_select(q.numpy(), z.numpy(), log_tau), ref_a.numpy())
        if log_tau == -1e-9 and A > 1:          # everything but the arg-max-logit action masked
            assert torch.equal(act.cpu()[7:], z[7:].argmax(-1))


def _bcq_rows(q, z, act, ret, penalty):
    from tianshou_b200._cabi import call, ptr, stream_ptr
    B, A = q.shape
    dq, dz = torch.empty(B, A, device=DEV), torch.empty(B, A, device=DEV)
    rows, losses = torch.empty(3, B, device=DEV), torch.empty(4, device=DEV)
    call("ts_discrete_bcq_rows", ptr(q), ptr(z), ptr(act), ptr(ret), B, A, penalty, ptr(dq), ptr(dz), ptr(rows), ptr(losses),
         stream_ptr(torch.device(DEV)))
    torch.cuda.synchronize()
    return losses.cpu().numpy(), dq.cpu().numpy(), dz.cpu().numpy()


@gpu
@pytest.mark.parametrize("A", A_CASES)
def test_rows_kernel_vs_fp64(A):
    """Losses and both gradients against the float64 restatement (itself pinned to autograd in test_oracle_discrete_bcq), with
    |td| on both sides of the Huber knee and exactly 1, and logit spreads that underflow probabilities."""
    g = torch.Generator().manual_seed(10 + A)
    B = past_grid_rows() if A == 6 else 301
    penalty = 0.3
    q = torch.randn(B, A, generator=g) * 2
    z = torch.randn(B, A, generator=g) * 3
    z[: B // 4] *= 40.0
    act = torch.randint(0, A, (B,), generator=g)
    ret = q[torch.arange(B), act] + torch.randn(B, generator=g) * 1.5
    ret[0], ret[1], ret[2] = 2.0, 2.0, q[2, act[2]]
    q[0, act[0]], q[1, act[1]] = 3.0, 1.0                          # |td| exactly 1 on both sides, and a zero
    losses, dq, dz = _bcq_rows(q.to(DEV), z.to(DEV), act.to(DEV), ret.to(DEV), penalty)
    r = odb.bcq_rows(q.numpy(), z.numpy(), act.numpy(), ret.numpy(), penalty)
    td = (q[torch.arange(B), act] - ret).double().numpy()
    assert (np.abs(td) < 1).any() and (np.abs(td) > 1).any() and (np.abs(td) == 1).sum() >= 2
    z64 = z.double().numpy()
    lp = odb.log_softmax(z64)
    if A > 1:
        assert (np.exp(lp).astype(np.float32) == 0).any(), "the case must underflow some probabilities"
    tag = f"dbcq_rows/A{A}"
    # per row: nll = lse - z[act] carries eps (|z| + |lse|) from the fp32 subtraction and the row bound on sum exp
    lse = z64[:, :1] - lp[:, :1]
    nll_err = EPS * (np.abs(z64).max(-1) + np.abs(lse[:, 0])) * 2 + row_bound(A, 1.0)
    sq_err = row_bound(A, (z64 ** 2).sum(-1))
    q_rows = np.where(np.abs(td) < 1, 0.5 * td * td, np.abs(td) - 0.5)
    bounds = np.array([0.0,
                       (4 * EPS * q_rows).mean() + block_bound(B, q_rows.mean()),
                       nll_err.mean() + block_bound(B, np.abs(-lp[np.arange(B), act.numpy()]).mean()),
                       sq_err.sum() / (B * A) + block_bound(B, (z64 ** 2).mean())])
    bounds[0] = bounds[1] + bounds[2] + penalty * bounds[3] + 4 * EPS * abs(r["losses"][0])
    err = np.abs(losses - r["losses"])
    assert np.all(err <= bounds + 1e-30), f"{tag}: losses off by {err} past {bounds}"
    record_parity(f"{tag}/losses", losses, r["losses"], rtol=0.0, atol=float(bounds.max()))
    record_parity(f"{tag}/dq", dq, r["dq"], rtol=8 * EPS, atol=1e-30)
    # dlogits = (p - hit) / B + 2 penalty z / (B A): p's relative error grows with |z - max| (the fp32 subtraction before exp)
    p = np.exp(lp)
    rel_p = row_bound(A, 1.0) + EPS * (z64.max(-1, keepdims=True) - z64) + 4 * EPS
    bound = (p * rel_p + 4 * EPS * (p + 1.0)) / B + 8 * EPS * np.abs(r["dlogits"]) + 1e-30
    err = np.abs(dz - r["dlogits"])
    assert np.all(err <= bound), f"{tag}: dlogits error {float((err - bound).max()):.3e} past its bound"
    record_parity(f"{tag}/dlogits", dz, r["dlogits"], rtol=0.0, atol=float(bound.max()))
    again = _bcq_rows(q.to(DEV), z.to(DEV), act.to(DEV), ret.to(DEV), penalty)
    assert all(np.array_equal(a, b) for a, b in zip((losses, dq, dz), again)), "two calls must be bit-identical"


# ------------------------------------------------------------------------------------------------------------ two heads
def make_trunk(kind, hidden=(48,), trunk_out=0, H=44, W=44, O=11, A=6):
    from tianshou_b200.env.atari import DQNet, ScaledObsInputActionReprNet
    from tianshou_b200.utils.net.common import Net
    if kind == "cnn":
        return ScaledObsInputActionReprNet(DQNet(4, H, W, A, features_only=True))
    return Net(state_shape=(O,), action_shape=trunk_out, hidden_sizes=hidden)


def make_heads(kind, shared, A, last_hidden, critic_b=False, **kw):
    """Head a = DiscreteActor(softmax_output=False); head b the same, or a DiscreteCritic (CRR)."""
    from tianshou_b200.utils.net.discrete import DiscreteActor, DiscreteCritic
    t1 = make_trunk(kind, A=A, **kw)
    t2 = t1 if shared else make_trunk(kind, A=A, **kw)
    a = DiscreteActor(preprocess_net=t1, action_shape=A, hidden_sizes=last_hidden, softmax_output=False)
    b = (DiscreteCritic(preprocess_net=t2, hidden_sizes=last_hidden, last_size=A) if critic_b
         else DiscreteActor(preprocess_net=t2, action_shape=A, hidden_sizes=last_hidden, softmax_output=False))
    return a.to(DEV), b.to(DEV)


def chain64(net):
    """float64 callable of a head's layers (the modules themselves cast their input to fp32)."""
    pre = net.preprocess
    body = pre.module.net if hasattr(pre, "module") else pre.model.model
    return lambda x: net.last.model(body(x))


def copy64(a, b):
    """float64 CPU copies of both heads, a shared trunk still shared."""
    return copy.deepcopy(torch.nn.ModuleList([a, b])).to("cpu", torch.float64)


def check_flat_grads(tag, params, group, grad, ref_params):
    """The GEMMs are fp32-faithful (bf16x3) and a weight gradient sums B products per element: 2e-4 relative plus 1e-4 of the
    tensor's largest value, as in test_discrete_sac_gpu."""
    for i, (p, r) in enumerate(zip(params, ref_params, strict=True)):
        ref = r.grad.numpy()
        got = group.view(grad, p).view(p.shape).cpu().numpy()
        record_parity(f"{tag}/grad_{i}", got, ref, rtol=2e-4, atol=1e-4 * float(np.abs(ref).max()) + 1e-12)


TRUNK_CASES = [("mlp_relu", "mlp", True, dict(hidden=(48, 40))), ("mlp_linear", "mlp", True, dict(hidden=(), trunk_out=64)),
               ("cnn_flatten", "cnn", True, {}), ("mlp_separate", "mlp", False, dict(hidden=(48,))), ("cnn_separate", "cnn", False, {})]


@gpu
@pytest.mark.parametrize("name,kind,shared,kw", TRUNK_CASES, ids=[c[0] for c in TRUNK_CASES])
def test_two_head_backward_vs_fp64_autograd(name, kind, shared, kw):
    """Forward both heads, backward two arbitrary head gradients: every parameter's gradient against float64 autograd, and on a
    shared trunk the gradient equals the sum of the two single-head gradients."""
    from tianshou_b200.algorithm.flat_params import FlatGroup
    from tianshou_b200.algorithm.obs_source import DeviceObsSource
    from tianshou_b200.algorithm.shared_trunk import TwoHeadNetwork, two_head_parameters
    torch.manual_seed(len(name))
    A, B = 5, 77
    a, b = make_heads(kind, shared, A, (24,), **kw)
    params = two_head_parameters(a, b)
    group = FlatGroup(params, torch.device(DEV))
    net = TwoHeadNetwork(a, b, group)
    assert net.shared == shared
    g = torch.Generator().manual_seed(3)
    if kind == "cnn":
        x = torch.rand(B, 4, 44, 44, generator=g)
        src = DeviceObsSource(B, x=x.permute(0, 2, 3, 1).contiguous().to(DEV))       # the first convolution reads NHWC rows
    else:
        x = torch.randn(B, 11, generator=g)
        src = DeviceObsSource(B, x=x.to(DEV))
    da, db = torch.randn(B, A, generator=g).to(DEV), torch.randn(B, A, generator=g).to(DEV)
    zero = torch.zeros(B, A, device=DEV)
    acts = net.forward(src, "t")
    ref = copy64(a, b)
    ya, yb = chain64(ref[0])(x.double()), chain64(ref[1])(x.double())
    record_parity(f"two_head/{name}/out_a", acts.a[-1].cpu().numpy(), ya.detach().numpy(), rtol=1e-4, atol=1e-5)
    record_parity(f"two_head/{name}/out_b", acts.b[-1].cpu().numpy(), yb.detach().numpy(), rtol=1e-4, atol=1e-5)
    net.backward(acts, da, db, "t")
    both = group.grad[: group.n].clone()
    torch.autograd.backward([ya, yb], [da.cpu().double(), db.cpu().double()])
    check_flat_grads(f"two_head/{name}", params, group, both, two_head_parameters(ref[0], ref[1]))
    net.backward(acts, da, zero, "t")
    only_a = group.grad[: group.n].clone()
    net.backward(acts, zero, db, "t")
    only_b = group.grad[: group.n].clone()
    scale = float(both.abs().max())
    assert float((both - (only_a + only_b)).abs().max()) <= 2e-5 * scale
    if shared:
        trunk = [p for p in a.preprocess.parameters()]
        assert all(float(group.view(only_a, p).abs().max()) > 0 and float(group.view(only_b, p).abs().max()) > 0 for p in trunk)


# ------------------------------------------------------------------------------------------------------------ vs reference
def heads_from_golden(g, critic_b=False):
    kind = str(g["cfg_kind"])
    kw = (dict(H=int(g["cfg_H"]), W=int(g["cfg_W"])) if kind == "cnn"
          else dict(O=int(g["cfg_obs"]), hidden=tuple(int(x) for x in g["cfg_hidden"]), trunk_out=int(g["cfg_trunk_out"])))
    a, b = make_heads(kind, bool(g["cfg_shared"]), int(g["cfg_A"]), tuple(int(x) for x in g["cfg_last_hidden"]), critic_b, **kw)
    both = torch.nn.ModuleList([a, b])
    if bool(g["cfg_compact"]):
        ods.seeded_params(both, int(g["cfg_init_seed"]))
    else:
        with torch.no_grad():
            for i, p in enumerate(both.parameters()):
                p.copy_(torch.as_tensor(g[f"p0_{i}"]).reshape(p.shape))
    return a, b


def buffer_from_golden(g, mirror=False):
    from tianshou_b200.data import Batch, VectorReplayBuffer
    E, cap = int(g["cfg_E"]), int(g["cfg_cap"])
    cnn = str(g["cfg_kind"]) == "cnn"
    kw = dict(stack_num=4, ignore_obs_next=True, save_only_last_obs=True) if cnn else {}
    buf = VectorReplayBuffer(E * cap, E, device=DEV, device_mirror=mirror, **kw)
    for i in range(int(g["cfg_steps"])):
        s = {k: g[f"roll{i}_{k}"] for k in ("obs", "act", "rew", "terminated", "truncated")}
        if cnn:
            s["obs"] = np.repeat(s["obs"][:, None], 4, axis=1)        # only the last frame is stored
            s["obs_next"] = s["obs"]
        else:
            s["obs_next"] = g[f"roll{i}_obs_next"]
        buf.add(Batch(**s), buffer_ids=np.arange(E))
    return buf


def check_final_state(tag, g, algo, lagged):
    """Final parameters / Adam moments / lagged parameters within the bars DESIGN.md section 4 uses for DQN and discrete SAC: Adam
    normalises a step to ~lr per element, so the absolute term is stated in units of one step."""
    view = ods.golden_view if bool(g["cfg_compact"]) else (lambda t: t.detach().cpu().numpy())
    lr = float(g["cfg_lr"])
    grp = algo._group
    for i, p in enumerate(grp.params):
        record_parity(f"{tag}/pf_{i}", view(p), g[f"pf_{i}"], rtol=1e-3, atol=0.1 * lr)
        m, v = g[f"m_{i}"], g[f"v_{i}"]
        record_parity(f"{tag}/m_{i}", view(grp.view(grp.exp_avg, p).view(p.shape)), m, rtol=2e-3, atol=2e-3 * float(np.abs(m).max()) + 1e-12)
        record_parity(f"{tag}/v_{i}", view(grp.view(grp.exp_avg_sq, p).view(p.shape)), v, rtol=4e-3, atol=4e-3 * float(np.abs(v).max()) + 1e-20)
    assert grp.sync_step_from_device() == int(g["adam_step"]) and algo._iter == int(g["iter"])
    for i, p in enumerate(lagged):
        record_parity(f"{tag}/old_{i}", view(p), g[f"old_{i}"], rtol=1e-3, atol=0.1 * lr)


def build_bcq(g):
    from tianshou_b200.algorithm import AdamOptimizerFactory, DiscreteBCQ, DiscreteBCQPolicy
    model, imitator = heads_from_golden(g)
    policy = DiscreteBCQPolicy(model=model, imitator=imitator, action_space=_Discrete(int(g["cfg_A"])),
                               target_update_freq=int(g["cfg_freq"]), unlikely_action_threshold=float(g["cfg_tau"]))
    return DiscreteBCQ(policy=policy, optim=AdamOptimizerFactory(lr=float(g["cfg_lr"])), gamma=float(g["cfg_gamma"]),
                       n_step_return_horizon=int(g["cfg_n_step"]), target_update_freq=int(g["cfg_freq"]),
                       imitation_logits_penalty=float(g["cfg_penalty"]))


@gpu
@pytest.mark.parametrize("variant,mirror", [("mlp", False), ("mlp", True), ("cnn", False), ("cnn", True), ("sep", False)])
def test_update_matches_reference(variant, mirror):
    """Update after update against the reference's run, across several lagged copies (the copy BEFORE the step: ``old_*`` of the
    golden is the online model one or two steps back)."""
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden(f"dbcq_ref_{variant}.npz")
    algo, buf = build_bcq(g), buffer_from_golden(g, mirror)
    assert list(algo.state_dict().keys()) == [str(k) for k in g["state_dict_keys"]]
    cap = {}
    orig_pre = algo._preprocess_batch

    def pre(batch, buffer, indices):
        b = orig_pre(batch, buffer, indices)
        cap["indices"], cap["returns"] = np.asarray(indices).copy(), b.returns.detach().cpu().numpy().copy()
        return b

    algo._preprocess_batch = pre
    for u in range(int(g["cfg_updates"])):
        np.random.seed(500 + u)
        with policy_within_training_step(algo.policy):
            stats = algo.update(buffer=buf, sample_size=int(g["cfg_bs"]))
        tag = f"dbcq_{variant}_m{int(mirror)}_u{u}"
        assert np.array_equal(cap["indices"], g[f"u{u}_indices"]), "sampled indices differ from the reference's"
        ref_ret = g[f"u{u}_returns"]
        record_parity(f"{tag}/returns", cap["returns"].reshape(ref_ret.shape), ref_ret, rtol=1e-5, atol=1e-5 * float(np.abs(ref_ret).max()))
        got = np.array([stats.loss, stats.q_loss, stats.i_loss, stats.reg_loss])
        record_parity(f"{tag}/losses", got, g[f"u{u}_losses"], rtol=2e-5, atol=2e-6)
    check_final_state(f"dbcq_{variant}_m{int(mirror)}", g, algo, list(algo.model_old.parameters()))
    assert list(algo.state_dict().keys()) == [str(k) for k in g["state_dict_keys"]]


@gpu
@pytest.mark.parametrize("name,kind,shared,kw", TRUNK_CASES[:4], ids=[c[0] for c in TRUNK_CASES[:4]])
def test_update_gradient_vs_fp64_autograd(name, kind, shared, kw):
    """One update: the flat gradient, snapshotted before its Adam step, against float64 autograd of the reference loss
    (discrete_bcq.py:244-252) on copies of the modules with the same weights, batch and returns.  Adam's first step is
    lr * sign(g), so a gradient off by a constant factor leaves the parameters unchanged; this is the check that sees it."""
    from tianshou_b200.algorithm import AdamOptimizerFactory, DiscreteBCQ, DiscreteBCQPolicy
    from tianshou_b200.algorithm.flat_params import FlatGroup
    from tianshou_b200.data import Batch, VectorReplayBuffer
    from tianshou_b200.utils import policy_within_training_step
    torch.manual_seed(5 + len(name))
    rng = np.random.default_rng(len(name))
    A, E, T, B, penalty = 6, 4, 48, 64, 0.2
    model, imitator = make_heads(kind, shared, A, (24,), **kw)
    algo = DiscreteBCQ(policy=DiscreteBCQPolicy(model=model, imitator=imitator, action_space=_Discrete(A), target_update_freq=3,
                                                unlikely_action_threshold=0.4),
                       optim=AdamOptimizerFactory(lr=1e-3), gamma=0.9, target_update_freq=3, imitation_logits_penalty=penalty)
    cnn = kind == "cnn"
    buf = VectorReplayBuffer(E * T, E, device=DEV, **(dict(stack_num=1, ignore_obs_next=True) if cnn else {}))
    obs_fn = (lambda: rng.integers(0, 256, (E, 4, 44, 44), dtype=np.uint8)) if cnn else (lambda: rng.standard_normal((E, 11)).astype(np.float32))
    obs = obs_fn()
    for t in range(T):
        nxt = obs_fn()
        term = rng.random(E) < 0.1
        buf.add(Batch(obs=obs, act=rng.integers(0, A, E), rew=rng.standard_normal(E) * 2, terminated=term,
                      truncated=np.full(E, t % 17 == 16) & ~term, obs_next=nxt), buffer_ids=np.arange(E))
        obs = nxt
    cap = {}
    grp = algo._group

    def adam(optimizer, mgn):
        cap["grad"], cap["flat"] = grp.grad[: grp.n].clone(), grp.flat.clone()
        FlatGroup.adam_step(grp, optimizer, mgn)

    grp.adam_step = adam
    orig_pre = algo._preprocess_batch

    def pre(batch, buffer, indices):
        b = orig_pre(batch, buffer, indices)
        cap["indices"], cap["returns"] = np.asarray(indices).copy(), b.returns.detach().reshape(-1).cpu().double()
        return b

    algo._preprocess_batch = pre
    ref = copy64(model, imitator)            # the weights before the step
    np.random.seed(7)
    with policy_within_training_step(algo.policy):
        stats = algo.update(buffer=buf, sample_size=B)
    idx = cap["indices"]
    raw = np.asarray(buf.obs)[idx]
    x = torch.as_tensor((raw.astype(np.float64) / 255.0).astype(np.float32) if cnn else raw).double()
    act = torch.as_tensor(np.asarray(buf.act)[idx].astype(np.int64))
    q, z = chain64(ref[0])(x), chain64(ref[1])(x)
    ql = torch.nn.functional.smooth_l1_loss(q[torch.arange(B), act], cap["returns"])
    il = torch.nn.functional.nll_loss(torch.log_softmax(z, -1), act)
    reg = z.pow(2).mean()
    loss = ql + il + penalty * reg
    loss.backward()
    from tianshou_b200.algorithm.shared_trunk import two_head_parameters
    check_flat_grads(f"dbcq_grad/{name}", grp.params, grp, cap["grad"], two_head_parameters(ref[0], ref[1]))
    record_parity(f"dbcq_grad/{name}/losses", np.array([stats.loss, stats.q_loss, stats.i_loss, stats.reg_loss]),
                  np.array([loss.item(), ql.item(), il.item(), reg.item()]), rtol=2e-5, atol=2e-6)


# ------------------------------------------------------------------------------------------------------------ state_dict
@gpu
@pytest.mark.parametrize("variant", ["mlp", "cnn"])
def test_state_dict_round_trip_continues_identically(variant):
    """A fresh algorithm loaded from another's ``state_dict()`` continues bit for bit: online, lagged and optimiser state.
    ``_iter`` is a plain attribute, as in the reference: whoever restores a run restores it too."""
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden(f"dbcq_ref_{variant}.npz")
    a, buf_a = build_bcq(g), buffer_from_golden(g)
    for u in range(3):
        np.random.seed(u)
        with policy_within_training_step(a.policy):
            a.update(buffer=buf_a, sample_size=int(g["cfg_bs"]))
    b = build_bcq(g)
    with torch.no_grad():
        for p in b.parameters():
            p.add_(0.01)
    b.load_state_dict(copy.deepcopy(a.state_dict()))
    b._iter = a._iter
    for algo in (a, b):
        buf = buffer_from_golden(g)
        for u in range(3):
            np.random.seed(10 + u)
            with policy_within_training_step(algo.policy):
                algo.update(buffer=buf, sample_size=int(g["cfg_bs"]))
    for ga, gb in ((a._group, b._group), (a._g_old, b._g_old)):
        assert torch.equal(ga.flat, gb.flat) and torch.equal(ga.exp_avg, gb.exp_avg) and torch.equal(ga.exp_avg_sq, gb.exp_avg_sq)
    assert a._group.step == b._group.step


# ------------------------------------------------------------------------------------------------------------ policy
@gpu
def test_policy_forward_and_exploration_noise():
    from tianshou_b200.algorithm import DiscreteBCQPolicy
    from tianshou_b200.data import Batch
    torch.manual_seed(0)
    A = 5
    model, imitator = make_heads("mlp", True, A, (16,), hidden=(32,))
    with torch.no_grad():          # a logit spread wide enough that the threshold masks some actions
        imitator.last.model[-1].weight.mul_(20.0)
    policy = DiscreteBCQPolicy(model=model, imitator=imitator, action_space=_Discrete(A), unlikely_action_threshold=0.5,
                               eps_inference=0.3)
    obs = np.random.default_rng(0).standard_normal((500, 11)).astype(np.float32)
    out = policy(Batch(obs=obs, info=Batch()))
    q, _ = model(obs)
    z, _ = imitator(obs)
    ref = (q - torch.finfo(torch.float32).max * ((z - z.max(-1, keepdim=True).values) < np.log(0.5)).float()).argmax(-1)
    assert torch.equal(out.act, ref) and torch.equal(out.q_value, q) and torch.equal(out.imitation_logits, z)
    assert out.logits is out.imitation_logits or torch.equal(out.logits, z)
    assert not torch.equal(ref, q.argmax(-1)), "the mask must change some choices"
    act = out.act.cpu().numpy()
    np.random.seed(4)
    noisy = policy.add_exploration_noise(act.copy(), Batch(obs=obs))
    np.random.seed(4)
    rand_mask = np.random.rand(500) < 0.3
    rand_act = np.random.rand(500, A).argmax(axis=1)
    assert np.array_equal(noisy, np.where(rand_mask, rand_act, act))
    policy.is_within_training_step = True          # eps_training is 0: offline, nothing is collected
    assert np.array_equal(policy.add_exploration_noise(act.copy(), Batch(obs=obs)), act)


# ------------------------------------------------------------------------------------------------------------ refusals
@gpu
def test_refusals():
    from tianshou_b200.algorithm import (AdamOptimizerFactory, DiscreteBCQ, DiscreteBCQPolicy, RMSpropOptimizerFactory,
                                         UnsupportedModelError)
    from tianshou_b200.data import Batch, VectorReplayBuffer
    from tianshou_b200.utils import policy_within_training_step
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.discrete import DiscreteActor
    A = 3

    def make(model=None, imitator=None, opt=AdamOptimizerFactory, n=A, **kw):
        m, i = make_heads("mlp", True, A, (8,), hidden=(16,))
        model, imitator = model or m, imitator or i
        return DiscreteBCQ(policy=DiscreteBCQPolicy(model=model, imitator=imitator, action_space=_Discrete(n)), optim=opt(lr=1e-3), **kw)

    algo = make()
    head = lambda trunk, **kw: DiscreteActor(preprocess_net=trunk, action_shape=A, **{"softmax_output": False, **kw}).to(DEV)
    net = lambda **kw: Net(state_shape=(11,), hidden_sizes=(16, 16), **kw)
    t1, t2 = net(), net()
    t2.model.model[0] = t1.model.model[0]
    with pytest.raises(UnsupportedModelError, match="share some parameters"):
        make(head(t1), head(t2))
    with pytest.raises(UnsupportedModelError, match="imitator: .*softmax_output=True"):
        make(imitator=head(net(), softmax_output=True))
    with pytest.raises(UnsupportedModelError, match="must read it the same way"):
        make(head(net()), head(Net(state_shape=(5,), hidden_sizes=(16,))))
    with pytest.raises(UnsupportedModelError, match="softmax preprocess"):
        make(head(net(softmax=True)), head(net()))
    with pytest.raises(UnsupportedModelError, match="outside the fused layered-network family"):
        make(head(net(norm_layer=torch.nn.LayerNorm)), head(net()))
    with pytest.raises(UnsupportedModelError, match="outputs for 4 actions"):
        make(n=4)
    with pytest.raises(UnsupportedModelError, match="Adam"):
        make(opt=RMSpropOptimizerFactory)
    with pytest.raises(UnsupportedModelError, match="no CPU path"):
        make(head(net()).cpu(), head(net()).cpu())
    for kw in (dict(gamma=1.5), dict(n_step_return_horizon=0), dict(target_update_freq=0)):
        with pytest.raises(AssertionError):
            make(**kw)
    # an action the networks have no output for is refused on the host, before any kernel indexes with it
    buf = VectorReplayBuffer(40, 4, device=DEV)
    rng = np.random.default_rng(0)
    for _ in range(8):
        buf.add(Batch(obs=rng.standard_normal((4, 11)).astype(np.float32), act=np.array([0, 1, 2, A]), rew=np.zeros(4),
                      terminated=np.zeros(4, bool), truncated=np.zeros(4, bool), obs_next=rng.standard_normal((4, 11)).astype(np.float32)),
                buffer_ids=np.arange(4))
    with pytest.raises(ValueError, match="actions in"), policy_within_training_step(algo.policy):
        algo.update(buffer=buf, sample_size=32)


# ------------------------------------------------------------------------------------------------------------ resources
@pytest.mark.parametrize("source,kernels", [("discrete_bcq.cu", ("discrete_bcq_rows_kernel", "discrete_bcq_target_kernel", "row_sums3_kernel")),
                                            ("discrete_crr.cu", ("discrete_crr_rows_kernel", "discrete_crr_sums_kernel", "row_sums3_kernel"))])
def test_kernels_have_no_stack_frame_or_spills(tmp_path, source, kernels):
    from tianshou_b200.csrc import build as B
    if shutil.which(B.NVCC) is None and not os.path.exists(B.NVCC):
        pytest.skip("nvcc not available")
    r = subprocess.run([B.NVCC, *B.FLAGS, "-c", os.path.join(B.HERE, source), "-o", str(tmp_path / "d.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    hits = re.findall(r"Compiling entry function '(\S+)' for 'sm_90a'\n(?:.*\n)*?\s*(\d+) bytes stack frame, (\d+) bytes spill "
                      r"stores, (\d+) bytes spill loads", r.stdout + r.stderr)
    assert hits and all(any(k in h[0] for k in kernels) for h in hits), hits
    assert all(tuple(map(int, h[1:])) == (0, 0, 0) for h in hits), hits
