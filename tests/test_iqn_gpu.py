"""IQN on the GPU: the cosine, mix, target and rows kernels against the float64 restatement (oracle/oracle_iqn.py),
``IQN.update()`` against outputs of the imported reference replayed with the reference's own fractions
(tests/golden/iqn_ref_*.npz from oracle/gen_golden_iqn.py), one update's gradient against float64 autograd, bit-identical
repeats, the ``state_dict()`` round trip, the policy's torch path, the refusals and the kernels' register report."""
import copy
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from oracle import oracle_discrete_sac as ods
from oracle import oracle_iqn as oi
from test_qrdqn_gpu import _Discrete, _st, buffer_from_golden, check_final_state, make_buffer, sms
from ts_testutil import load_golden, record_parity

DEV = "cuda:0"
gpu = pytest.mark.gpu
EPS = float(np.finfo(np.float32).eps)
VARIANTS = ["iqn_ref_mlp", "iqn_ref_sizes", "iqn_ref_cnn", "iqn_ref_per"]
ACTS = {"none": 0, "relu": 1, "tanh": 2}


def dev(a, dt=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dt, device=DEV)


# ------------------------------------------------------------------------------------------------------------ cosine
def _cos(taus, C):
    from tianshou_b200._cabi import call, ptr
    t = dev(taus.reshape(-1))
    out = torch.empty(t.numel(), C, device=DEV)
    call("ts_iqn_cos", ptr(t), t.numel(), C, ptr(out), _st())
    torch.cuda.synchronize()
    return out.cpu().numpy()


@gpu
@pytest.mark.parametrize("C", [1, 17, 64])
def test_cos_kernel_argument_and_accuracy(C):
    """CUDA's cosf (without fast math) is within 2 ulp of the exact cosine of its fp32 argument.  The bound is against the
    float64 cosine of the reference's fp32 argument fl(tau * fl(fl32(pi) * i)); at these arguments (up to 64 pi) one ulp of the
    argument moves the cosine by up to ~1e-5, hundreds of ulp of the result, so an argument formed any other way (a double pi, a
    fused product) falls outside the bound.  The case with C = 64 checks that it does.  tau = 0 gives 1 exactly; tau just
    below 1 is the largest fraction torch.rand returns.  R runs past the one-warp-per-row grid."""
    rng = np.random.default_rng(C)
    R = sms() * 16 * 8 + 37 if C == 17 else 300
    taus = rng.random(R).astype(np.float32)
    taus[0], taus[1] = 0.0, np.nextafter(np.float32(1.0), np.float32(0.0))
    got = _cos(taus, C)
    want = oi.cos_features(taus, C)
    bound = 2 * np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)
    err = np.abs(got - want)
    assert np.all(err <= bound), f"cos off by {float((err / bound).max()):.2f} x its 2-ulp bound"
    record_parity(f"iqn_cos/C{C}", got, want, rtol=0.0, atol=float(bound.max()))
    assert np.all(got[0] == 1.0)
    if C == 64:
        other = np.cos((taus.astype(np.float64)[:, None] * (np.pi * np.arange(1, C + 1))).astype(np.float32).astype(np.float64))
        assert np.count_nonzero(np.abs(got - other) > bound) > R, "the bound must tell the fp32 argument from a double-pi one"
    assert np.array_equal(got, _cos(taus, C)), "two calls must be bit-identical"


# ------------------------------------------------------------------------------------------------------------ mix
def _mix_case(B, S, D, rng):
    feat = rng.standard_normal((B, D)).astype(np.float32)
    e = np.maximum(rng.standard_normal((B * S, D)), 0.0).astype(np.float32)        # a ReLU output: exact zeros at the kink
    dh = rng.standard_normal((B * S, D)).astype(np.float32)
    return feat, e, dh


@gpu
@pytest.mark.parametrize("act", ["none", "relu", "tanh"])
@pytest.mark.parametrize("S", [2, 8, 64])
@pytest.mark.parametrize("D", [64, 37, 3136])
def test_mix_and_mix_backward_vs_fp64(D, S, act):
    """h = feat * e is one fp32 product: exact against numpy's.  de_pre = dh * feat where e > 0 is one product too, exact, and
    exactly 0 wherever e is exactly 0.  dfeat sums S products in order (each product and add rounded, or fused): off by at most
    (S + 1) eps times sum_s |dh e|; the tanh derivative 1 - y^2 (one fused rounding) and the product add 2 eps, the ReLU mask
    nothing.  B runs past the element-wise grid (8 blocks per SM) in the largest case."""
    from tianshou_b200._cabi import call, ptr
    rng = np.random.default_rng(D * 100 + S * 3 + ACTS[act])
    B = sms() * 8 * 256 // D + 5 if (D, S) == (3136, 8) else 33
    feat, e, dh = _mix_case(B, S, D, rng)
    if act == "relu":
        feat = np.maximum(feat, 0.0)
    elif act == "tanh":
        feat = np.tanh(feat).astype(np.float32)
    f_d, e_d, dh_d = dev(feat), dev(e), dev(dh)
    h = torch.empty(B * S, D, device=DEV)
    call("ts_iqn_mix", ptr(f_d), ptr(e_d), B, S, D, ptr(h), _st())
    want_h = (np.repeat(feat, S, axis=0) * e).astype(np.float32)
    assert np.array_equal(h.cpu().numpy(), want_h)

    def backward():
        dfeat, de = torch.empty(B, D, device=DEV), torch.empty(B * S, D, device=DEV)
        call("ts_iqn_mix_backward", ptr(dh_d), ptr(f_d), ptr(e_d), B, S, D, ACTS[act], ptr(f_d) if act != "none" else None,
             ptr(dfeat), ptr(de), _st())
        torch.cuda.synchronize()
        return dfeat.cpu().numpy(), de.cpu().numpy()

    dfeat, de = backward()
    ref_df, ref_de = oi.mix_backward(dh, feat, e, S, act, feat)
    assert np.array_equal(de, (dh * np.repeat(feat, S, axis=0) * (e > 0)).astype(np.float32))
    assert np.all(de[e == 0] == 0.0) and np.count_nonzero(e == 0) > 0
    mag = (np.abs(dh.astype(np.float64) * e).reshape(B, S, D)).sum(1)
    deriv = {"none": 1.0, "relu": 1.0, "tanh": np.abs(1.0 - feat.astype(np.float64) ** 2)}[act]
    bound = (S + 1) * EPS * mag * deriv + (2 * EPS * np.abs(ref_df) if act == "tanh" else 0.0) + 1e-30
    err = np.abs(dfeat - ref_df)
    assert np.all(err <= bound), f"dfeat off by {float((err / bound).max()):.2f} x its bound"
    record_parity(f"iqn_mix_backward/D{D}_S{S}_{act}/dfeat", dfeat, ref_df, rtol=0.0, atol=float(bound.max()))
    again = backward()
    assert np.array_equal(dfeat, again[0]) and np.array_equal(de, again[1]), "two launches must be bit-identical"


# ------------------------------------------------------------------------------------------------------------ target
@gpu
@pytest.mark.parametrize("S_on,S_next", [(8, 8), (8, 5), (3, 40), (64, 32)])
@pytest.mark.parametrize("A", [1, 2, 6, 18])
def test_target_kernel_exact(A, S_on, S_next):
    """Exact.  Integer-valued quantiles make every sample sum exact in fp32 and float64 alike, so the means order the actions
    the same way in both and equal sums are exact ties: the first action of a tie must win.  A NaN mean is the maximum.  B
    runs past the one-warp-per-row grid in one case; the same-buffer call is ``target_update_freq == 0``."""
    from tianshou_b200._cabi import call, ptr
    g = torch.Generator().manual_seed(A * 1000 + S_on * 10 + S_next)
    B = sms() * 16 * 8 + 37 if (A, S_on) == (6, 8) and S_next == 5 else 301
    q = torch.randint(-3, 4, (B, S_on, A), generator=g).float()
    q_next = torch.randn(B, S_next, A, generator=g)
    if A > 1:
        q[: B // 3, :, A - 1] = q[: B // 3, :, 0]                      # two equal columns: the first wins where they lead
        q[B - 1, S_on - 1, A - 1] = float("nan")                       # a NaN mean wins
    out, act = torch.empty(B, S_next, device=DEV), torch.empty(B, dtype=torch.int64, device=DEV)
    qd, nd = q.to(DEV), q_next.to(DEV)
    call("ts_iqn_target", ptr(qd), ptr(nd), B, A, S_on, S_next, ptr(out), ptr(act), _st())
    torch.cuda.synchronize()
    ref_a = q.mean(1).argmax(1)
    assert torch.equal(act.cpu(), ref_a)
    assert torch.equal(out.cpu(), q_next[torch.arange(B), :, ref_a])
    if A > 1:
        lead = q[: B // 3].sum(1).argmax(1) == 0
        assert bool(lead.any()) and bool((act.cpu()[: B // 3][lead] == 0).all())
        assert int(act[B - 1]) == A - 1
    out_same = torch.empty(B, S_on, device=DEV)
    call("ts_iqn_target", ptr(qd), ptr(qd), B, A, S_on, S_on, ptr(out_same), None, _st())
    torch.cuda.synchronize()
    torch.testing.assert_close(out_same.cpu(), q[torch.arange(B), :, ref_a], rtol=0, atol=0, equal_nan=True)


# ------------------------------------------------------------------------------------------------------------ rows
def _rows(q, act, ret, taus, w):
    from tianshou_b200._cabi import call, ptr
    B, S_on, A = q.shape
    S_t = ret.shape[1]
    dq, prio = torch.empty(B, S_on, A, device=DEV), torch.empty(B, device=DEV)
    rows, losses = torch.empty(3, B, device=DEV), torch.empty(4, device=DEV)
    call("ts_iqn_rows", ptr(q), ptr(act), ptr(ret), ptr(taus), ptr(w), B, A, S_on, S_t, ptr(dq), ptr(prio), ptr(rows), ptr(losses),
         _st())
    torch.cuda.synchronize()
    return losses.cpu().numpy(), dq.cpu().numpy(), prio.cpu().numpy()


@gpu
@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("S_on,S_t", [(2, 3), (8, 8), (64, 32)])
@pytest.mark.parametrize("A", [1, 2, 6, 18])
def test_rows_kernel_vs_fp64(A, S_on, S_t, weighted):
    """Loss, priorities and d loss / d q against the float64 restatement (pinned to autograd of the reference's expression in
    test_oracle_iqn), with pairs at u == 0 exactly, |u| == 1 exactly (both signs) and a fraction of exactly 0.

    Error model (fp32, eps = 2^-23): u = t - c is one rounding, h and |tau - 1[u <= 0]| a few more, and each thread sums its
    S_t pair terms in order: a quantile's sum is off by at most (S_t + 4) eps times the sum of its terms' magnitudes; the CTA
    then adds the per-thread partials, five butterfly levels and eight warp partials, (S_t + 20) eps in all for qr_b and prio_b
    (every term is >= 0).  The batch mean comes from row_sums3_kernel: (B / 1024 + 12) eps times the mean magnitude."""
    rng = np.random.default_rng(A * 7919 + S_on * 31 + S_t + weighted * 3)
    B = sms() * 8 + 37 if (A, S_on, weighted) == (6, 8, True) else 41
    q = (rng.standard_normal((B, S_on, A)) * 2).astype(np.float32)
    act = rng.integers(0, A, B)
    ret = (q[np.arange(B), 0, act][:, None] + rng.standard_normal((B, S_t)) * 1.5).astype(np.float32)
    ret[0, 0] = q[0, S_on - 1, act[0]]                                     # u = 0 exactly
    q[1, 0, act[1]], ret[1, 0], ret[1, 1] = 0.5, -0.5, 1.5                 # |u| = 1 exactly, both signs
    taus = rng.random((B, S_on)).astype(np.float32)
    taus[2, 0] = 0.0
    w = rng.uniform(0.2, 1.0, B).astype(np.float32) if weighted else None
    args = (dev(q), dev(act, torch.int64), dev(ret), dev(taus), None if w is None else dev(w))
    losses, dq, prio = _rows(*args)
    q64, ret64, tau64 = q.astype(np.float64), ret.astype(np.float64), taus.astype(np.float64)
    wb = np.ones(B) if w is None else w.astype(np.float64)
    ref = oi.iqn_rows(q64, act, ret64, tau64, None if w is None else wb)
    rel = (S_t + 20) * EPS
    tag = f"iqn_rows/A{A}_S{S_on}x{S_t}_w{int(weighted)}"
    record_parity(f"{tag}/prio", prio, ref["prio"], rtol=rel, atol=1e-30)
    bound = (wb * ref["qr_b"] * rel).mean() + (np.ceil(B / 1024) + 12) * EPS * (wb * ref["qr_b"]).mean() + 1e-30
    assert abs(losses[0] - ref["loss"]) <= bound and losses[1] == losses[0] and losses[2] == 0.0
    record_parity(f"{tag}/loss", losses[:1], [ref["loss"]], rtol=0.0, atol=float(bound))
    c = q64[np.arange(B), :, act]
    u = ret64[:, None, :] - c[:, :, None]
    wt = np.abs(tau64[:, :, None] - (u <= 0.0))
    mag = np.abs(wt * np.clip(u, -1, 1)).sum(-1)                         # [B, S_on]
    dbound = np.zeros((B, S_on, A))
    dbound[np.arange(B), :, act] = (S_t + 4) * EPS * mag * (wb / (B * S_on))[:, None]
    dbound += 4 * EPS * np.abs(ref["dq"]) + 1e-30
    e = np.abs(dq - ref["dq"])
    assert np.all(e <= dbound), f"{tag}: dq error {float((e - dbound).max()):.3e} past its bound"
    record_parity(f"{tag}/dq", dq, ref["dq"], rtol=0.0, atol=float(dbound.max()))
    assert np.count_nonzero(dq) <= B * S_on                              # nothing outside the taken action's column
    again = _rows(*args)
    assert all(np.array_equal(a, b) for a, b in zip((losses, dq, prio), again)), "two calls must be bit-identical"


@gpu
def test_rows_kernel_refuses_what_shared_memory_cannot_hold():
    from tianshou_b200._cabi import call, ptr
    x = torch.zeros(16, device=DEV)
    a = torch.zeros(1, dtype=torch.int64, device=DEV)
    for S_on, S_t in ((8, 12289), (2, 100000), (0, 8)):
        with pytest.raises(RuntimeError, match="ts_iqn_rows"):
            call("ts_iqn_rows", ptr(x), ptr(a), ptr(x), ptr(x), None, 1, 1, S_on, S_t, ptr(x), ptr(x), ptr(x), ptr(x), _st())


# ------------------------------------------------------------------------------------------------------------ vs reference
def model_from_cfg(kind, A, C=64, obs=4, hidden=(64,), trunk_out=64, last=(64,), H=44, W=44, scale=True):
    from tianshou_b200.env.atari import DQNet, ScaledObsInputActionReprNet
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.discrete import ImplicitQuantileNetwork
    if kind == "cnn":
        pre = DQNet(c=4, h=H, w=W, action_shape=A, features_only=True)
        pre = ScaledObsInputActionReprNet(pre) if scale else pre
    else:
        pre = Net(state_shape=(obs,), action_shape=trunk_out, hidden_sizes=hidden)
    return ImplicitQuantileNetwork(preprocess_net=pre, action_shape=A, hidden_sizes=last, num_cosines=C).to(DEV)


def build_from_golden(g, mirror_taus=None):
    from tianshou_b200.algorithm import IQN, AdamOptimizerFactory, IQNPolicy
    kind = str(g["cfg_kind"])
    kw = (dict(H=int(g["cfg_H"]), W=int(g["cfg_W"]), scale=bool(g["cfg_scale"])) if kind == "cnn"
          else dict(obs=int(g["cfg_obs"]), hidden=tuple(int(x) for x in g["cfg_hidden"]), trunk_out=int(g["cfg_trunk_out"])))
    A = int(g["cfg_A"])
    model = model_from_cfg(kind, A, int(g["cfg_C"]), last=tuple(int(x) for x in g["cfg_last"]), **kw)
    ods.seeded_params(model, int(g["cfg_init_seed"]))
    policy = IQNPolicy(model=model, action_space=_Discrete(A), sample_size=int(g["cfg_S"]), online_sample_size=int(g["cfg_S_on"]),
                       target_sample_size=int(g["cfg_S_t"]))
    return IQN(policy=policy, optim=AdamOptimizerFactory(lr=float(g["cfg_lr"])), gamma=float(g["cfg_gamma"]),
               n_step_return_horizon=int(g["cfg_n_step"]), target_update_freq=int(g["cfg_freq"]))


def replay_taus(algo, taus):
    """Replace the update's one fraction draw with ``taus`` (device tensors) in order, checking each shape."""
    it = iter(taus)

    def draw(rows, S):
        t = next(it)
        assert tuple(t.shape) == (rows, S), f"draw of {(rows, S)} where the reference drew {tuple(t.shape)}"
        return t

    algo._draw_taus = draw
    return it


def _golden_taus(g):
    n = sum(int(g[f"u{u}_ntaus"]) for u in range(int(g["cfg_updates"])))
    return [dev(g[f"taus_{k}"]) for k in range(n)]


@gpu
@pytest.mark.parametrize("mirror", [False, True])
@pytest.mark.parametrize("variant", VARIANTS)
def test_update_matches_reference_run(variant, mirror):
    """Update after update against the reference's run, on the fractions it drew: the same sampled indices, n-step returns
    over S_t (or, with ``target_update_freq == 0``, S_on) columns, the loss, the priorities written back (PER: and the sum-tree
    leaves), then the final state at the QR-DQN bars (DESIGN.md section 4) and the reference's ``state_dict()`` keys."""
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden(f"{variant}.npz")
    algo, buf = build_from_golden(g), buffer_from_golden(g, mirror)
    keys = [str(k) for k in g["state_dict_keys"]]
    assert list(algo.state_dict().keys()) == keys
    rest = replay_taus(algo, _golden_taus(g))
    cap = {}
    orig_pre, orig_post = algo._preprocess_batch, algo._postprocess_batch

    def pre(batch, buffer, indices):
        b = orig_pre(batch, buffer, indices)
        cap["indices"], cap["returns"] = np.asarray(indices).copy(), b.returns.detach().cpu().numpy().copy()
        return b

    def post(batch, buffer, indices):
        cap["prio"] = batch.weight.detach().cpu().numpy().copy()
        return orig_post(batch, buffer, indices)

    algo._preprocess_batch, algo._postprocess_batch = pre, post
    for u in range(int(g["cfg_updates"])):
        np.random.seed(500 + u)
        with policy_within_training_step(algo.policy):
            stats = algo.update(buffer=buf, sample_size=int(g["cfg_bs"]))
        tag = f"{variant}_m{int(mirror)}_u{u}"
        assert np.array_equal(cap["indices"], g[f"u{u}_indices"]), "sampled indices differ from the reference's"
        ref_ret = g[f"u{u}_returns"]
        record_parity(f"{tag}/returns", cap["returns"], ref_ret, rtol=1e-5, atol=1e-5 * float(np.abs(ref_ret).max()))
        record_parity(f"{tag}/losses", np.array([stats.loss]), g[f"u{u}_losses"], rtol=2e-5, atol=2e-6)
        record_parity(f"{tag}/prio", cap["prio"], g[f"u{u}_prio"], rtol=2e-5, atol=2e-6)
        if bool(g["cfg_per"]):
            leaves = np.asarray(buf.weight[np.arange(len(buf))])
            record_parity(f"{tag}/tree_leaves", leaves, g[f"u{u}_tree_leaves"], rtol=2e-5, atol=1e-7)
    assert next(rest, None) is None, "every fraction the reference drew is used, in order"
    check_final_state(f"{variant}_m{int(mirror)}", g, algo)
    assert list(algo.state_dict().keys()) == keys


def fp64_quantiles(model64, x, taus):
    """q[B, A, S] of a float64 copy of an ImplicitQuantileNetwork on given fractions: the reference's forward
    (discrete.py:205-215) with its ``torch.rand`` replaced by ``taus``."""
    pre = model64.preprocess
    feat = (pre.net if hasattr(pre, "net") else pre.model.model)(x)      # the layer chains: Net / MLP cast their input to fp32
    B, S = taus.shape
    h = (feat.unsqueeze(1) * model64.embed_model(taus)).view(B * S, -1)
    return model64.last.model(h).view(B, S, -1).transpose(1, 2)


@gpu
@pytest.mark.parametrize("kind", ["mlp", "relu_trunk", "cnn"])
def test_update_gradient_vs_fp64_autograd(kind):
    """One update: the flat gradient, snapshotted before its Adam step, against float64 autograd of the reference's loss
    (iqn.py:163-179) on a copy of the module with the same weights, batch, returns and fractions.  Adam's first step is
    lr * sign(g), so a gradient off by a constant factor leaves the parameters unchanged; this is the check that sees it.  The
    GEMMs are fp32-faithful (bf16x3) and a weight gradient sums B * S products per element; the cosine argument is fp32 on the
    device and float64 here (a relative 6e-8 per element): 2e-4 relative plus 1e-4 of the tensor's largest value, as in
    test_qrdqn_gpu."""
    from tianshou_b200.algorithm import IQN, AdamOptimizerFactory, IQNPolicy
    from tianshou_b200.algorithm.flat_params import FlatGroup
    from tianshou_b200.utils import policy_within_training_step
    torch.manual_seed(3)
    rng = np.random.default_rng(4)
    A, B = 5, 64
    if kind == "cnn":
        model = model_from_cfg("cnn", A, C=33, last=(48,))
    else:
        model = model_from_cfg("mlp", A, C=33, hidden=(48,), trunk_out=40 if kind == "mlp" else 0, last=(40,))
    policy = IQNPolicy(model=model, action_space=_Discrete(A), online_sample_size=6, target_sample_size=7)
    algo = IQN(policy=policy, optim=AdamOptimizerFactory(lr=1e-3), gamma=0.9, n_step_return_horizon=2, target_update_freq=3)
    assert algo._trunk_act == (1 if kind == "relu_trunk" else 0)
    buf = make_buffer(kind, A, rng)
    cap = {}
    grp = algo._group

    def adam(optimizer, mgn):
        cap["grad"] = grp.grad[: grp.n].clone()
        FlatGroup.adam_step(grp, optimizer, mgn)

    grp.adam_step = adam
    draws = []
    orig_draw = algo._draw_taus

    def draw(rows, S):
        draws.append(orig_draw(rows, S))
        return draws[-1]

    algo._draw_taus = draw
    orig_pre = algo._preprocess_batch

    def pre(batch, buffer, indices):
        b = orig_pre(batch, buffer, indices)
        cap["indices"], cap["returns"] = np.asarray(indices).copy(), b.returns.detach().cpu().double()
        return b

    algo._preprocess_batch = pre
    ref = copy.deepcopy(model).to("cpu", torch.float64)         # the weights before the step
    np.random.seed(7)
    with policy_within_training_step(algo.policy):
        stats = algo.update(buffer=buf, sample_size=B)
    assert len(draws) == 3 and draws[0].shape == (B, 6) and draws[1].shape == (B, 7) and draws[2].shape == (B, 6)
    idx = cap["indices"]
    raw = np.asarray(buf.obs)[idx]
    if kind == "cnn":
        x = torch.as_tensor((raw.astype(np.float64) / 255.0).astype(np.float32)).double()
        ref.preprocess = ref.preprocess.module                  # the scaling done above, as the device's frame reader does
    else:
        x = torch.as_tensor(raw).double()
    q = fp64_quantiles(ref, x, draws[2].cpu().double())
    act = np.asarray(buf.act)[idx].astype(np.int64)
    loss, _ = oi.reference_loss(q, act, cap["returns"], draws[2].cpu().double(), 1.0)
    loss.backward()
    for i, (p, r) in enumerate(zip(grp.params, ref.parameters(), strict=True)):
        want = r.grad.numpy()
        got = grp.view(cap["grad"], p).view(p.shape).cpu().numpy()
        record_parity(f"iqn_grad/{kind}/grad_{i}", got, want, rtol=2e-4, atol=1e-4 * float(np.abs(want).max()) + 1e-12)
    record_parity(f"iqn_grad/{kind}/loss", np.array([stats.loss]), np.array([loss.item()]), rtol=2e-5, atol=2e-6)


# ------------------------------------------------------------------------------------------------------------ repeats, state_dict
def _seeded_draws(seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return lambda rows, S: torch.rand(rows, S, dtype=torch.float32, device=DEV, generator=g)


@gpu
def test_two_updates_from_one_state_agree_bit_for_bit():
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden("iqn_ref_sizes.npz")
    algos = [build_from_golden(g), build_from_golden(g)]
    for a in algos:
        a._draw_taus = _seeded_draws(5)
        buf = buffer_from_golden(g)
        for u in range(2):
            np.random.seed(20 + u)
            with policy_within_training_step(a.policy):
                a.update(buffer=buf, sample_size=int(g["cfg_bs"]))
    a, b = algos
    for ga, gb in ((a._group, b._group), (a._g_old, b._g_old)):
        assert torch.equal(ga.flat, gb.flat) and torch.equal(ga.exp_avg, gb.exp_avg) and torch.equal(ga.exp_avg_sq, gb.exp_avg_sq)


@gpu
@pytest.mark.parametrize("variant", ["iqn_ref_sizes", "iqn_ref_cnn"])
def test_state_dict_round_trip_continues_identically(variant):
    """A fresh algorithm loaded from another's ``state_dict()`` continues bit for bit on the same fractions: online, lagged and
    optimiser state.  ``_iter`` is a plain attribute, as in the reference: whoever restores a run restores it too."""
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden(f"{variant}.npz")
    a, buf_a = build_from_golden(g), buffer_from_golden(g)
    a._draw_taus = _seeded_draws(1)
    for u in range(3):
        np.random.seed(u)
        with policy_within_training_step(a.policy):
            a.update(buffer=buf_a, sample_size=int(g["cfg_bs"]))
    b = build_from_golden(g)
    with torch.no_grad():
        for p in b.policy.parameters():
            p.add_(0.01)
    b.load_state_dict(copy.deepcopy(a.state_dict()))
    b._iter = a._iter
    for algo in (a, b):
        algo._draw_taus = _seeded_draws(2)
        buf = buffer_from_golden(g)
        for u in range(3):
            np.random.seed(10 + u)
            with policy_within_training_step(algo.policy):
                algo.update(buffer=buf, sample_size=int(g["cfg_bs"]))
    pairs = [(a._group, b._group)] + ([(a._g_old, b._g_old)] if a._g_old is not None else [])
    for ga, gb in pairs:
        assert torch.equal(ga.flat, gb.flat) and torch.equal(ga.exp_avg, gb.exp_avg) and torch.equal(ga.exp_avg_sq, gb.exp_avg_sq)
    assert a._group.step == b._group.step


# ------------------------------------------------------------------------------------------------------------ policy
@gpu
def test_policy_sample_sizes_and_arg_max():
    from tianshou_b200.algorithm import IQNPolicy
    from tianshou_b200.data import Batch
    from tianshou_b200.utils.net.discrete import ImplicitQuantileNetwork
    torch.manual_seed(0)
    model = model_from_cfg("mlp", 5, C=17, hidden=(32,), trunk_out=0, last=(24,))
    assert isinstance(model, ImplicitQuantileNetwork)
    policy = IQNPolicy(model=model, action_space=_Discrete(5), sample_size=11, online_sample_size=6, target_sample_size=4)
    obs = np.random.default_rng(0).standard_normal((300, 4)).astype(np.float32)
    batch = Batch(obs=obs, info=Batch())
    policy.train()
    out = policy(batch)
    assert out.logits.shape == (300, 5, 6) and out.taus.shape == (300, 6)
    assert np.array_equal(out.act, out.logits.mean(2).argmax(1).cpu().numpy())
    old = copy.deepcopy(model)
    assert policy(batch, model=old).logits.shape == (300, 5, 4)
    policy.eval()
    out = policy(batch)
    assert out.logits.shape == (300, 5, 11) and out.taus.shape == (300, 11)
    assert np.array_equal(out.act, out.logits.mean(2).argmax(1).cpu().numpy())
    torch.manual_seed(9)
    (logits, taus), _ = model(obs, sample_size=11)
    torch.manual_seed(9)
    again = policy(batch)
    assert torch.equal(again.logits, logits) and torch.equal(again.taus, taus)
    for kw in (dict(sample_size=1), dict(online_sample_size=1), dict(target_sample_size=1)):
        with pytest.raises(AssertionError, match="should be greater than 1"):
            IQNPolicy(model=model, action_space=_Discrete(5), **kw)


# ------------------------------------------------------------------------------------------------------------ refusals
@gpu
def test_refusals():
    from torch import nn

    from tianshou_b200.algorithm import IQN, QRDQN, AdamOptimizerFactory, IQNPolicy, RMSpropOptimizerFactory, UnsupportedModelError
    from tianshou_b200.data import Batch, VectorReplayBuffer
    from tianshou_b200.utils import policy_within_training_step
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.discrete import ImplicitQuantileNetwork
    A = 3

    def make(model=None, opt=AdamOptimizerFactory, n=A, **kw):
        model = model or model_from_cfg("mlp", A, C=8, hidden=(16,), trunk_out=16, last=(16,))
        return IQN(policy=IQNPolicy(model=model, action_space=_Discrete(n)), optim=opt(lr=1e-3), **kw)

    algo = make()
    assert isinstance(algo, QRDQN)

    class Opaque(nn.Module):
        def __init__(self):
            super().__init__()
            self.w = nn.Parameter(torch.zeros(4))

        def get_output_dim(self):
            return 4

    with pytest.raises(UnsupportedModelError, match="model: "):
        make(ImplicitQuantileNetwork(preprocess_net=Opaque(), action_shape=A).to(DEV))
    soft = Net(state_shape=(4,), action_shape=16, hidden_sizes=(16,), softmax=True)
    with pytest.raises(UnsupportedModelError, match="softmax"):
        make(ImplicitQuantileNetwork(preprocess_net=soft, action_shape=A, num_cosines=8).to(DEV))
    with pytest.raises(UnsupportedModelError, match="outputs, not 4 actions"):
        make(n=4)
    bad = model_from_cfg("mlp", A, C=8, hidden=(16,), trunk_out=16, last=(16,))
    bad.last = nn.Sequential(nn.Linear(16, A), nn.ReLU()).to(DEV)
    with pytest.raises(UnsupportedModelError, match="must end in a linear layer over the actions"):
        make(bad)
    with pytest.raises(UnsupportedModelError, match="ImplicitQuantileNetwork|DiscreteCritic"):
        make(Net(state_shape=(4,), action_shape=A, hidden_sizes=(16,)).to(DEV))
    with pytest.raises(UnsupportedModelError, match="Adam"):
        make(opt=RMSpropOptimizerFactory)
    with pytest.raises(UnsupportedModelError, match="no CPU path"):
        make(model_from_cfg("mlp", A, C=8, hidden=(16,), trunk_out=16, last=(16,)).cpu())
    for kw in (dict(gamma=1.5), dict(n_step_return_horizon=0), dict(num_quantiles=1)):
        with pytest.raises(AssertionError):
            make(**kw)
    # an action the network has no quantiles for is refused on the host, before any kernel indexes with it
    buf = VectorReplayBuffer(40, 4, device=DEV)
    rng = np.random.default_rng(0)
    for _ in range(8):
        buf.add(Batch(obs=rng.standard_normal((4, 4)).astype(np.float32), act=np.array([0, 1, 2, A]), rew=np.zeros(4),
                      terminated=np.zeros(4, bool), truncated=np.zeros(4, bool), obs_next=rng.standard_normal((4, 4)).astype(np.float32)),
                buffer_ids=np.arange(4))
    with pytest.raises(ValueError, match="actions in"), policy_within_training_step(algo.policy):
        algo.update(buffer=buf, sample_size=32)


# ------------------------------------------------------------------------------------------------------------ resources
def _register_report(src, tmp_path):
    from tianshou_b200.csrc import build as B
    if shutil.which(B.NVCC) is None and not os.path.exists(B.NVCC):
        pytest.skip("nvcc not available")
    r = subprocess.run([B.NVCC, *B.FLAGS, "-c", os.path.join(B.HERE, src), "-o", str(tmp_path / "k.o")], capture_output=True,
                       text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    return re.findall(r"Compiling entry function '(\S+)' for 'sm_90a'\n(?:.*\n)*?\s*(\d+) bytes stack frame, (\d+) bytes spill "
                      r"stores, (\d+) bytes spill loads", r.stdout + r.stderr)


def test_kernels_have_no_stack_frame_or_spills(tmp_path):
    hits = _register_report("iqn.cu", tmp_path)
    kernels = ("iqn_cos_kernel", "iqn_mix_kernel", "iqn_mix_backward_kernel", "iqn_target_kernel", "iqn_rows_kernel",
               "row_sums3_kernel")
    assert len(hits) == len(kernels) and all(any(k in h[0] for h in hits) for k in kernels), hits
    assert all(tuple(map(int, h[1:])) == (0, 0, 0) for h in hits), hits
    hits = _register_report("qrdqn.cu", tmp_path)
    assert len(hits) == 3 and all(tuple(map(int, h[1:])) == (0, 0, 0) for h in hits), hits
