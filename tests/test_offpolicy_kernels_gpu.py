"""The off-policy loss, optimiser and gather kernels of csrc/net_ops.cu, called one by one through the C ABI and compared
with a plain float64 torch restatement of the reference expression (autograd for the backward kernels).

The inputs are built to reach the branches the end-to-end goldens never take: the [-20, 2] log-sigma clamp on and just
past both bounds, tanh saturation, exact ties in min / argmax, Huber rows on both sides of delta and exactly at it,
weights, and row counts past the grid cap of TS_LAUNCH_1D (16 blocks of 256 threads per SM)."""
import numpy as np
import pytest
import torch

from offpolicy_testutil import DEV, sm_count, stream
from ts_testutil import record_parity

pytestmark = pytest.mark.gpu
F32_EPS = float(np.finfo(np.float32).eps)
SIG_MIN, SIG_MAX = -20.0, 2.0


_LIVE: list = []      # the tensors whose raw pointers the pending call uses: kept alive until it has run


def _call(name, *args):
    from tianshou_b200._cabi import call
    call(name, *args, stream())
    torch.cuda.synchronize()
    _LIVE.clear()


def _p(t):
    """Raw pointer of ``t``; holds a reference so that a temporary (``_p(_d(x))``) is not freed and its memory handed to
    the next argument's allocation before the kernel reads it."""
    from tianshou_b200._cabi import ptr
    _LIVE.append(t)
    return ptr(t)


def _d(a, dtype=None):
    t = torch.as_tensor(np.ascontiguousarray(a))
    return (t if dtype is None else t.to(dtype)).to(DEV).contiguous()


def _nan(*shape):
    return torch.full(shape, float("nan"), dtype=torch.float32, device=DEV)


def _h(t):
    return t.detach().cpu().numpy().astype(np.float64)


# ------------------------------------------------------------------------------------ tanh-squashed Gaussian head
class _Fp32RoundedTanh(torch.autograd.Function):
    """tanh in float64 whose output is rounded to float32 -- the value the reference's fp32 forward hands on -- with
    torch's tanh backward, grad * (1 - y^2), evaluated on that rounded output."""

    @staticmethod
    def forward(ctx, x):
        y = torch.tanh(x).to(torch.float32).to(torch.float64)
        ctx.save_for_backward(y)
        return y

    @staticmethod
    def backward(ctx, g):
        (y,) = ctx.saved_tensors
        return g * (1.0 - y * y)


def _sg_inputs(B, A, seed):
    """head = (mu, raw log-sigma) with raw below, at, inside and above the clamp range; pre-tanh x spread over +-12 (so that
    fp32 tanh reaches +-1 exactly for |x| > 9.01).  Row kinds by b mod 3: 0 'edge' rows whose raw values cycle through
    -25, -20, 2, 3.5 and two interior values; 1 'high' rows whose raw values are all at or above the upper bound (2, 3.5,
    5) with unsaturated x in [-3, 3], where fp32 loses no digits; 2 'regular' rows with raw in [-3, 1.5]."""
    rng = np.random.default_rng(seed)
    raw = rng.uniform(-3.0, 1.5, (B, A))
    edge_rows = (np.arange(B) % 3) == 0
    cycle = np.array([-25.0, -20.0, 2.0, 3.5, -7.5, 0.0])
    raw[edge_rows] = cycle[(np.arange(B)[edge_rows, None] * A + np.arange(A)[None, :]) % len(cycle)]
    raw = raw.astype(np.float32)
    noise = rng.standard_normal((B, A)).astype(np.float32)
    x_target = rng.uniform(-12.0, 12.0, (B, A))
    x_target[:, ::2] = rng.uniform(-3.0, 3.0, (B, (A + 1) // 2))       # half the columns unsaturated
    high_rows = (np.arange(B) % 3) == 1
    raw[high_rows] = np.array([2.0, 3.5, 5.0])[(np.arange(B)[high_rows, None] + np.arange(A)[None, :]) % 3]
    x_target[high_rows] = rng.uniform(-3.0, 3.0, (int(high_rows.sum()), A))
    sigma = np.exp(np.clip(raw.astype(np.float64), SIG_MIN, SIG_MAX))
    mu = (x_target - sigma * noise).astype(np.float32)
    head = np.concatenate([mu, raw], axis=1)
    return head, noise, edge_rows, high_rows


def _sg_forward_torch(head, noise, A, dtype):
    """SACPolicy.forward (sac.py:108-131) + correct_log_prob_gaussian_tanh in ``dtype`` on the CPU."""
    h = torch.as_tensor(head).to(dtype)
    n = torch.as_tensor(noise).to(dtype)
    mu, raw = h[:, :A], h[:, A:]
    sigma = raw.clamp(SIG_MIN, SIG_MAX).exp()
    x = mu + sigma * n
    t = torch.tanh(x)
    logp = torch.distributions.Normal(mu, sigma).log_prob(x).sum(-1) - torch.log(1 - t.pow(2) + F32_EPS).sum(-1)
    return t.numpy().astype(np.float64), logp.numpy().astype(np.float64), sigma.numpy().astype(np.float64)


SG_SHAPES = [(B, A) for B in (1, 255, 257, 4099) for A in (1, 6, 17, 21)]


@pytest.mark.parametrize("B,A", SG_SHAPES, ids=[f"B{b}-A{a}" for b, a in SG_SHAPES])
def test_squashed_gaussian_forward_vs_fp64(B, A):
    """act, logp and sigma against float64.  The bound is 8x torch fp32's own error against float64 plus a floor, taken
    separately over the three row kinds of _sg_inputs: at sigma = e^-20 the fp32 sum mu + sigma * noise rounds to mu, so
    fp32 loses the -noise^2 / 2 of the Normal term in every implementation, and near |t| = 1 log(1 - t^2 + eps) is
    ill-conditioned in t -- that loosens the edge rows' logp bound.  The clamped-high rows (sigma = e^2, unsaturated) lose
    no digits and keep a tight logp bound, so a log-prob bug confined to clamped rows shows there."""
    head, noise, edge, high = _sg_inputs(B, A, seed=B * 31 + A)
    act, logp, sigma = _nan(B, A), _nan(B), _nan(B, A)
    _call("ts_squashed_gaussian", _p(_d(head)), 2 * A, _p(_d(noise)), B, A, SIG_MIN, SIG_MAX, F32_EPS, _p(act), _p(logp), _p(sigma))
    t64, lp64, s64 = _sg_forward_torch(head, noise, A, torch.float64)
    t32, lp32, s32 = _sg_forward_torch(head, noise, A, torch.float32)
    got = dict(act=_h(act), logp=_h(logp), sigma=_h(sigma))
    ref = dict(act=t64, logp=lp64, sigma=s64)
    f32 = dict(act=t32, logp=lp32, sigma=s32)
    for rows, kind in ((~edge & ~high, "regular"), (edge, "edge"), (high, "clamped_high")):
        if not rows.any():
            continue
        for k in ("act", "logp", "sigma"):
            r, g, f = ref[k][rows], got[k][rows], f32[k][rows]
            scale = float(np.abs(r).max())
            # floors: 4 ulp of 1 for tanh, 1e-6 relative for exp / log sums (tanhf / expf / logf are within 2 ulp)
            floor = 3e-7 if k == "act" else 1e-6 * scale
            record_parity(f"offk_sg_fwd/{B}x{A}/{kind}/{k}", g, r, rtol=1e-6 if k == "sigma" else 0.0,
                          atol=8.0 * float(np.abs(f - r).max()) + floor)


@pytest.mark.parametrize("B,A", SG_SHAPES, ids=[f"B{b}-A{a}" for b, a in SG_SHAPES])
def test_squashed_gaussian_bwd_vs_autograd(B, A):
    """dhead = d/d(mu, raw) of  sum(alpha / B * logp) + sum(dact * act)  with a random dact (the critics' input gradient
    is scaled by 1 / B like the log-prob term).

    Yardstick: float64 autograd of the reference expression, with the tanh output rounded to fp32 (_Fp32RoundedTanh) and
    fed to the kernel as its ``act`` input.  Away from saturation that is plain float64 autograd (the rounding moves act by
    one fp32 ulp).  Where 1 - t^2 cancels, the gradient is ill-conditioned in t: at fp32 t = +-1 (|x| > 9.01) the
    reference's fp32 backward gives d act / dx = 0 and d log(1 - t^2 + eps) / dx = 0, while float64 at x = 9.5 still gives
    2 (1 - t^2) / (1 - t^2 + eps) = 0.31.  There the right yardstick is torch's fp32 backward formula on the fp32 output,
    which is what the rounded-output autograd evaluates; the saturated elements are also checked directly against torch
    fp32 autograd (both must be exactly 0 for mu).  The clamp gradient is inclusive at -20 and 2, as in torch.clamp."""
    head, noise, _, _ = _sg_inputs(B, A, seed=B * 17 + A)
    rng = np.random.default_rng(B + 1000 * A)
    alpha = 0.5
    dact = (rng.standard_normal((B, A)) / B).astype(np.float32)
    h64 = torch.as_tensor(head).to(torch.float64).requires_grad_(True)
    n64 = torch.as_tensor(noise).to(torch.float64)
    mu, raw = h64[:, :A], h64[:, A:]
    sig = raw.clamp(SIG_MIN, SIG_MAX).exp()
    x = mu + sig * n64
    t = _Fp32RoundedTanh.apply(x)
    logp = torch.distributions.Normal(mu, sig).log_prob(x).sum(-1) - torch.log(1 - t.pow(2) + F32_EPS).sum(-1)
    (alpha / B * logp.sum() + (torch.as_tensor(dact).to(torch.float64) * t).sum()).backward()
    ref = h64.grad.numpy()
    act_in = t.detach().to(torch.float32).numpy()
    sig_in = sig.detach().to(torch.float32).numpy()
    dhead = _nan(B, 2 * A)
    _call("ts_squashed_gaussian_bwd", _p(_d(head)), 2 * A, _p(_d(noise)), _p(_d(act_in)), _p(_d(sig_in)), _p(_d(dact)), B, A,
          SIG_MIN, SIG_MAX, F32_EPS, alpha / B, _p(dhead))
    got = _h(dhead)
    for cols, name in ((slice(0, A), "dmu"), (slice(A, 2 * A), "draw")):
        r = ref[:, cols]
        # a handful of fp32 roundings per element, some of them in sums of opposite-signed terms: 1e-4 relative plus
        # 1e-4 of the block's largest value (the mutations this must catch move elements by alpha / B ~ 1e-2 of max)
        record_parity(f"offk_sg_bwd/{B}x{A}/{name}", got[:, cols], r, rtol=1e-4, atol=1e-4 * float(np.abs(r).max()))
    raw_np = head[:, A:]
    outside = (raw_np < SIG_MIN) | (raw_np > SIG_MAX)
    assert np.all(got[:, A:][outside] == 0.0), "log-sigma outside [-20, 2] must get no gradient"
    on_bound = (raw_np == SIG_MIN) | (raw_np == SIG_MAX)
    if on_bound.any():
        assert np.all(got[:, A:][on_bound] != 0.0), "the clamp is inclusive: raw = -20 / 2 keeps its gradient"
    # saturated elements vs torch fp32 autograd (CPU): fp32 t = +-1 exactly, so d/dmu is exactly 0 in both
    sat = np.abs(act_in) == 1.0
    if sat.any():
        h32 = torch.as_tensor(head).requires_grad_(True)
        m32, r32 = h32[:, :A], h32[:, A:]
        s32 = r32.clamp(SIG_MIN, SIG_MAX).exp()
        x32 = m32 + s32 * torch.as_tensor(noise)
        t32 = torch.tanh(x32)
        lp32 = torch.distributions.Normal(m32, s32).log_prob(x32).sum(-1) - torch.log(1 - t32.pow(2) + F32_EPS).sum(-1)
        (alpha / B * lp32.sum() + (torch.as_tensor(dact) * t32).sum()).backward()
        sat32 = sat & (t32.detach().abs().numpy() == 1.0)
        assert np.array_equal(got[:, :A][sat32], h32.grad[:, :A].numpy()[sat32].astype(np.float64))
        assert np.all(got[:, :A][sat] == 0.0)


# ------------------------------------------------------------------------------------------------ per-row losses
@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("B", [1, 257, 4099])
def test_critic_mse_vs_autograd(B, weighted):
    """ddpg.py:279-284: td = q - target, loss = mean(td^2 * w); dq vs autograd of the mean (the factor 2 and the 1 / B)."""
    rng = np.random.default_rng(B)
    q = rng.standard_normal(B).astype(np.float32)
    tgt = rng.standard_normal(B).astype(np.float32)
    w = rng.uniform(0.05, 1.0, B).astype(np.float32) if weighted else None
    td, dq, rows = _nan(B), _nan(B), _nan(B)
    _call("ts_critic_mse", _p(_d(q)), _p(_d(tgt)), _p(_d(w)) if weighted else None, B, _p(td), _p(dq), _p(rows))
    q64 = torch.as_tensor(q).to(torch.float64).requires_grad_(True)
    w64 = torch.as_tensor(w).to(torch.float64) if weighted else 1.0
    td64 = q64 - torch.as_tensor(tgt).to(torch.float64)
    rows64 = td64.pow(2) * w64
    rows64.mean().backward()
    tag = f"offk_critic_mse/B{B}_w{int(weighted)}"
    # one to three fp32 roundings per element
    record_parity(tag + "/td", _h(td), td64.detach().numpy(), rtol=2e-7, atol=0.0)
    record_parity(tag + "/dq", _h(dq), q64.grad.numpy(), rtol=1e-6, atol=0.0)
    record_parity(tag + "/loss_rows", _h(rows), rows64.detach().numpy(), rtol=1e-6, atol=0.0)


def _dqn_case(B, A, seed, huber):
    rng = np.random.default_rng(seed)
    q = (np.round(rng.standard_normal((B, A)) * 64) / 64).astype(np.float32)       # multiples of 1/64: exact +-delta rows
    act = rng.integers(0, A, B)
    act[0] = 0
    act[-1] = A - 1
    qs = q[np.arange(B), act].astype(np.float64)
    d = rng.uniform(-3.0, 3.0, B)
    if huber:
        d[1::5], d[2::5] = 1.0, -1.0                     # exactly at +-delta (delta = 1)
        d[3::5] = rng.uniform(-0.99, 0.99, len(d[3::5]))  # quadratic branch
    ret = (qs - d).astype(np.float32)
    return q, act, ret


@pytest.mark.parametrize("A", [1, 2, 18])
@pytest.mark.parametrize("mode", ["mse", "mse_weighted", "huber"])
def test_dqn_loss_vs_autograd(mode, A):
    """dqn.py:384-399: q_sel = q[b, act[b]]; MSE (weighted) or F.huber_loss(q_sel, returns, delta) mean.  dq vs autograd
    w.r.t. the whole Q matrix (zero off the taken action); actions 0 and A - 1 both occur; Huber rows lie on both sides of
    delta = 1 and exactly at +-delta (q and returns are multiples of 1/64, so q_sel - returns = +-1 exactly in fp32)."""
    B = 1031
    q, act, ret = _dqn_case(B, A, seed=A * 7 + len(mode), huber=mode == "huber")
    w = np.random.default_rng(A).uniform(0.05, 1.0, B).astype(np.float32) if mode == "mse_weighted" else None
    delta = 1.0 if mode == "huber" else 0.0
    td, dq, rows = _nan(B), _nan(B, A), _nan(B)
    _call("ts_dqn_loss", _p(_d(q)), _p(_d(act, torch.int64)), _p(_d(ret)), _p(_d(w)) if w is not None else None, B, A, delta,
          _p(td), _p(dq), _p(rows))
    q64 = torch.as_tensor(q).to(torch.float64).requires_grad_(True)
    r64 = torch.as_tensor(ret).to(torch.float64)
    qsel = q64.gather(1, torch.as_tensor(act).view(-1, 1)).view(-1)
    if mode == "huber":
        rows64 = torch.nn.functional.huber_loss(qsel, r64, delta=delta, reduction="none")
    else:
        rows64 = (r64 - qsel).pow(2) * (torch.as_tensor(w).to(torch.float64) if w is not None else 1.0)
    rows64.mean().backward()
    tag = f"offk_dqn_loss/{mode}/A{A}"
    record_parity(tag + "/td", _h(td), (r64 - qsel).detach().numpy(), rtol=2e-7, atol=0.0)
    record_parity(tag + "/dq", _h(dq), q64.grad.numpy(), rtol=1e-6, atol=0.0)
    record_parity(tag + "/loss_rows", _h(rows), rows64.detach().numpy(), rtol=1e-6, atol=0.0)


@pytest.mark.parametrize("is_double", [True, False])
@pytest.mark.parametrize("A", [1, 2, 18])
def test_dqn_target_first_maximum_wins(A, is_double):
    """dqn.py:365-380: double -> q_target[b, argmax_a q_online[b]], vanilla -> max_a q_target[b].  Rows with two or three
    exactly equal maxima at random positions: the first one wins, as in torch.argmax.  Selection only: bit-exact."""
    B = 2053
    rng = np.random.default_rng(A)
    q_on = rng.standard_normal((B, A)).astype(np.float32)
    q_tg = rng.standard_normal((B, A)).astype(np.float32)
    if A > 1:
        for b in range(0, B, 2):
            k = 2 if A == 2 else int(rng.integers(2, 4))
            pos = rng.choice(A, k, replace=False)
            q_on[b, pos] = q_on[b].max() + 0.5
            q_tg[b, pos] = q_tg[b].max() + 0.5 + np.arange(k, dtype=np.float32)   # the vanilla target's ties are values only
    out = _nan(B)
    _call("ts_dqn_target", _p(_d(q_on)), _p(_d(q_tg)), B, A, int(is_double), _p(out))
    if is_double:
        ref = q_tg[np.arange(B), torch.as_tensor(q_on).argmax(dim=1).numpy()]
    else:
        ref = torch.as_tensor(q_tg).max(dim=1).values.numpy()
    got = out.cpu().numpy()
    assert np.array_equal(got, ref), f"{int((got != ref).sum())} rows differ"


@pytest.mark.parametrize("B", [1, 257, 4099])
def test_sac_target_vs_fp64(B):
    """td3.py:94-102 / sac.py:298-302: min(q1, q2) - alpha * logp, with exact ties q1 == q2 in every third row."""
    rng = np.random.default_rng(B)
    q1 = rng.standard_normal(B).astype(np.float32)
    q2 = rng.standard_normal(B).astype(np.float32)
    q2[::3] = q1[::3]
    logp = (rng.standard_normal(B) * 5).astype(np.float32)
    alpha = 0.2
    out = _nan(B)
    _call("ts_sac_target", _p(_d(q1)), _p(_d(q2)), _p(_d(logp)), alpha, B, _p(out))
    ref = np.minimum(q1.astype(np.float64), q2) - np.float64(np.float32(alpha)) * logp
    # two fp32 roundings, the second after a possible cancellation: bounded by the operands' size
    record_parity(f"offk_sac_target/B{B}", _h(out), ref, rtol=2e-7, atol=2e-7 * float(np.abs(q1).max() + alpha * np.abs(logp).max()))


@pytest.mark.parametrize("B", [1, 257, 4099])
def test_sac_actor_q_grad_ties_vs_autograd(B):
    """d mean(alpha * logp - torch.min(q1, q2)) / d(q1, q2): exact ties in every other row (the default SAC config, where
    critic2 is a deep copy of critic, ties in every row) must give each critic half, as torch.minimum's backward does."""
    rng = np.random.default_rng(B + 5)
    q1 = rng.standard_normal(B).astype(np.float32)
    q2 = rng.standard_normal(B).astype(np.float32)
    q2[::2] = q1[::2]
    logp = (rng.standard_normal(B) * 5).astype(np.float32)
    alpha = 0.2
    dq1, dq2, rows = _nan(B), _nan(B), _nan(B)
    _call("ts_sac_actor_q_grad", _p(_d(q1)), _p(_d(q2)), _p(_d(logp)), alpha, B, _p(dq1), _p(dq2), _p(rows))
    a = torch.as_tensor(q1).to(torch.float64).requires_grad_(True)
    c = torch.as_tensor(q2).to(torch.float64).requires_grad_(True)
    rows64 = np.float64(np.float32(alpha)) * torch.as_tensor(logp).to(torch.float64) - torch.min(a, c)
    rows64.mean().backward()
    tag = f"offk_sac_actor_q/B{B}"
    record_parity(tag + "/dq1", _h(dq1), a.grad.numpy(), rtol=1e-7, atol=0.0)        # -1/B rounded once to fp32
    record_parity(tag + "/dq2", _h(dq2), c.grad.numpy(), rtol=1e-7, atol=0.0)
    record_parity(tag + "/loss_rows", _h(rows), rows64.detach().numpy(), rtol=2e-7,
                  atol=2e-7 * float(np.abs(q1).max() + alpha * np.abs(logp).max()))


@pytest.mark.parametrize("n", [1, 1023, 1024, 1025, 1_000_003])
def test_mean_vs_fp64(n):
    """One block of 1024 lanes: each lane sums ceil(n / 1024) values in order, then a 10-level tree.  For non-negative
    values (loss rows) the relative error is at most (ceil(n / 1024) + 10 + 1) * 2^-24."""
    x = np.random.default_rng(n).uniform(0.0, 2.0, n).astype(np.float32)
    out = _nan(1)
    _call("ts_mean", _p(_d(x)), n, _p(out))
    ref = np.array([x.astype(np.float64).sum() / n])
    record_parity(f"offk_mean/n{n}", _h(out), ref, rtol=((n + 1023) // 1024 + 11) * 2.0 ** -24, atol=0.0)


# ------------------------------------------------------------------------------------------------------- Adam
ADAM_CASES = [(0.0, None), (0.1, None), (0.0, 0.5), (0.1, 0.5), (0.1, 1e6)]


@pytest.mark.parametrize("wd,max_norm", ADAM_CASES, ids=[f"wd{w}-clip{m}" for w, m in ADAM_CASES])
@pytest.mark.parametrize("n", [1, 255, 65_537, 300_001])
def test_adam_step_vs_torch_and_device_step_bit_identical(n, wd, max_norm):
    """Five steps of ts_adam_step and of ts_adam_step_dev against clip_grad_norm_ (when max_norm is set; 0.5 clips every
    step, 1e6 never does) followed by torch.optim.Adam(foreach=False) on the same fp32 GPU tensors.  The host-step and
    the device-step variants must agree bit for bit (the CUDA-graph SAC path swaps one for the other).  n = 65,537 and
    300,001 exceed 256 blocks x 256 threads, so the norm's sumsq_kernel runs its grid-stride loop."""
    lr, b1, b2, eps = 1e-3, 0.9, 0.999, 1e-8
    g = torch.Generator(device="cpu").manual_seed(n)
    p0 = torch.randn(n, generator=g)
    grads = [torch.randn(n, generator=g) * (1.0 + k) for k in range(5)]
    p_ref = p0.clone().to(DEV).requires_grad_(True)
    opt = torch.optim.Adam([p_ref], lr=lr, betas=(b1, b2), eps=eps, weight_decay=wd, foreach=False)
    ph, mh, vh = p0.clone().to(DEV), torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    pd, md, vd = p0.clone().to(DEV), torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    scratch_h = torch.zeros(256, dtype=torch.float64, device=DEV)
    scratch_d = torch.zeros(256, dtype=torch.float64, device=DEV)
    step_dev = torch.zeros(1, dtype=torch.int64, device=DEV)
    for k in range(5):
        gk = grads[k].to(DEV)
        p_ref.grad = gk.clone()
        if max_norm is not None:
            torch.nn.utils.clip_grad_norm_([p_ref], max_norm)
        opt.step()
        mn = float(max_norm or 0.0)
        _call("ts_adam_step", _p(ph), _p(gk), _p(mh), _p(vh), n, k + 1, lr, b1, b2, eps, wd, mn, _p(scratch_h))
        _call("ts_adam_step_dev", _p(pd), _p(gk), _p(md), _p(vd), n, _p(step_dev), lr, b1, b2, eps, wd, mn, _p(scratch_d))
        assert torch.equal(ph, pd) and torch.equal(mh, md) and torch.equal(vh, vd), f"step {k + 1}: host / device step differ"
    assert int(step_dev.item()) == 5
    tag = f"offk_adam/n{n}_wd{wd}_clip{max_norm}"
    st = opt.state[p_ref]
    # the same fp32 operation order as torch's single-tensor step; the clip coefficient comes from an fp64 sum of squares
    # (torch: fp32 norms), so it may differ in its last bit: parameters within a few ulp plus 2e-3 of one step, moments
    # 2e-6 relative
    record_parity(tag + "/param", _h(ph), _h(p_ref), rtol=1e-6, atol=2e-3 * lr)
    record_parity(tag + "/exp_avg", _h(mh), _h(st["exp_avg"]), rtol=2e-6, atol=1e-7 * float(st["exp_avg"].abs().max()))
    record_parity(tag + "/exp_avg_sq", _h(vh), _h(st["exp_avg_sq"]), rtol=2e-6, atol=1e-7 * float(st["exp_avg_sq"].abs().max()))


@pytest.mark.parametrize("tau", [0.0, 0.005, 1.0])
def test_polyak_update_bit_exact(tau):
    """utils/lagged_network.py:8-18: tgt = tau * src + (1 - tau) * tgt, two fp32 products and an add, as torch evaluates it."""
    n = 300_001
    g = torch.Generator(device="cpu").manual_seed(3)
    src = torch.randn(n, generator=g).to(DEV)
    tgt = torch.randn(n, generator=g).to(DEV)
    ref = tau * src + (1 - tau) * tgt
    _call("ts_polyak_update", _p(tgt), _p(src), n, tau)
    assert torch.equal(tgt, ref)


# ------------------------------------------------------------------------------------ rows past the launch grid cap
ROW_KERNELS = ["stack_prev", "squashed_gaussian", "squashed_gaussian_bwd", "critic_mse", "dqn_loss", "dqn_target",
               "sac_target", "sac_actor_q_grad"]


@pytest.mark.parametrize("kernel", ROW_KERNELS)
def test_per_row_kernels_write_rows_past_the_grid_cap(kernel):
    """TS_LAUNCH_1D caps the grid at num_sms * 16 blocks of 256 threads.  Each per-row kernel gets 1000 rows (elements, for
    the head backward) more than that, with NaN-prefilled outputs: every row must be written and correct."""
    sms = sm_count()
    n = sms * 16 * 256 + 1000
    rng = np.random.default_rng(7)
    if kernel == "stack_prev":
        out = torch.full((n, 2), -1, dtype=torch.int64, device=DEV)
        idx = torch.arange(n, dtype=torch.int64, device=DEV)
        offset = _d(np.array([0, n], np.int64))
        done = torch.zeros(n, dtype=torch.uint8, device=DEV)
        _call("ts_stack_prev_indices", _p(idx), n, 2, _p(offset), 1, _p(done), _p(_d(np.array([n - 1], np.int64))),
              _p(_d(np.array([n], np.int64))), _p(out))
        ref = torch.stack([(idx - 1).clamp(min=0), idx], dim=1)        # prev(0) = 0: the episode start is its own predecessor
        assert torch.equal(out, ref), f"{int((out != ref).any(1).sum())} rows wrong"
        return
    if kernel in ("squashed_gaussian", "squashed_gaussian_bwd"):
        # unsaturated (|x| < 3): the row count is the point here, not the edges
        head = np.concatenate([rng.uniform(-1, 1, (n, 1)), rng.uniform(-2, -1, (n, 1))], axis=1).astype(np.float32)
        noise = rng.standard_normal((n, 1)).astype(np.float32)
        t64, lp64, s64 = _sg_forward_torch(head, noise, 1, torch.float64)
        if kernel == "squashed_gaussian":
            act, logp, sig = _nan(n, 1), _nan(n), _nan(n, 1)
            _call("ts_squashed_gaussian", _p(_d(head)), 2, _p(_d(noise)), n, 1, SIG_MIN, SIG_MAX, F32_EPS, _p(act), _p(logp), _p(sig))
            record_parity("offk_rows/squashed_gaussian/act", _h(act), t64, rtol=0.0, atol=1e-5)
            record_parity("offk_rows/squashed_gaussian/logp", _h(logp), lp64, rtol=1e-5, atol=1e-5)
            return
        dact = rng.standard_normal((n, 1)).astype(np.float32)
        dhead = _nan(n, 2)
        t_in = t64.astype(np.float32).astype(np.float64)
        _call("ts_squashed_gaussian_bwd", _p(_d(head)), 2, _p(_d(noise)), _p(_d(t_in.astype(np.float32))), _p(_d(s64.astype(np.float32))),
              _p(_d(dact)), n, 1, SIG_MIN, SIG_MAX, F32_EPS, 0.1, _p(dhead))
        one_m = 1 - t_in ** 2
        t64 = t_in
        gx = 0.1 * 2 * t64 * one_m / (one_m + F32_EPS) + dact * one_m
        ref = np.concatenate([gx, (gx * noise - 0.1 / s64) * s64], axis=1)
        record_parity("offk_rows/squashed_gaussian_bwd", _h(dhead), ref, rtol=1e-4, atol=1e-5)
        return
    q1 = rng.standard_normal(n).astype(np.float32)
    q2 = rng.standard_normal(n).astype(np.float32)
    logp = rng.standard_normal(n).astype(np.float32)
    if kernel == "critic_mse":
        td, dq, rows = _nan(n), _nan(n), _nan(n)
        _call("ts_critic_mse", _p(_d(q1)), _p(_d(q2)), None, n, _p(td), _p(dq), _p(rows))
        d = q1.astype(np.float64) - q2
        record_parity("offk_rows/critic_mse/dq", _h(dq), 2 * d / n, rtol=1e-6, atol=0.0)
        record_parity("offk_rows/critic_mse/loss_rows", _h(rows), d * d, rtol=1e-6, atol=0.0)
    elif kernel == "dqn_loss":
        q = np.stack([q1, q2], 1)
        act = rng.integers(0, 2, n)
        td, dq, rows = _nan(n), _nan(n, 2), _nan(n)
        _call("ts_dqn_loss", _p(_d(q)), _p(_d(act, torch.int64)), _p(_d(logp)), None, n, 2, 0.0, _p(td), _p(dq), _p(rows))
        d = logp.astype(np.float64) - q[np.arange(n), act]
        ref = np.zeros((n, 2))
        ref[np.arange(n), act] = -2 * d / n
        record_parity("offk_rows/dqn_loss/dq", _h(dq), ref, rtol=1e-6, atol=0.0)
        record_parity("offk_rows/dqn_loss/td", _h(td), d, rtol=2e-7, atol=0.0)
    elif kernel == "dqn_target":
        out = _nan(n)
        q = np.stack([q1, q2], 1)
        _call("ts_dqn_target", _p(_d(q)), _p(_d(q[:, ::-1])), n, 2, 1, _p(out))
        assert np.array_equal(out.cpu().numpy(), q[:, ::-1][np.arange(n), q.argmax(1)])
    elif kernel == "sac_target":
        out = _nan(n)
        _call("ts_sac_target", _p(_d(q1)), _p(_d(q2)), _p(_d(logp)), 0.2, n, _p(out))
        record_parity("offk_rows/sac_target", _h(out), np.minimum(q1, q2).astype(np.float64) - np.float32(0.2) * logp.astype(np.float64),
                      rtol=1e-6, atol=1e-6)
    else:
        dq1, dq2, rows = _nan(n), _nan(n), _nan(n)
        _call("ts_sac_actor_q_grad", _p(_d(q1)), _p(_d(q2)), _p(_d(logp)), 0.2, n, _p(dq1), _p(dq2), _p(rows))
        g = np.float64(np.float32(-1.0 / n))
        assert np.array_equal(_h(dq1), np.where(q1 < q2, g, 0.0)) and np.array_equal(_h(dq2), np.where(q2 < q1, g, 0.0))
        record_parity("offk_rows/sac_actor_q_grad/loss_rows", _h(rows),
                      np.float32(0.2) * logp.astype(np.float64) - np.minimum(q1, q2), rtol=1e-6, atol=1e-6)
