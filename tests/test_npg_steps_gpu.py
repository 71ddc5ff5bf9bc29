"""The NPG / TRPO vector kernels of csrc/npg.cu, on their own at their edges and inside ``NPG.update`` / ``TRPO.update``.

Direct tests drive ``ts_npg_mean_rows``, ``ts_npg_normalize_adv``, ``ts_npg_axpy``, ``ts_trpo_step_size`` and
``ts_trpo_decide`` across the row counts where a one-block kernel's strided loop starts or stops taking a second iteration
(1023, 1024, 1025 rows), past the axpy grid's cap, at 10^6 rows, and through every branch of the line-search decision,
including the strict comparisons at exactly the threshold and a NaN KL.

The update tests wrap the C ABI inside npg.py / trpo.py, snapshot what each of these kernels (and ``ts_cg_step``) reads
just before it runs and what it wrote just after, and check every call against float64 from that captured state.  Nothing
is compared across calls, so no bar grows with the iteration, minibatch or candidate index.  The matrix work is checked on
float64 CPU copies of oracle/oracle_npg.py's modules loaded from the captured flat buffers: the surrogate rows and the
vanilla gradient at the minibatch's actor, F p before every CG step and F x before the TRPO step size
(``oracle_npg.fisher_product``), the KL and surrogate rows at every candidate, and around every critic optimiser step the
MSE gradient, the vf-loss column and one float64 Adam / RMSprop step from the kernel's own moments and step count.

Bars (fp32 unit roundoff u = 2^-24, one fp32 ulp of x at most 2^-23 |x|):
  * means of rows: the kernel sums in float64 in a fixed order and rounds once, so within 1 ulp of fl32(fp64 mean);
  * normalisation: fl32(mean) and fl32(std) each carry u relative, the subtraction and the division one rounding each:
    |err| <= u (|mean| / std + 3 |ref|) (1 + 2^-20);
  * axpy ``theta + c dir``: the compiler may fuse it into one FMA or round twice: within 1 ulp of |theta| + |c dir|;
  * TRPO step size ``sqrt(2 max_kl / (s . (z + damping s)))``: fl32(2 max_kl), the fp32 damped product, the cast of the fp64
    dot product and the division each add u relative under the square root, which halves them, and sqrtf rounds once:
    3u relative, inside 2 ulp; the damped product only stays within u of the dot product when its terms do not cancel,
    which every input here ensures (z = s * positive) or which the update's positive-definite F p gives up to the
    condition number Sum |s (z + damping s)| / s . (z + damping s), folded into the bar;
  * one CG iteration from the kernel's own x, r, p, r.r and z = F p: fp32 vector updates with fp64 dot products, each vector
    element within 2 ulp of its fp32 terms plus the alpha (beta) relative error times its |alpha p| (|beta p|) term, where
    alpha's relative error is u (cast) + u times the condition number of p . (z + damping p);
  * every line-search decision must equal the float64 decision on the kernel's own rows (the kernel compares the fp32
    roundings of those means, so only a margin within one ulp of the mean could flip it) and every CG convergence test
    the float64 test on the kernel's own r; a margin within 2 ulp (decisions) or 8 ulp (residual) of its threshold is
    refused as an input, never skipped; the step shrink is bitwise fl32(step * fl32(backtrack_coeff)).
"""
import math
import warnings

import numpy as np
import pytest
import torch

from ts_testutil import Box, load_golden, record_parity, restore_vector_buffer, synth_rollout

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
U = 2.0 ** -24
ULP = 2.0 ** -23
STRIDE = 8
SENTINEL = np.float32(7.25)
EPS32 = float(np.finfo(np.float32).eps)
# the bar of the three-product weight-gradient MMAs (tests/test_npg_gpu.py FVP test), for every quantity that passes
# through the forward, tangent or backward GEMMs: rows at the captured parameters, the gradients, F v
FVP_RTOL, FVP_ATOL = 2e-4, 1e-4


def _cabi():
    from tianshou_b200 import _cabi as c
    return c


def call(name, *args):
    _cabi().call(name, *args)


def ptr(t):
    return _cabi().ptr(t)


def stream():
    return _cabi().stream_ptr(torch.device(DEV))


def dev(a, dtype=None):
    t = torch.as_tensor(np.ascontiguousarray(a), device=DEV)
    return t if dtype is None else t.to(dtype)


def spacing32(x):
    return np.spacing(np.abs(np.asarray(x, dtype=np.float32))).astype(np.float64)


def mean64(rows):
    return math.fsum(np.asarray(rows, dtype=np.float64).tolist()) / len(rows)


def check_mean(key, got, rows):
    """``got`` within 1 ulp of the fp32 rounding of the fp64 mean of ``rows``; an inf row (a categorical KL where a new
    probability underflows to 0, as torch's kl_divergence gives) makes the mean inf."""
    ref = np.float32(mean64(rows))
    if not np.isfinite(ref):
        assert np.array_equal(np.float32(got), ref, equal_nan=True), (key, float(got), float(ref))
        return
    assert abs(float(got) - float(ref)) <= float(spacing32(ref)), (key, float(got), float(ref))
    record_parity(key, [got], [float(ref)], rtol=0.0, atol=float(spacing32(ref)))


# ====================================================================================================== direct tests
@pytest.mark.parametrize("B", [1, 1023, 1024, 1025, 10 ** 6 + 3])
def test_mean_rows_vs_fp64(B):
    rng = np.random.default_rng(B)
    rows = (0.7 + 3.0 * rng.standard_normal(B)).astype(np.float32)
    rows[rng.random(B) < 0.01] *= 1e4
    d = dev(rows)
    outs = [torch.full((2,), float("nan"), device=DEV) for _ in range(2)]
    for o in outs:
        call("ts_npg_mean_rows", ptr(d), B, ptr(o), stream())
    got = [o.cpu().numpy() for o in outs]
    check_mean(f"ts_npg_mean_rows B={B}", got[0][0], rows)
    assert np.isnan(got[0][1]), "wrote past its one output"
    assert got[0][:1].view(np.uint32) == got[1][:1].view(np.uint32), "two calls differ"


def normalize_ref(a):
    a = a.astype(np.float64)
    mean = mean64(a)
    std = math.sqrt(math.fsum(((a - mean) ** 2).tolist()) / (len(a) - 1))
    return (a - mean) / std, mean, std


@pytest.mark.parametrize("n", [2, 1024, 1025, 10 ** 6 + 3])
def test_normalize_adv_vs_fp64(n):
    rng = np.random.default_rng(n)
    adv = (5.0 + 2.0 * rng.standard_normal(n)).astype(np.float32)
    d = dev(adv)
    call("ts_npg_normalize_adv", ptr(d), n, stream())
    ref, mean, std = normalize_ref(adv)
    tol = U * (abs(mean) / std + 3.0 * np.abs(ref)) * (1 + 2.0 ** -20)
    record_parity(f"ts_npg_normalize_adv n={n}", d.cpu().numpy(), ref, rtol=0.0, atol=float(tol.max()))
    assert np.all(np.abs(d.cpu().numpy() - ref) <= tol)


def test_normalize_adv_constant_is_nan_and_one_row_is_refused():
    """Constant advantages: std 0 and 0 / 0, NaN as torch's ``(adv - mean) / std`` gives.  One row has no unbiased std."""
    adv = np.full(1500, 3.0, dtype=np.float32)
    d = dev(adv)
    call("ts_npg_normalize_adv", ptr(d), len(adv), stream())
    t = torch.as_tensor(adv)
    assert torch.isnan((t - t.mean()) / t.std()).all()
    assert torch.isnan(d).all()
    with pytest.raises(RuntimeError, match="at least two rows"):
        call("ts_npg_normalize_adv", ptr(dev(adv[:1])), 1, stream())


def axpy_cap():
    return torch.cuda.get_device_properties(0).multi_processor_count * 8 * 256


@pytest.mark.parametrize("scaled", [False, True], ids=["coef", "scale_on_device"])
@pytest.mark.parametrize("n", ["1", "1000", "past_grid"])
def test_axpy_vs_fp64(n, scaled):
    """out = theta + c dir with c = coef, or fl32(*scale * fl32(coef)) from a device scalar; negative coef as the natural step
    and the line search use; past the grid's cap every thread takes more than one element.  Nothing past n is written."""
    n = {"1": 1, "1000": 1000, "past_grid": axpy_cap() * 3 + 77}[n]
    rng = np.random.default_rng(n)
    theta = rng.standard_normal(n).astype(np.float32)
    d = (rng.standard_normal(n) * 10.0 ** rng.uniform(-3, 2, n)).astype(np.float32)
    coef, scale = (-1.0, 0.3719) if scaled else (-0.5, None)
    c = np.float32(np.float32(scale) * np.float32(coef)) if scaled else np.float32(coef)
    out = torch.full((n + 16,), float(SENTINEL), device=DEV)
    sc = dev(np.array([scale], dtype=np.float32)) if scaled else None
    d_theta, d_dir = dev(theta), dev(d)            # held: a freed temporary's block would be handed to the next one
    call("ts_npg_axpy", ptr(out), ptr(d_theta), ptr(d_dir), coef, ptr(sc), n, stream())
    got = out.cpu().numpy()
    ref = theta.astype(np.float64) + float(c) * d.astype(np.float64)
    tol = spacing32(np.abs(theta.astype(np.float64)) + np.abs(float(c) * d.astype(np.float64)))
    assert np.all(np.abs(got[:n] - ref) <= tol)
    record_parity(f"ts_npg_axpy {'scaled' if scaled else 'coef'}", got[:n], ref, rtol=0.0, atol=float(tol.max()))
    assert np.all(got[n:] == SENTINEL)


def step_size_ref(s, z, damping, max_kl):
    s64, z64 = s.astype(np.float64), z.astype(np.float64)
    terms = s64 * (z64 + float(np.float32(damping)) * s64)
    d = math.fsum(terms.tolist())
    return math.sqrt(2.0 * max_kl / d), math.fsum(np.abs(terms).tolist()) / d


def run_step_size(s, z, damping, max_kl):
    step = torch.full((1,), float("nan"), device=DEV)
    row = torch.full((STRIDE,), float(SENTINEL), device=DEV)
    d_s, d_z = dev(s), dev(z)
    call("ts_trpo_step_size", ptr(d_s), ptr(d_z), len(s), damping, max_kl, ptr(step), ptr(row), stream())
    return float(step.item()), row.cpu().numpy()


def step_size_tol(ref, cond):
    return (2 * ULP + 0.5 * U * (cond - 1.0)) * ref


@pytest.mark.parametrize("max_kl", [0.01, 2.0])
@pytest.mark.parametrize("n", [1, 1023, 1025, 10 ** 6])
def test_trpo_step_size_vs_fp64(n, max_kl):
    """``sqrt(2 max_kl / (s . (z + 0.1 s)))`` with z = s * positive (no cancellation in the dot product); the row gets kl = 0,
    step size = step, accepted index = -1 and failed = 0 (columns 2, 3, 5, 6), and no other column changes."""
    rng = np.random.default_rng(n)
    s = rng.standard_normal(n).astype(np.float32)
    z = (s * rng.uniform(0.01, 3.0, n)).astype(np.float32)
    got, row = run_step_size(s, z, 0.1, max_kl)
    ref, cond = step_size_ref(s, z, 0.1, max_kl)
    tol = step_size_tol(ref, cond)
    record_parity(f"ts_trpo_step_size max_kl={max_kl}", [got], [ref], rtol=0.0, atol=tol)
    assert row[2] == 0.0 and row[3] == np.float32(got) and row[5] == -1.0 and row[6] == 0.0
    assert np.all(row[[0, 1, 4, 7]] == SENTINEL)


def decide_ref(loss_rows, kl_rows, i, max_backtracks, max_kl, coeff, step, actor_loss):
    """trpo.py:170-186 in float64 on the kernel's rows: (flag, step after, expected row, (kl margin, loss margin), (kl,
    new loss))."""
    kl, new_loss = mean64(kl_rows), mean64(loss_rows)
    mk = float(np.float32(max_kl))
    row = np.full(STRIDE, SENTINEL, dtype=np.float32)
    row[0] = actor_loss
    row[2] = np.float32(kl)
    if kl < mk and new_loss < actor_loss:
        flag = 1
        row[3], row[5] = step, i
    elif i < max_backtracks - 1:
        flag = 0
        step = np.float32(np.float32(step) * np.float32(coeff))
    else:
        flag = 2
        row[3], row[6] = 0.0, 1.0
    return flag, np.float32(step), row, (kl - mk, new_loss - float(actor_loss)), (kl, new_loss)


def run_decide(loss_rows, kl_rows, i, max_backtracks, max_kl, coeff, step, actor_loss):
    d_step = dev(np.array([step], dtype=np.float32))
    row = np.full(STRIDE, SENTINEL, dtype=np.float32)
    row[0] = actor_loss
    d_row = dev(row)
    flag = torch.full((1,), -5, dtype=torch.int32, device=DEV)
    d_loss, d_kl = dev(loss_rows), dev(kl_rows)
    call("ts_trpo_decide", ptr(d_loss), ptr(d_kl), len(loss_rows), i, max_backtracks, max_kl, coeff, ptr(d_step),
         ptr(d_row), ptr(flag), stream())
    return int(flag.item()), np.float32(d_step.item()), d_row.cpu().numpy()


def rows_with_mean(rng, B, mean, spread):
    """fp32 rows whose fp64 mean lies near ``mean``; B = 1 is the single value."""
    r = (mean + spread * rng.standard_normal(B)).astype(np.float32)
    return r


DECIDE_CASES = {   # name: (i, max_backtracks, kl rows mean, loss rows mean relative to actor loss, expected flag)
    "accepted": (3, 10, 0.5, -0.5, 1),
    "accepted_first": (0, 10, 0.5, -0.5, 1),
    "rejected_for_kl": (0, 10, 1.5, -0.5, 0),
    "rejected_for_loss": (2, 10, 0.5, 0.5, 0),
    "failed_last": (9, 10, 0.5, 0.5, 2),
    "failed_for_kl_last": (9, 10, 1.5, -0.5, 2),
    "single_accepted": (0, 1, 0.5, -0.5, 1),
    "single_failed": (0, 1, 1.5, -0.5, 2),
}


@pytest.mark.parametrize("B", [1, 1025, 10 ** 6])
@pytest.mark.parametrize("case", list(DECIDE_CASES))
def test_trpo_decide_branches(case, B):
    """Every branch of the decision on rows whose means sit well away from the thresholds: the flag, the step (kept,
    shrunk bitwise, or kept on failure), and the stats row (kl always; step size and accepted index on acceptance; step
    size 0 and failed 1 on failure; nothing else)."""
    i, maxb, kl_rel, loss_rel, flag_ref = DECIDE_CASES[case]
    rng = np.random.default_rng(B + 13 * len(case))
    max_kl, coeff, step, actor_loss = 0.01, 0.8, np.float32(0.731), np.float32(-0.25)
    kl_rows = np.abs(rows_with_mean(rng, B, kl_rel * max_kl, 0.2 * max_kl if B > 1 else 0.0))
    loss_rows = rows_with_mean(rng, B, float(actor_loss) + loss_rel * 0.5, 0.3 if B > 1 else 0.0)
    got = run_decide(loss_rows, kl_rows, i, maxb, max_kl, coeff, step, actor_loss)
    ref = decide_ref(loss_rows, kl_rows, i, maxb, max_kl, coeff, step, actor_loss)
    assert ref[0] == flag_ref, "the case's inputs do not produce its branch"
    assert got[0] == ref[0]
    assert got[1].view(np.uint32) == ref[1].view(np.uint32)
    check_mean(f"ts_trpo_decide kl B={B}", got[2][2], kl_rows)
    row_ref = ref[2].copy()
    row_ref[2] = got[2][2]
    assert np.array_equal(got[2].view(np.uint32), row_ref.view(np.uint32)), (got[2], row_ref)


@pytest.mark.parametrize("B", [1, 1025, 10 ** 6])
def test_trpo_decide_strict_comparisons_and_nan(B):
    """The reference compares ``kl < max_kl`` and ``new_loss < loss`` strictly: a KL mean exactly fl32(max_kl) and a new
    loss exactly the actor loss are both rejected (constant rows of an fp32 value: every fp64 partial sum is exact); a
    NaN KL is rejected as well, and fails the search on the last candidate."""
    max_kl, coeff, step, actor_loss = 0.01, 0.8, np.float32(0.5), np.float32(-0.125)
    mk = np.float32(max_kl)
    good_kl = np.full(B, np.float32(0.25 * max_kl))
    good_loss = np.full(B, np.float32(actor_loss - 1.0))
    for name, kl_rows, loss_rows in [("kl == max_kl", np.full(B, mk), good_loss),
                                     ("loss == actor loss", good_kl, np.full(B, actor_loss)),
                                     ("nan kl", np.where(np.arange(B) == B // 2, np.float32(np.nan), good_kl), good_loss)]:
        for i, maxb, flag_ref in [(0, 3, 0), (2, 3, 2)]:
            flag, st, row = run_decide(loss_rows.astype(np.float32), kl_rows.astype(np.float32), i, maxb, max_kl, coeff, step,
                                       actor_loss)
            assert flag == flag_ref, (name, i, flag)
            if flag_ref == 0:
                assert st == np.float32(step * np.float32(coeff)), name
            else:
                assert st == step and row[3] == 0.0 and row[6] == 1.0, name
            assert row[5] == SENTINEL, name
            if name == "kl == max_kl":
                assert row[2] == mk
            if name == "nan kl":
                assert np.isnan(row[2])
    # and one step inside each threshold is accepted
    flag, _, _ = run_decide(np.full(B, np.nextafter(actor_loss, np.float32(-1))).astype(np.float32),
                            np.full(B, np.nextafter(mk, np.float32(0))).astype(np.float32), 0, 3, max_kl, coeff, step, actor_loss)
    assert flag == 1


# ====================================================================================================== inside update()
class Capture:
    """Wraps ``call`` / ``ptr`` of npg.py and trpo.py: records every tensor whose pointer the update passes, and around each
    call of a checked kernel synchronises and snapshots what it reads before and what it wrote after."""

    def __init__(self, algo, real_call, real_ptr):
        self.algo, self.real_call, self.real_ptr = algo, real_call, real_ptr
        self.tensors = {}
        self.stats = None
        self.pending = None          # parameters the actor must hold at the next call (after a decision / NPG's step)
        self.arm_npg_step = False
        self.counts = {}
        self.decisions = []          # (flag, i, kl margin, loss margin, kl finite)
        L = algo._layered
        self.L, self.categorical = L, bool(L.categorical)
        from tianshou_b200.algorithm import TRPO
        self.trpo = isinstance(algo, TRPO)
        self.actor, self.critic = algo.policy.actor, algo.critic
        self.hp = None

    # ---------------------------------------------------------------------------------------------- fp64 modules
    def modules64(self, flat, group, module, build):
        """A float64 CPU copy (oracle_npg's module ``build()``) of ``module`` with the parameters of the flat buffer ``flat``."""
        m = build().double()
        for p, q in zip(module.parameters(), m.parameters(), strict=True):
            assert p.shape == q.shape
            o = group.offset(p)
            q.data = torch.as_tensor(flat[o:o + p.numel()], dtype=torch.float64).reshape(q.shape).clone()
        return m

    def actor64(self, flat):
        from oracle import oracle_npg as on
        act = torch.nn.ReLU if self.categorical else torch.nn.Tanh
        fam = self.family
        return self.modules64(flat, self.L.group, self.actor, lambda: on.Actor(fam[1], fam[2], fam[3], act, self.categorical))

    def critic64(self, flat):
        from oracle import oracle_npg as on
        act = torch.nn.ReLU if self.categorical else torch.nn.Tanh
        fam = self.family
        return self.modules64(flat, self.L.critic_group, self.critic, lambda: on.critic_net(fam[1], fam[3], act))

    def head64(self, a64):
        return a64.head(a64.trunk(self.mb["obs"]))

    def logp64(self, a64):
        """Row log-probabilities at ``a64``: Categorical clamps its probabilities at float32's eps, as the fp32 rows do (a
        float64 Categorical clamps at 2.2e-16 and would disagree on saturated rows)."""
        h = self.head64(a64)
        if self.categorical:
            return torch.softmax(h, -1).clamp(EPS32, 1 - EPS32).log().gather(1, self.mb["act"].reshape(-1).long()[:, None])[:, 0]
        sigma = a64.sigma_param.reshape(-1).exp().expand_as(h)
        return torch.distributions.Normal(h, sigma).log_prob(self.mb["act"]).sum(-1)

    def rows64(self, a64, ratio):
        lp = self.logp64(a64)
        return -(((lp - self.mb["lpo"]).exp() if ratio else lp) * self.mb["adv"])

    def minibatch(self, orig):
        """Records the minibatch's rows (float64, CPU) and its statistics row, then runs it."""
        def f(batch, idx, row):
            torch.cuda.synchronize()
            i = idx.cpu()
            get = lambda t: t.detach().cpu()[i].double()                       # noqa: E731
            self.mb = {"obs": get(batch.obs), "act": batch.act.detach().cpu()[i] if self.categorical else get(batch.act),
                       "adv": get(batch.adv), "ret": get(batch.returns), "lpo": get(batch.logp_old), "row": row}
            self.mb["theta"] = self.L.group.flat.cpu().numpy().copy()
            self.mb["a64"] = self.actor64(self.mb["theta"])
            return orig(batch, idx, row)
        return f

    def critic_step(self, orig):
        """Around each critic optimiser step: the MSE gradient against float64 autograd at the captured critic, the step
        against one float64 Adam / RMSprop step from the kernel's own moments and step count, the vf-loss column."""
        def f(optimizer, max_grad_norm):
            from tianshou_b200._cabi import OPT_RMSPROP
            from tianshou_b200.algorithm.flat_params import optimizer_hyperparams
            cg = self.L.critic_group
            torch.cuda.synchronize()
            n = cg.n
            p0, g, m0, v0 = (t[:n].double().cpu().numpy() for t in (cg.flat, cg.grad, cg.exp_avg, cg.exp_avg_sq))
            step0 = cg.sync_step_from_device()
            c64 = self.critic64(cg.flat.cpu().numpy())
            loss = torch.nn.functional.mse_loss(self.mb["ret"], c64(self.mb["obs"]).flatten())
            ref_g = torch.cat([t.reshape(-1) for t in torch.autograd.grad(loss, list(c64.parameters()))]).numpy()
            record_parity("update/critic mse gradient", g, ref_g, rtol=2e-4, atol=1e-4 * float(np.abs(ref_g).max()))
            vf = float(self.mb["row"][1].item())
            record_parity("update/vf loss column", [vf], [float(loss)], rtol=2e-4, atol=0.0)
            orig(optimizer, max_grad_norm)
            torch.cuda.synchronize()
            p1, m1, v1 = (t[:n].double().cpu().numpy() for t in (cg.flat, cg.exp_avg, cg.exp_avg_sq))
            step1 = cg.sync_step_from_device()
            assert step1 == step0 + 1
            hp = optimizer_hyperparams(optimizer)
            assert hp["weight_decay"] == 0.0
            e = 4.0 * U                                 # a few fp32 roundings of each term (the epoch-step test's bars)
            b2 = hp["beta2"]                            # RMSprop: alpha
            record_parity("update/critic exp_avg_sq", v1, b2 * v0 + (1 - b2) * g * g, rtol=0.0,
                          atol=float((e * (b2 * v0 + (1 - b2) * g * g)).max()) + 1e-30)
            if hp["optimizer"] == OPT_RMSPROP:
                assert np.array_equal(m1, m0), "RMSprop must leave exp_avg untouched"
                delta = hp["lr"] * g / (np.sqrt(v1) + hp["adam_eps"])
            else:
                b1 = hp["beta1"]
                record_parity("update/critic exp_avg", m1, b1 * m0 + (1 - b1) * g, rtol=0.0,
                              atol=float((e * (b1 * np.abs(m0) + (1 - b1) * np.abs(g))).max()) + 1e-30)
                delta = hp["lr"] / (1.0 - b1 ** step1) * m1 / (np.sqrt(v1) / np.sqrt(1.0 - b2 ** step1) + hp["adam_eps"])
            bar = 8 * 2 * U * np.abs(delta) + 2 * 2 * U * np.abs(p0) + 1e-30
            assert np.all(np.abs(p1 - (p0 - delta)) <= bar), "critic step"
            record_parity(f"update/critic {'rmsprop' if hp['optimizer'] == OPT_RMSPROP else 'adam'} step", p1, p0 - delta,
                          rtol=0.0, atol=float(bar.max()))
            self.counts["critic_step"] = self.counts.get("critic_step", 0) + 1
        return f

    def ptr(self, t):
        p = self.real_ptr(t)
        if t is not None:
            self.tensors[p] = t
        return p

    def alloc_stats(self, orig):
        def f(rows):
            self.stats = orig(rows)
            return self.stats
        return f

    def view(self, addr, n):
        """The n elements at device address ``addr``: a recorded tensor, or a column of the statistics table."""
        if self.stats is not None and 0 <= addr - self.stats.data_ptr() < 4 * self.stats.numel():
            off = (addr - self.stats.data_ptr()) // 4
            return self.stats.reshape(-1)[off:off + n]
        assert addr in self.tensors, "pointer of an unknown buffer"
        return self.tensors[addr].reshape(-1)[:n]

    def snap(self, addr, n):
        return self.view(addr, n).detach().cpu().numpy().copy()

    def __call__(self, name, *a):
        check = getattr(self, "_" + name, None)
        if self.pending is not None:
            flat = self.algo._layered.group.flat.cpu().numpy()
            assert np.array_equal(flat.view(np.uint32), self.pending.view(np.uint32)), "line search left the wrong parameters"
            self.pending = None
        if check is None:
            return self.real_call(name, *a)
        torch.cuda.synchronize()
        after = check(*a)
        self.real_call(name, *a)
        torch.cuda.synchronize()
        after()
        self.counts[name] = self.counts.get(name, 0) + 1

    # ---------------------------------------------------------------------------------------------- kernels
    def _ts_npg_rows(self, head, logstd, act, adv, lpo, B, A, cat, ratio, loss_rows, dhead, dls, st):
        """Surrogate rows at the minibatch's actor (with the gradient) or at a TRPO candidate (rows only) vs float64."""
        a64 = self.mb["a64"] if dhead is not None else self.actor64(self.cand)

        def after():
            ref = self.rows64(a64, ratio).detach().numpy()
            record_parity(f"update/ts_npg_rows {'actor' if dhead is not None else 'candidate'}", self.snap(loss_rows, B), ref,
                          rtol=FVP_RTOL, atol=FVP_ATOL * float(np.abs(ref).max()))
        return after

    def _ts_cg_init(self, g, x, r, p, n, state, st):
        """The vanilla gradient (rows -> mean -> backward GEMMs, log-std column sums) vs float64 autograd."""
        got = self.snap(g, n)
        a64 = self.mb["a64"]
        ref = torch.cat([t.reshape(-1) for t in torch.autograd.grad(self.rows64(a64, self.trpo).mean(),
                                                                     list(a64.parameters()))]).numpy()
        record_parity("update/vanilla gradient", got, ref, rtol=FVP_RTOL, atol=FVP_ATOL * float(np.abs(ref).max()))
        return lambda: None

    def fvp_check(self, key, v, fv):
        from oracle import oracle_npg as on
        ref = on.fisher_product(self.mb["a64"], self.mb["obs"], torch.as_tensor(v, dtype=torch.float64)).numpy()
        record_parity(key, fv, ref, rtol=FVP_RTOL, atol=FVP_ATOL * float(np.abs(ref).max()))

    def _ts_npg_kl_rows(self, head_old, logstd_old, head_new, logstd_new, B, A, cat, kl_rows, st):
        """KL(old || candidate) rows vs float64 at the captured actor and candidate; an inf row (torch's rule where a new
        probability is 0) must be inf in torch's fp32 kl_divergence of the same heads too."""
        a_new = self.actor64(self.cand)

        def after():
            got = self.snap(kl_rows, B).astype(np.float64)
            ho, hn = self.head64(self.mb["a64"]), self.head64(a_new)
            if self.categorical:
                po = torch.softmax(ho, -1)
                lg = lambda h: torch.softmax(h, -1).clamp(EPS32, 1 - EPS32).log()              # noqa: E731
                ref = (po * (lg(ho) - lg(hn))).sum(-1).detach().numpy()
                inf = np.isinf(got)
                if inf.any():
                    C = torch.distributions.Categorical
                    k32 = torch.distributions.kl_divergence(C(probs=torch.softmax(ho.float(), -1)), C(probs=torch.softmax(hn.float(), -1)))
                    assert np.isinf(k32.detach().numpy()[inf]).all(), "inf KL row where torch's fp32 KL is finite"
                got, ref = got[~inf], ref[~inf]
            else:
                N = lambda a, h: torch.distributions.Normal(h, a.sigma_param.reshape(-1).exp().expand_as(h))   # noqa: E731
                ref = torch.distributions.kl_divergence(N(self.mb["a64"], ho), N(a_new, hn)).sum(-1).detach().numpy()
            record_parity("update/ts_npg_kl_rows candidate", got, ref, rtol=FVP_RTOL, atol=FVP_ATOL * float(np.abs(ref).max()))
            if not self.trpo:
                self.arm_npg_step = True                  # the next mean is the kl column, then g.flat <- cand
        return after

    def _ts_npg_normalize_adv(self, adv, n, st):
        before = self.snap(adv, n)

        def after():
            ref, mean, std = normalize_ref(before)
            tol = U * (abs(mean) / std + 3.0 * np.abs(ref)) * (1 + 2.0 ** -20)
            got = self.snap(adv, n)
            assert np.all(np.abs(got - ref) <= tol)
            record_parity("update/ts_npg_normalize_adv", got, ref, rtol=0.0, atol=float(tol.max()))
        return after

    def _ts_npg_mean_rows(self, rows, B, out, st):
        before = self.snap(rows, B)

        def after():
            check_mean("update/ts_npg_mean_rows", self.snap(out, 1)[0], before)
            if self.arm_npg_step:                       # NPG: the natural step is taken after this call
                self.arm_npg_step, self.pending = False, self.cand
        return after

    def _ts_cg_step(self, x, r, p, z, n, damping, tol, state, iters_out, st):
        x0, r0, p0, z0 = (self.snap(v, n).astype(np.float64) for v in (x, r, p, z))
        s0 = self.snap(state, 3)
        if s0[1] == 0.0:
            self.fvp_check("update/F p before ts_cg_step", p0, z0)      # z = F p at the kernel's own p

        def after():
            x1, r1, p1 = (self.snap(v, n).astype(np.float64) for v in (x, r, p))
            s1 = self.snap(state, 3)
            assert self.snap(iters_out, 1)[0] == s1[2], "the CG-iterations column"
            if s0[1] != 0.0:                             # converged earlier: a no-op
                assert np.array_equal(x1, x0) and np.array_equal(r1, r0) and np.array_equal(p1, p0)
                assert np.array_equal(s1, s0)
                return
            zd = z0 + float(np.float32(damping)) * p0
            terms = p0 * zd
            pz = math.fsum(terms.tolist())
            cond = math.fsum(np.abs(terms).tolist()) / pz
            alpha = s0[0] / pz
            da = U + U * cond                            # relative error of the kernel's fp32 alpha
            ap, az = np.abs(alpha * p0), np.abs(alpha * zd)
            for what, got, ref, bar in [
                    ("x", x1, x0 + alpha * p0, 2 * ULP * (np.abs(x0) + ap) + da * ap),
                    ("r", r1, r0 - alpha * zd, 2 * ULP * (np.abs(r0) + az) + da * az + U * az)]:
                assert np.all(np.abs(got - ref) <= bar), f"cg {what}"
                record_parity(f"update/ts_cg_step {what}", got, ref, rtol=0.0, atol=float(bar.max()))
            rr = math.fsum((r1 * r1).tolist())          # the residual of the kernel's own r
            assert abs(rr - tol) > 8 * ULP * tol, "residual within fp32 noise of the tolerance: choose other inputs"
            assert s1[2] == s0[2] + 1.0
            if rr < tol:
                assert s1[1] == 1.0 and np.array_equal(p1, p0), "converged: p keeps its value"
            else:
                assert s1[1] == 0.0
                # the kernel's fixed-order fp64 sum of positive terms: n / 1024 in-thread additions, then the tree
                assert abs(s1[0] - rr) <= (n / 1024 + 12) * 2.0 ** -52 * rr
                beta = rr / s0[0]
                bp = np.abs(beta * p0)
                tolp = 2 * ULP * (np.abs(r1) + bp) + U * bp
                assert np.all(np.abs(p1 - (r1 + beta * p0)) <= tolp), "cg p"
                record_parity("update/ts_cg_step p", p1, r1 + beta * p0, rtol=0.0, atol=float(tolp.max()))
        return after

    def _ts_trpo_step_size(self, s, z, n, damping, max_kl, step, row, st):
        s0, z0 = self.snap(s, n), self.snap(z, n)
        self.fvp_check("update/F x before ts_trpo_step_size", s0.astype(np.float64), z0.astype(np.float64))

        def after():
            got = float(self.snap(step, 1)[0])
            ref, cond = step_size_ref(s0, z0, damping, max_kl)
            record_parity("update/ts_trpo_step_size", [got], [ref], rtol=0.0, atol=step_size_tol(ref, cond))
            r = self.snap(row, STRIDE)
            assert r[2] == 0.0 and r[3] == np.float32(got) and r[5] == -1.0 and r[6] == 0.0
        return after

    def _ts_npg_axpy(self, out, theta, d, coef, scale, n, st):
        th, dd = self.snap(theta, n).astype(np.float64), self.snap(d, n).astype(np.float64)
        c = np.float32(coef) if scale is None else np.float32(self.snap(scale, 1)[0] * np.float32(coef))
        self.theta = th.astype(np.float32)

        def after():
            got = self.snap(out, n)
            ref = th + float(c) * dd
            tol = spacing32(np.abs(th) + np.abs(float(c) * dd))
            assert np.all(np.abs(got - ref) <= tol), "candidate"
            record_parity("update/ts_npg_axpy", got, ref, rtol=0.0, atol=float(tol.max()))
            self.cand = got.copy()
        return after

    def _ts_trpo_decide(self, loss_rows, kl_rows, B, i, maxb, max_kl, coeff, step, row, flag, st):
        lr, kr = self.snap(loss_rows, B), self.snap(kl_rows, B)
        st0, row0 = self.snap(step, 1)[0], self.snap(row, STRIDE)

        def after():
            fl, st1, row1 = int(self.snap(flag, 1)[0]), self.snap(step, 1)[0], self.snap(row, STRIDE)
            ref_flag, ref_step, _, (mkl, mloss), (kl, new_loss) = decide_ref(lr, kr, i, maxb, max_kl, coeff, st0, row0[0])
            # the kernel compares fl32 of these fp64 means: its decision can differ only within one ulp of the threshold
            assert (not np.isfinite(kl) or abs(mkl) > 2 * spacing32(kl)) and abs(mloss) > 2 * spacing32(new_loss), \
                "decision within fp32 noise of its threshold: choose other inputs"
            check_mean("update/ts_trpo_decide kl", row1[2], kr)
            assert fl == ref_flag, (fl, ref_flag, mkl, mloss)
            assert st1.view(np.uint32) == ref_step.view(np.uint32)
            if fl == 1:
                assert row1[3] == st0 and row1[5] == i and row1[6] == 0.0
                self.pending = self.cand
            elif fl == 2:
                assert row1[3] == 0.0 and row1[6] == 1.0 and row1[5] == -1.0
                self.pending = self.theta
            self.decisions.append((fl, i, mkl, mloss, bool(np.isfinite(kl))))
        return after


def _algo(cls, family, lr=1e-3, **kw):
    from tianshou_b200.algorithm import (AdamOptimizerFactory, DiscreteActorPolicy, ProbabilisticActorPolicy,
                                         RMSpropOptimizerFactory)
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.continuous import ContinuousActorProbabilistic, ContinuousCritic
    from tianshou_b200.utils.net.discrete import DiscreteActor, DiscreteCritic
    categorical, O, A, hidden, act = family
    torch.manual_seed(O + A)
    net_a = Net(state_shape=(O,), hidden_sizes=hidden, activation=act)
    net_c = Net(state_shape=(O,), hidden_sizes=hidden, activation=act)
    if categorical:
        from test_ppo_discrete_gpu import Discrete
        actor, critic = DiscreteActor(preprocess_net=net_a, action_shape=(A,)).to(DEV), DiscreteCritic(preprocess_net=net_c).to(DEV)
        policy = DiscreteActorPolicy(actor=actor, dist_fn=torch.distributions.Categorical, action_space=Discrete(A))
    else:
        actor = ContinuousActorProbabilistic(preprocess_net=net_a, action_shape=(A,), unbounded=True).to(DEV)
        critic = ContinuousCritic(preprocess_net=net_c).to(DEV)
        from test_npg_gpu import _gaussian_dist
        policy = ProbabilisticActorPolicy(actor=actor, dist_fn=_gaussian_dist, action_scaling=True, action_bound_method="clip",
                                          action_space=Box(A))
    from test_npg_gpu import _perturb
    _perturb(actor, O, A)
    optim = RMSpropOptimizerFactory(lr=lr) if kw.pop("rmsprop", False) else AdamOptimizerFactory(lr=lr)
    return cls(policy=policy, critic=critic, optim=optim, **kw)


def _buffer(family, N, seed, saturate):
    from tianshou_b200.data import Batch, VectorReplayBuffer
    categorical, O, A = family[:3]
    E = 1
    rng = np.random.default_rng(seed)
    buf = VectorReplayBuffer(N, E, device=DEV)
    for t, s in enumerate(synth_rollout(rng, E, N, O, A, p_term=0.01, trunc_len=300)):
        if categorical:
            s["act"] = rng.integers(0, A, E)
        if saturate and t % 17 == 0:
            s["obs"] = s["obs"] * np.float32(40.0)
        s["rew"] = s["rew"] + 0.5 * np.sin(0.01 * t)
        buf.add(Batch(**s), buffer_ids=np.arange(E))
    return buf


GAUSS_SMALL = (False, 17, 6, (64, 64), torch.nn.Tanh)
CAT = (True, 8, 5, (64, 64), torch.nn.ReLU)
GAUSS_WIDE = (False, 376, 17, (256, 256), torch.nn.Tanh)
FAMILIES = {"gauss17": GAUSS_SMALL, "cat8": CAT, "gauss376": GAUSS_WIDE}

# name: (family, rows, batch size, repeat, keyword arguments)
NPG_CASES = {
    "gauss17_1024": ("gauss17", 1024, None, 1, dict(advantage_normalization=True)),
    "cat8_1025_scaled": ("cat8", 1025, None, 1, dict(advantage_normalization=False, return_scaling=True)),
    "gauss376_4099": ("gauss376", 4099, None, 1, dict(rmsprop=True)),
    "gauss17_minibatched": ("gauss17", 4099, 1000, 2, dict(return_scaling=True)),
}
TRPO_CASES = {
    "gauss17_1025_kl0.01": ("gauss17", 1025, None, 1, dict(max_kl=0.01)),
    "cat8_4099_kl2_bt1": ("cat8", 4099, None, 1, dict(max_kl=2.0, max_backtracks=1, advantage_normalization=False)),
    "gauss376_1024_kl2": ("gauss376", 1024, None, 1, dict(max_kl=2.0, return_scaling=True)),
    "gauss17_minibatched_bt1": ("gauss17", 4099, 1000, 2, dict(max_kl=0.01, max_backtracks=1)),
    "cat8_minibatched_kl0.01": ("cat8", 4099, 1000, 2, dict(max_kl=0.01, return_scaling=True)),
    "gauss376_4099_kl2_bt10": ("gauss376", 4099, None, 1, dict(max_kl=2.0, max_backtracks=10, advantage_normalization=False)),
    "gauss17_1025_kl2": ("gauss17", 1025, None, 1, dict(max_kl=2.0)),
    "gauss17_2049_kl2_two_minibatches": ("gauss17", 2049, 1024, 1, dict(max_kl=2.0)),
    # the reference's own rollouts on which its line search rejects candidates for the loss alone (11 -> (64, 64) -> 3)
    "golden_trpo_ref_backtrack": ("golden", "trpo_ref_backtrack"),
    "golden_trpo_ref_fail": ("golden", "trpo_ref_fail"),
}


def _run(cls, case, monkeypatch):
    """One ``update()`` of a synthetic case, or the two updates of a reference golden (``("golden", variant)``: the
    reference's own rollouts, parameters and minibatch orders), under a Capture."""
    from tianshou_b200.algorithm.modelfree import npg as npg_mod
    from tianshou_b200.algorithm.modelfree import trpo as trpo_mod
    from tianshou_b200.data.batch import minibatch_bounds
    from tianshou_b200.utils import policy_within_training_step
    if case[0] == "golden":
        from test_npg_gpu import _golden_algo
        g = load_golden(f"{case[1]}.npz")
        algo, _, _ = _golden_algo(g)
        family = (bool(g["cfg_categorical"]), int(g["cfg_obs"]), int(g["cfg_act"]), (64, 64))
        E, N, bs = int(g["cfg_E"]), int(g["u0_adv"].shape[0]), int(g["cfg_bs"])
        bs, repeat, kw = (None if bs < 0 else bs), int(g["cfg_repeat"]), {}
        runs = [(restore_vector_buffer(g, f"u{u}_", E, int(g["cfg_cap"]), device=DEV), int(g[f"u{u}_np_seed"])) for u in range(2)]
    else:
        fam, N, bs, repeat, kw = case
        algo = _algo(cls, FAMILIES[fam], **dict(kw))
        family = FAMILIES[fam][:4]
        runs = [(_buffer(FAMILIES[fam], N, N, saturate=fam == "cat8"), N)]
    cap = Capture(algo, npg_mod.call, npg_mod.ptr)
    cap.family = family
    monkeypatch.setattr(algo, "_minibatch", cap.minibatch(algo._minibatch))
    cg = algo._layered.critic_group
    monkeypatch.setattr(cg, "optimizer_step", cap.critic_step(cg.optimizer_step))
    for mod in (npg_mod, trpo_mod):
        monkeypatch.setattr(mod, "call", cap)
        monkeypatch.setattr(mod, "ptr", cap.ptr)
    monkeypatch.setattr(algo, "_alloc_stats", cap.alloc_stats(algo._alloc_stats))
    for buf, seed in runs:
        np.random.seed(seed)
        with warnings.catch_warnings(), policy_within_training_step(algo.policy):
            warnings.simplefilter("ignore")
            algo.update(buffer=buf, batch_size=bs, repeat=repeat)
    n_mb = repeat * len(minibatch_bounds(N, bs or N, merge_last=True))
    table = algo.last_stats_table
    assert table.shape[0] == n_mb
    assert cap.counts["ts_cg_step"] == 10 * n_mb * len(runs)
    assert cap.counts["ts_cg_init"] == n_mb * len(runs)
    assert cap.counts["critic_step"] == algo.optim_critic_iters * n_mb * len(runs)
    return cap, table, kw


@pytest.mark.parametrize("name", list(NPG_CASES))
def test_npg_update_every_vector_kernel_call_vs_fp64(name, monkeypatch):
    from tianshou_b200.algorithm import NPG
    cap, table, kw = _run(NPG, NPG_CASES[name], monkeypatch)
    n_mb = table.shape[0]
    assert cap.counts["ts_npg_mean_rows"] == 2 * n_mb                  # actor loss, kl
    assert cap.counts["ts_npg_axpy"] == n_mb
    assert cap.counts.get("ts_npg_normalize_adv", 0) == int(kw.get("advantage_normalization", True))


def test_trpo_update_every_vector_kernel_call_and_decision_vs_fp64(monkeypatch):
    """All TRPO cases in one test, because the coverage of the line search is asserted across them: the float64 decisions
    include a candidate rejected for kl >= max_kl, one rejected for the loss alone, one accepted at i > 0 and a failed
    search."""
    from tianshou_b200.algorithm import TRPO
    seen = []
    for name, case in TRPO_CASES.items():
        cap, table, kw = _run(TRPO, case, monkeypatch)
        n_mb = table.shape[0] * (2 if case[0] == "golden" else 1)
        assert cap.counts["ts_trpo_step_size"] == n_mb
        assert cap.counts["ts_trpo_decide"] == cap.counts["ts_npg_axpy"] == len(cap.decisions)
        seen += [(name, *d) for d in cap.decisions]
        monkeypatch.undo()
    kinds = {"rejected for a finite kl >= max_kl": [s for s in seen if s[1] != 1 and s[3] >= 0 and s[5]],
             "rejected for the loss alone": [s for s in seen if s[1] != 1 and s[3] < 0 and s[4] >= 0],
             "accepted at i > 0": [s for s in seen if s[1] == 1 and s[2] > 0],
             "failed": [s for s in seen if s[1] == 2]}
    for k, v in kinds.items():
        assert v, f"no line-search decision {k} across the TRPO cases: (case, flag, i, kl margin, loss margin, finite) {seen}"
