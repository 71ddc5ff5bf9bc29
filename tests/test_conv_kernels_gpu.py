"""The kernels that connect the layers of a ``FusedStack`` (csrc/net_ops.cu: im2col from uint8 frames and from fp32 NHWC
activations, col2im, the flatten permutes, concat2; csrc/net_gemm.cu: the bias-gradient column sum; csrc/ppo_rows.cu: the
layer-wise loss table), called one by one through the C ABI and compared bit for bit with a numpy restatement of their
documented order, or with an fp64 sum within a stated bound.  Then whole conv stacks through ``compile_sequential`` +
``FusedStack`` and ``DQN.update()`` against fp64 autograd.

The geometries are the ones the square, exactly tiled NatureCNN inputs cannot tell apart: H != W (an exchanged H and W
shows), input rows and columns no window covers (their gradient must be exactly 0), a stride larger than the kernel,
1 x 1 kernels, windows as tall as the input, C in {1, 2, 3, 4, 5}, convolutions without an activation in front of the
next convolution or the flatten, and element counts past the grid cap of TS_LAUNCH_1D (16 blocks of 256 threads per SM)."""
import copy
import functools
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from torch import nn

from ts_testutil import record_parity

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
U = 2.0 ** -24                 # unit roundoff of fp32


_LIVE: list = []      # the tensors whose raw pointers the pending call uses: kept alive until it has run


def _call(name, *args):
    from tianshou_b200._cabi import call, stream_ptr
    call(name, *args, stream_ptr(torch.device(DEV)))
    torch.cuda.synchronize()
    _LIVE.clear()


def _p(t):
    from tianshou_b200._cabi import ptr
    _LIVE.append(t)
    return ptr(t)


def _d(a):
    return torch.as_tensor(np.ascontiguousarray(a)).to(DEV).contiguous()


def _dn(a):
    """``_d`` for arrays that may be empty: the entry points want non-null pointers even when nothing is read."""
    return _d(a) if np.asarray(a).size else torch.zeros(1, device=DEV)


def _h(t):
    return t.detach().cpu().numpy()


@functools.cache
def _grid_cap() -> int:
    """Threads of the largest grid TS_LAUNCH_1D launches: 16 blocks of 256 threads per SM."""
    return torch.cuda.get_device_properties(DEV).multi_processor_count * 16 * 256


def _bits(a) -> np.ndarray:
    return np.ascontiguousarray(np.asarray(a, dtype=np.float32)).view(np.int32)


def _exact(key, got, ref):
    """Bit-exact comparison (``-0.0`` and ``+0.0`` differ), recorded with a zero bar."""
    got, ref = np.asarray(got, np.float32), np.asarray(ref, np.float32)
    assert got.shape == ref.shape, (key, got.shape, ref.shape)
    diff = _bits(got) != _bits(ref)
    assert not diff.any(), f"{key}: {int(diff.sum())} of {diff.size} elements differ, first at {np.argwhere(diff)[0].tolist()}"
    record_parity(key, got, ref, rtol=0.0, atol=0.0)


def _bounded(key, got, ref, bound):
    """``|got - ref| <= bound`` element by element; recorded with the largest element of the bound as its atol and the
    largest err / bound as ``max_err_over_bound``."""
    got, ref, bound = (np.asarray(a, np.float64) for a in (got, ref, bound))
    err = np.abs(got - ref)
    use = float((err / np.maximum(bound, 1e-300)).max()) if err.size else 0.0
    assert not (err > bound).any(), f"{key}: {int((err > bound).sum())} elements past the bound, worst err / bound {use:.3e}"
    e = record_parity(key, got, ref, rtol=0.0, atol=float(bound.max()) if bound.size else 0.0)
    e["max_err_over_bound"] = use
    return e


def _out_hw(H, W, k, s):
    return (H - k) // s + 1, (W - k) // s + 1


# (C, H, W, k, s): none of them square and exactly tiled at once
GEOMS = [
    (4, 38, 22, 8, 4),        # H > W, 2 rows and 2 columns uncovered
    (3, 17, 29, 4, 2),        # H < W, the last row and column uncovered
    (1, 84, 84, 8, 4),        # single-frame DQNet conv 1: K = 64
    (5, 23, 19, 2, 3),        # stride > kernel: every third row / column never read; 2 trailing columns uncovered
    (4, 5, 7, 1, 1),          # 1 x 1
    (3, 9, 6, 1, 2),          # 1 x 1, stride 2: odd rows and columns never read
    (1, 12, 9, 3, 3),         # k == s
    (4, 8, 13, 8, 4),         # window as tall as the input: Ho = 1, one column uncovered
]
GEOM_IDS = [f"C{c}-{h}x{w}-k{k}s{s}" for c, h, w, k, s in GEOMS]


def _batch(kind, per_sample):
    """B for a batch kind: 1, 3, or just past the grid cap given the elements one sample spreads over."""
    return {"B1": 1, "B3": 3, "cap": _grid_cap() // per_sample + 3}[kind]


def _windows(x_nchw, k, s):
    """[B, C, H, W] -> [B * Ho * Wo, C * k * k] in torch's weight order (c, kh, kw) -- numpy gather."""
    B, C = x_nchw.shape[:2]
    v = np.lib.stride_tricks.sliding_window_view(x_nchw, (k, k), axis=(2, 3))[:, :, ::s, ::s]   # [B, C, Ho, Wo, k, k]
    Ho, Wo = v.shape[2], v.shape[3]
    return np.ascontiguousarray(v.transpose(0, 2, 3, 1, 4, 5)).reshape(B * Ho * Wo, C * k * k)


def _stack_idx(rng, B, C, S):
    """Frame slots per sample with repeated slots inside a sample and across samples, slots out of order and the last
    slot of the storage."""
    idx = rng.integers(0, S, (B, C))
    idx[0, :] = S - 1
    if B > 1:
        idx[1, :] = np.arange(C)[::-1] + S - 1 - C          # descending
    if B > 2:
        idx[2, :] = idx[0, 0]                               # the same slot as sample 0
    return idx.astype(np.int64)


# ------------------------------------------------------------------------------------------------------ im2col (u8)
DENOMS = [255.0, 4.0, 3.0, 1.0, 2.2]


@pytest.mark.parametrize("denom", DENOMS)
@pytest.mark.parametrize("bk", ["B1", "B3", "cap"])
@pytest.mark.parametrize("C,H,W,k,s", GEOMS, ids=GEOM_IDS)
def test_im2col_u8_vs_numpy_gather(C, H, W, k, s, bk, denom):
    """``ts_im2col_u8`` bit-exact against a numpy gather of the stacked frames followed by the reference's scaling,
    fp32(v / denom) with the division in float64."""
    Ho, Wo = _out_hw(H, W, k, s)
    B = _batch(bk, Ho * Wo * C * k * k)
    rng = np.random.default_rng(C * 1000 + H * 10 + W + k + s + B)
    S = B * C + 4
    frames = rng.integers(0, 256, (S, H, W), dtype=np.uint8)
    sidx = _stack_idx(rng, B, C, S)
    col = torch.full((B * Ho * Wo, C * k * k), float("nan"), device=DEV)
    _call("ts_im2col_u8", _p(_d(frames)), _p(_d(sidx)), B, C, H, W, k, s, float(denom), _p(col))
    ref = (_windows(frames[sidx], k, s).astype(np.float64) / denom).astype(np.float32)
    if bk == "cap":
        assert col.numel() > _grid_cap()
    _exact(f"conv_kernels/im2col_u8/C{C}_{H}x{W}_k{k}s{s}/{bk}/d{denom}", _h(col), ref)


@pytest.mark.parametrize("denom", DENOMS)
def test_im2col_u8_value_table(denom):
    """Every byte value through the value table (a 1 x 1 gather of a frame holding 0 .. 255): fp32(v / denom) with the
    division in float64, as numpy computes ``obs / denom`` before the cast.  For 2.2 an fp32 division gives other bits,
    so this case tells the two apart."""
    frames = np.arange(256, dtype=np.uint8).reshape(1, 16, 16)
    col = torch.full((256, 1), float("nan"), device=DEV)
    _call("ts_im2col_u8", _p(_d(frames)), _p(_d(np.zeros((1, 1), np.int64))), 1, 1, 16, 16, 1, 1, float(denom), _p(col))
    v = np.arange(256)
    ref = (v.astype(np.float64) / denom).astype(np.float32)
    _exact(f"conv_kernels/im2col_u8/table/d{denom}", _h(col).reshape(-1), ref)
    f32_div = v.astype(np.float32) / np.float32(denom)
    assert (_bits(f32_div) != _bits(ref)).any() == (denom == 2.2)


# ----------------------------------------------------------------------------------------------------- im2col (f32)
def _nhwc_input(rng, B, H, W, C):
    x = rng.standard_normal((B, H, W, C)).astype(np.float32)
    x.reshape(-1)[::7] = -0.0
    return x


@pytest.mark.parametrize("bk", ["B1", "B3", "cap"])
@pytest.mark.parametrize("C,H,W,k,s", GEOMS, ids=GEOM_IDS)
def test_im2col_f32_vs_unfold(C, H, W, k, s, bk):
    """``ts_im2col_f32`` of an NHWC tensor bit-exact against ``F.unfold`` of the same tensor permuted to NCHW (a pure
    copy: -0.0 must stay -0.0)."""
    Ho, Wo = _out_hw(H, W, k, s)
    B = _batch(bk, Ho * Wo * C * k * k)
    rng = np.random.default_rng(C + H * 7 + W * 3 + k * 11 + s + B)
    x = _nhwc_input(rng, B, H, W, C)
    col = torch.full((B * Ho * Wo, C * k * k), float("nan"), device=DEV)
    _call("ts_im2col_f32", _p(_d(x)), B, C, H, W, k, s, _p(col))
    u = F.unfold(torch.from_numpy(x).permute(0, 3, 1, 2).contiguous(), k, stride=s)       # [B, C k k, Ho Wo]
    ref = u.transpose(1, 2).reshape(B * Ho * Wo, C * k * k).numpy()
    if bk == "cap":
        assert col.numel() > _grid_cap()
    _exact(f"conv_kernels/im2col_f32/C{C}_{H}x{W}_k{k}s{s}/{bk}", _h(col), ref)


# ------------------------------------------------------------------------------------------------------------ col2im
def _col2im_ref32(dcol, B, C, H, W, k, s):
    """The kernel's fp32 sum restated: each input pixel starts from +0.0f and adds the window elements that cover it in
    (kh, kw) ascending order."""
    Ho, Wo = _out_hw(H, W, k, s)
    d = dcol.reshape(B, Ho, Wo, C, k, k)
    dx = np.zeros((B, H, W, C), np.float32)
    for kh in range(k):
        for kw in range(k):
            dx[:, kh:kh + s * (Ho - 1) + 1:s, kw:kw + s * (Wo - 1) + 1:s, :] += d[:, :, :, :, kh, kw]
    return dx


def _fold64(dcol, B, C, H, W, k, s):
    """F.fold in float64 -> NHWC."""
    Ho, Wo = _out_hw(H, W, k, s)
    t = torch.from_numpy(np.asarray(dcol, np.float64)).reshape(B, Ho * Wo, C * k * k).transpose(1, 2)
    return F.fold(t, (H, W), k, stride=s).permute(0, 2, 3, 1).numpy()


def _mask_values(rng, shape):
    """ReLU-mask sources: positives, +0.0, -0.0 and negatives in equal shares (only > 0 passes)."""
    pick = rng.integers(0, 4, shape)
    v = np.abs(rng.standard_normal(shape)).astype(np.float32) + np.float32(1e-3)
    return np.where(pick == 0, v, np.where(pick == 1, np.float32(0.0), np.where(pick == 2, np.float32(-0.0), -v))).astype(np.float32)


@pytest.mark.parametrize("masked", [False, True], ids=["nomask", "relu"])
@pytest.mark.parametrize("bk", ["B1", "B3", "cap"])
@pytest.mark.parametrize("C,H,W,k,s", GEOMS, ids=GEOM_IDS)
def test_col2im_f32_vs_fp32_restatement_and_fp64_fold(C, H, W, k, s, bk, masked):
    """``ts_col2im_f32``: bit-exact against the fp32 restatement of its (kh, kw)-ascending order; within
    (covering windows) x 2^-24 x sum |terms| of an fp64 ``F.fold``; pixels no window covers exactly +0.0; with a
    ``relu_src`` only pixels whose source is > 0 (not +0.0, not -0.0) pass."""
    Ho, Wo = _out_hw(H, W, k, s)
    B = _batch(bk, H * W * C)
    rng = np.random.default_rng(C * 3 + H + W * 5 + k + s * 13 + B + int(masked))
    dcol = rng.standard_normal((B * Ho * Wo, C * k * k)).astype(np.float32)
    src = _mask_values(rng, (B, H, W, C)) if masked else None
    dx = torch.full((B, H, W, C), float("nan"), device=DEV)
    _call("ts_col2im_f32", _p(_d(dcol)), B, C, H, W, k, s, _p(_d(src)) if masked else None, _p(dx))
    got = _h(dx)
    if bk == "cap":
        assert dx.numel() > _grid_cap()
    keep = (src > 0) if masked else np.ones((B, H, W, C), bool)
    tag = f"conv_kernels/col2im/C{C}_{H}x{W}_k{k}s{s}/{bk}/{'relu' if masked else 'nomask'}"
    _exact(tag + "/fp32_order", got, np.where(keep, _col2im_ref32(dcol, B, C, H, W, k, s), np.float32(0.0)))
    cnt = _fold64(np.ones_like(dcol), B, C, H, W, k, s)
    absum = _fold64(np.abs(dcol), B, C, H, W, k, s)
    ref64 = np.where(keep, _fold64(dcol, B, C, H, W, k, s), 0.0)
    _bounded(tag + "/fp64", got, ref64, cnt * U * absum)
    uncovered = cnt == 0
    assert uncovered.any() == ((H - k) % s != 0 or (W - k) % s != 0 or s > k)
    assert (_bits(got[uncovered]) == 0).all(), "an input pixel no window covers must get exactly +0.0"
    if masked:
        assert (_bits(got[~keep]) == 0).all()


# ----------------------------------------------------------------------------------------------- flatten permutes
FLAT_SHAPES = [(1, 1, 1), (3, 1, 64), (5, 49, 1), (7, 15, 13), ("cap", 49, 64)]
FLAT_IDS = [f"B{b}-HW{hw}-C{c}" for b, hw, c in FLAT_SHAPES]


@pytest.mark.parametrize("B,HW,C", FLAT_SHAPES, ids=FLAT_IDS)
def test_flatten_permutes_bit_exact(B, HW, C):
    """``ts_nhwc_to_nchw_flat`` (nn.Flatten of the NCHW tensor) and its backward ``ts_nchw_flat_to_nhwc`` with the
    mask NULL and with a mask of positives, +0.0, -0.0 and negatives: bit-exact."""
    if B == "cap":
        B = _grid_cap() // (HW * C) + 3
    rng = np.random.default_rng(HW * 100 + C + B)
    x = _nhwc_input(rng, B, HW, 1, C).reshape(B, HW, C)
    y = torch.full((B, C * HW), float("nan"), device=DEV)
    _call("ts_nhwc_to_nchw_flat", _p(_d(x)), B, HW, C, _p(y))
    tag = f"conv_kernels/flatten/B{B}_HW{HW}_C{C}"
    _exact(tag + "/fwd", _h(y), x.transpose(0, 2, 1).reshape(B, C * HW))
    dy = _nhwc_input(rng, B, C * HW, 1, 1).reshape(B, C * HW)
    want = dy.reshape(B, C, HW).transpose(0, 2, 1)
    for masked in (False, True):
        src = _mask_values(rng, (B, HW, C)) if masked else None
        dx = torch.full((B, HW, C), float("nan"), device=DEV)
        _call("ts_nchw_flat_to_nhwc", _p(_d(dy)), B, HW, C, _p(_d(src)) if masked else None, _p(dx))
        _exact(f"{tag}/bwd_{'relu' if masked else 'nomask'}", _h(dx), np.where(src > 0, want, np.float32(0.0)) if masked else want)


# ------------------------------------------------------------------------------------------------------------ concat2
@pytest.mark.parametrize("wa,wb", [(1, 1), (17, 6), (376, 17), (0, 5)])
@pytest.mark.parametrize("rows", [0, 1, 37, "cap"])
def test_concat2_bit_exact(wa, wb, rows):
    """``ts_concat2`` (the SAC / GAIL critic input obs ++ act) bit-exact, including an empty left part and zero rows
    (nothing written)."""
    if rows == "cap":
        rows = _grid_cap() // (wa + wb) + 3
    rng = np.random.default_rng(wa * 31 + wb + rows)
    a = rng.standard_normal((rows, wa)).astype(np.float32)
    b = rng.standard_normal((rows, wb)).astype(np.float32)
    out = torch.full((rows * (wa + wb) + 1,), float("nan"), device=DEV)
    _call("ts_concat2", _p(_dn(a)), wa, _p(_dn(b)), wb, rows, _p(out))
    got = _h(out)
    _exact(f"conv_kernels/concat2/{wa}+{wb}/r{rows}", got[:-1].reshape(rows, wa + wb), np.concatenate([a, b], axis=1))
    assert np.isnan(got[-1]), "nothing past rows x (wa + wb) is written"


# ------------------------------------------------------------------------------------------------------------ colsum
def _colsum_ref32(x, M, N, old, accumulate):
    """``colsum_kernel`` restated: row lane w (0 .. 7) sums rows w, w + 8, ... in fp32 from +0.0f, the eight lanes are
    folded in order 0 .. 7 from +0.0f, then ``accumulate`` adds the old value."""
    acc = np.zeros((8, N), np.float32)
    full = M // 8
    for blk in x[:full * 8, :N].reshape(full, 8, N):
        acc += blk
    if M - full * 8:
        acc[:M - full * 8] += x[full * 8:M, :N]
    t = np.zeros(N, np.float32)
    for w in range(8):
        t = t + acc[w]
    return (old + t) if accumulate else t


COLSUM_CASES = ([(M, N) for M in (0, 1, 7, 8, 9, 255) for N in (1, 6, 31, 32, 33, 512)]
                + [(12800, N) for N in (1, 32, 33, 512)] + [(63648, N) for N in (31, 32, 33)]
                + [(524288, N) for N in (1, 6, 33)])


@pytest.mark.parametrize("M,N", COLSUM_CASES, ids=[f"M{m}-N{n}" for m, n in COLSUM_CASES])
def test_net_colsum_vs_fixed_order_and_fp64(M, N):
    """``ts_net_colsum`` (every layer-wise bias gradient and the layer-wise log-std gradient): dense (ld = N) and
    strided (ld = N + 3, the padding NaN) input, ``accumulate`` 0 and 1; bit-exact against the restatement of its
    fixed order, within (ceil(M / 8) + 8) x 2^-24 x (sum |x| + |old|) of an fp64 sum per column, and the output past
    N untouched.  Tall M is the conv-bias case: B x Ho x Wo rows."""
    rng = np.random.default_rng(M * 3 + N)
    x = (rng.standard_normal((M, N)) + 0.5).astype(np.float32)
    old = rng.standard_normal(N).astype(np.float32)
    tail = np.array([3.5, -0.0, np.nan, 7.25], np.float32)
    for ld in (N, N + 3):
        xs = np.full((M, ld), np.nan, np.float32)
        xs[:, :N] = x
        xs_t = _dn(xs)
        for accumulate in (0, 1):
            out = _d(np.concatenate([old, tail]))
            _call("ts_net_colsum", _p(xs_t), ld, M, N, _p(out), accumulate)
            got = _h(out)
            tag = f"conv_kernels/colsum/M{M}_N{N}/ld{ld - N}/acc{accumulate}"
            _exact(tag + "/fixed_order", got[:N], _colsum_ref32(xs, M, N, old, accumulate))
            assert (_bits(got[N:]) == _bits(tail)).all(), "out past N must stay untouched"
            ref64 = x.astype(np.float64).sum(0) + (old.astype(np.float64) if accumulate else 0.0)
            mag = np.abs(x.astype(np.float64)).sum(0) + (np.abs(old.astype(np.float64)) if accumulate else 0.0)
            _bounded(tag + "/fp64", got[:N], ref64, (math.ceil(M / 8) + 8) * U * mag)


# --------------------------------------------------------------------------------------------------- ppo rows stats
@pytest.mark.parametrize("B", [1, 255, 256, 257, 16384, 524288])
def test_ppo_rows_stats_vs_fixed_order(B):
    """``ts_ppo_rows_stats`` (the layer-wise loss table row): slots 1 .. 3 bit-exact against the restatement -- 256 lanes
    summing rows t, t + 256, ... in fp32, the tree 128 -> 1, an IEEE division by B (slot 1 negated); slot 0 (the loss
    with the fp32-rounded vf / ent coefficients; nvcc may contract it into FMAs) within four roundings of the fp64
    combination of slots 1 .. 3; slot 5 = B; slots 4, 6 and 7 untouched."""
    import ctypes

    from tianshou_b200._cabi import PPOHParams
    rng = np.random.default_rng(B)
    rows = np.stack([rng.standard_normal(B), np.abs(rng.standard_normal(B)) * 3.0, 1.4 + 0.1 * rng.standard_normal(B)],
                    axis=1).astype(np.float32)
    hp = PPOHParams(eps_clip=0.2, vf_coef=0.25, ent_coef=0.01)
    init = np.array([9.0, 9.0, 9.0, 9.0, 3.5, 9.0, -0.0, np.nan], np.float32)
    stats = _d(init)
    _call("ts_ppo_rows_stats", _p(_d(rows)), B, ctypes.byref(hp), _p(stats))
    got = _h(stats)
    lanes = np.zeros((256, 3), np.float32)
    full = B // 256
    for blk in rows[:full * 256].reshape(full, 256, 3):
        lanes += blk
    if B - full * 256:
        lanes[:B - full * 256] += rows[full * 256:]
    off = 128
    while off:
        lanes[:off] = lanes[:off] + lanes[off:2 * off]
        off //= 2
    nb = np.float32(B)
    ref = np.array([-lanes[0, 0] / nb, lanes[0, 1] / nb, lanes[0, 2] / nb], np.float32)
    tag = f"conv_kernels/ppo_rows_stats/B{B}"
    _exact(tag + "/slots123", got[1:4], ref)
    vf, ent = float(np.float32(0.25)), float(np.float32(0.01))
    s1, s2, s3 = (float(v) for v in got[1:4])
    terms = abs(s1) + abs(vf * s2) + abs(ent * s3)
    _bounded(tag + "/slot0", got[:1], np.array([s1 + vf * s2 - ent * s3]), np.array([4 * U * terms]))
    assert got[5] == B
    assert (_bits(got[[4, 6, 7]]) == _bits(init[[4, 6, 7]])).all(), "slots 4, 6 and 7 must stay untouched"


# ------------------------------------------------------------------------------------- FusedStack conv stacks vs fp64
def _flat_modules(mods):
    out = []
    for m in mods:
        out += _flat_modules(list(m)) if isinstance(m, nn.Sequential) else [m]
    return out


def _gemm_gamma(K: int) -> float:
    """Relative accuracy of one ``ts_net_gemm`` output element against sum_k |a_k w_k| (+ |bias|), as the GEMM tests
    state it: each of the 6 x ceil(K / 16) bf16 MMAs may round by 2^-24 of the running sum, split-K adds up to K / 64
    partials in fp32, plus a few roundings for the operand split, the bias and the output."""
    return (6 * math.ceil(K / 16) + math.ceil(K / 64) + 8) * U


def _forward64_with_bound(mods, x64):
    """fp64 forward of the module chain and an element-wise bound on the fp32-faithful forward's error: per layer
    E_out = gamma(K) (|W| |a| + |b|) + |W| E_in (the GEMM's own error plus the propagated one); ReLU and Tanh are
    1-Lipschitz, tanhf adds 4 ulp of its output."""
    a, E = x64, torch.zeros_like(x64)
    for m in _flat_modules(mods):
        if isinstance(m, nn.Conv2d):
            W, b, s = m.weight, m.bias, m.stride[0]
            K = W.shape[1] * W.shape[2] * W.shape[3]
            E = _gemm_gamma(K) * F.conv2d(a.abs(), W.abs(), b.abs(), stride=s) + F.conv2d(E, W.abs(), None, stride=s)
            a = F.conv2d(a, W, b, stride=s)
        elif isinstance(m, nn.Linear):
            W, b = m.weight, m.bias
            E = _gemm_gamma(W.shape[1]) * F.linear(a.abs(), W.abs(), b.abs()) + F.linear(E, W.abs())
            a = F.linear(a, W, b)
        elif isinstance(m, nn.ReLU):
            a = torch.relu(a)
        elif isinstance(m, nn.Tanh):
            a = torch.tanh(a)
            E = E + 4 * U * a.abs()
        elif isinstance(m, nn.Flatten):
            a, E = a.flatten(1), E.flatten(1)
        else:
            raise AssertionError(m)
    return a, E


def _check_layers(tag, layers, mods64, acts, x64, B):
    """Every layer's output in the stack's activation list against fp64 of the same layer applied to the stack's own
    fp32 input (the frames' table values for the first): within gamma(K) (|W| |a| + |b|) element by element (+ 4 ulp of
    tanhf) -- the GEMM's stated accuracy with nothing propagated; the flatten permutes bit-exact."""
    mods = [m for m in _flat_modules(mods64) if isinstance(m, (nn.Conv2d, nn.Linear, nn.Flatten))]
    assert len(mods) == len(layers)
    for i, (L, m) in enumerate(zip(layers, mods)):
        y = _h(acts[i + 1])
        if L.kind == "flatten":
            _exact(f"{tag}/layer{i}_flatten", y, _h(acts[i].view(B, L.H, L.W, L.C).permute(0, 3, 1, 2).reshape(B, -1)))
            continue
        if L.kind == "conv":
            a = x64 if i == 0 else acts[i].cpu().double().view(B, L.H, L.W, L.C).permute(0, 3, 1, 2)
            pre, mag = F.conv2d(a, m.weight, m.bias, stride=L.s), F.conv2d(a.abs(), m.weight.abs(), m.bias.abs(), stride=L.s)
            pre, mag = (t.permute(0, 2, 3, 1).reshape(-1, L.out_dim) for t in (pre, mag))
        else:
            a = acts[i].cpu().double().view(B, L.in_dim)
            pre, mag = F.linear(a, m.weight, m.bias), F.linear(a.abs(), m.weight.abs(), m.bias.abs())
        ref = torch.relu(pre) if L.act == 1 else (torch.tanh(pre) if L.act == 2 else pre)
        bound = _gemm_gamma(L.in_dim) * mag + (4 * U * ref.abs() if L.act == 2 else 0.0)
        _bounded(f"{tag}/layer{i}_{L.kind}", y, ref.detach().numpy(), bound.detach().numpy())


def _model(name):
    """(module chain, (C, H, W)) of the stacks under test."""
    from tianshou_b200.env.atari import DQNet
    if name.startswith("dqnet"):
        c, h, w = (int(v) for v in name.split("_")[1].split("x"))
        return DQNet(c, h, w, 5).net, (c, h, w)
    if name == "odd":
        # 3 x 41 x 30 -> 8 x 19 x 14 -> (k 2 < s 3) 5 x 6 x 5 -> (1 x 1, no activation) 7 x 6 x 5 -> (no activation
        # before the flatten) 6 x 4 x 3 -> Linear(72, 9) + Tanh -> Linear(9, 4)
        return nn.Sequential(nn.Conv2d(3, 8, 4, 2), nn.ReLU(), nn.Conv2d(8, 5, 2, 3), nn.ReLU(), nn.Conv2d(5, 7, 1, 1),
                             nn.Conv2d(7, 6, 3, 1), nn.Flatten(), nn.Linear(72, 9), nn.Tanh(), nn.Linear(9, 4)), (3, 41, 30)
    if name == "row":
        # 2 x 7 x 40 -> 6 x 1 x 12 (a one-row output) -> (1 x 1, stride 2: odd columns uncovered) 3 x 1 x 6 -> Linear(18, 4)
        return nn.Sequential(nn.Conv2d(2, 6, 5, 3), nn.ReLU(), nn.Conv2d(6, 3, 1, 2), nn.Flatten(), nn.Linear(18, 4)), (2, 7, 40)
    raise AssertionError(name)


STACKS = ["dqnet_4x64x48", "dqnet_4x210x160", "dqnet_1x84x84", "odd", "row"]


@pytest.mark.parametrize("B", [1, 3, 33])
@pytest.mark.parametrize("name", STACKS)
def test_fused_conv_stack_vs_fp64_autograd(name, B):
    """Forward from uint8 frames (fused frame-stack gather + im2col) and every parameter gradient of sum(q * coef)
    through ``compile_sequential`` + ``FusedStack``, against fp64 autograd on a copy of the same modules.  The forward bars
    are element-wise and derived from the GEMM's stated accuracy, not from a torch fp32 forward (TF32 on this GPU): each
    layer on its own input (``_check_layers``), and q against the fp64 forward with the worst-case propagation of those
    errors (``_forward64_with_bound``).  The gradients take the existing conv test's bar against fp64 autograd with the
    stack's own ReLU decisions.  Two identical forward + backward calls must give bit-identical outputs and gradients."""
    from tianshou_b200.algorithm.flat_params import FlatGroup
    from tianshou_b200.algorithm.netgraph import FusedStack, compile_sequential
    torch.manual_seed(STACKS.index(name) * 100 + B)
    net, (C, H, W) = _model(name)
    net = net.to(DEV)
    net64 = copy.deepcopy(net).to("cpu", torch.float64)
    layers = compile_sequential(list(net), (C, H, W))
    convs = [L for L in layers if L.kind == "conv"]
    params = [p for L in layers if L.weight is not None for p in (L.weight, L.bias)]
    group = FlatGroup(params, torch.device(DEV))
    stack = FusedStack(layers, group)
    rng = np.random.default_rng(B + len(name))
    S = B * C + 3
    frames = rng.integers(0, 256, (S, H, W), dtype=np.uint8)
    sidx = _stack_idx(rng, B, C, S)
    x64 = torch.from_numpy((frames[sidx].astype(np.float64) / 255.0).astype(np.float32).astype(np.float64))
    with torch.no_grad():
        q64, bound = _forward64_with_bound(list(net64), x64)
    # the compiled output sizes are torch's own (an H / W exchange in compile_sequential changes them for H != W)
    shapes, a = [], x64
    with torch.no_grad():
        for m in _flat_modules(list(net64)):
            a = m(a)
            if isinstance(m, nn.Conv2d):
                shapes.append(tuple(a.shape[2:]))
    assert [(L.Ho, L.Wo) for L in convs] == shapes
    A = q64.shape[1]
    coef = torch.from_numpy(rng.standard_normal((B, A)).astype(np.float32))
    fr, si = _d(frames), _d(sidx)
    runs = []
    for _ in range(2):
        acts = stack.forward(None, B, "t", frames=(fr, si, 255.0))
        stack.backward(acts, coef.to(DEV).contiguous(), B, "t")
        torch.cuda.synchronize()
        runs.append((acts[-1].clone(), group.grad.clone()))
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1]), "two identical calls must agree bit for bit"
    q, grad = runs[1]
    tag = f"conv_stack_fp64/{name}/B{B}"
    _bounded(tag + "/q", _h(q), q64.numpy(), bound.numpy())
    with torch.no_grad():
        _check_layers(tag, layers, list(net64), acts, x64, B)
    # the fp64 backward takes the ReLU decisions of the stack's own forward: with B x Ho x Wo = 65,637 conv-1 rows
    # (210 x 160, B 33) some pre-activations lie within the forward's rounding of 0, and one that takes the other branch
    # moves a weight gradient by a whole row's term (observed 7.8e-4 of max on conv 1 with fp64's own decisions)
    out, li = x64, 0
    for m in _flat_modules(list(net64)):
        if isinstance(m, nn.ReLU):
            L, keep = layers[li - 1], (acts[li] > 0).cpu().to(torch.float64)
            out = out * (keep.view(B, L.Ho, L.Wo, L.out_dim).permute(0, 3, 1, 2) if L.kind == "conv" else keep.view(B, L.out_dim))
        else:
            out = m(out)
            li += isinstance(m, (nn.Conv2d, nn.Linear, nn.Flatten))
    (out * coef.double()).sum().backward()
    ref_params = [p for m in _flat_modules(list(net64)) if isinstance(m, (nn.Conv2d, nn.Linear)) for p in (m.weight, m.bias)]
    for i, (p, rp) in enumerate(zip(params, ref_params, strict=True)):
        got = group.view(grad, p).view(p.shape)
        ref = rp.grad.numpy()
        record_parity(f"{tag}/grad{i}", _h(got), ref, rtol=1e-4, atol=2e-5 * float(np.abs(ref).max()))


# ------------------------------------------------------------------------------------ DQN.update() on these geometries
class _Discrete:
    def __init__(self, n):
        self.n = n
        self.shape = ()


def _copy64(mod, group, flat):
    """Deep copy of ``mod`` on the CPU in float64 with its parameters read from ``flat`` (a snapshot of ``group.flat``)."""
    c = copy.deepcopy(mod).to("cpu", torch.float64)
    with torch.no_grad():
        for (_, p), (_, q) in zip(mod.named_parameters(), c.named_parameters(), strict=True):
            q.copy_(group.view(flat, p).view(p.shape).to(torch.float64))
    return c


DQN_CASES = [(4, 64, 48, 4), (1, 84, 84, 1)]


@pytest.mark.parametrize("C,H,W,stack_num", DQN_CASES, ids=[f"C{c}-{h}x{w}-stack{s}" for c, h, w, s in DQN_CASES])
def test_dqn_update_gradients_vs_fp64_autograd_on_frames(C, H, W, stack_num):
    """``DQN.update()`` (double DQN, 1-step returns, MSE, no target network) on single-frame uint8 storage: DQNet(4, 64, 48)
    stacked through the prev() chain (stack_num 4; conv 2 leaves an input row and column uncovered) and DQNet(1, 84, 84)
    on single frames (stack_num 1, conv 1 K = 64).  Two updates: the flat gradient snapshotted at the optimiser step
    against fp64 autograd of the reference loss (dqn.py:384-401) on a copy of the module with the same parameters and
    batch, and the returns against r + gamma (1 - terminated) Q(s', argmax_a Q(s', a)) in fp64."""
    from tianshou_b200.algorithm import AdamOptimizerFactory
    from tianshou_b200.algorithm.modelfree.dqn import DQN, DiscreteQLearningPolicy
    from tianshou_b200.data import Batch, VectorReplayBuffer
    from tianshou_b200.env.atari import DQNet, ScaledObsInputActionReprNet
    from tianshou_b200.utils import policy_within_training_step
    E, T, A, gamma, Bs = 4, 40, 6, 0.9, 32
    rng = np.random.default_rng(H + W + stack_num)
    torch.manual_seed(H * W)
    kw = dict(stack_num=4, save_only_last_obs=True) if stack_num == 4 else {}
    buf = VectorReplayBuffer(E * T, E, ignore_obs_next=True, device=DEV, **kw)
    for t in range(T):
        frame = rng.integers(0, 256, (E, H, W), dtype=np.uint8)
        obs = np.repeat(frame[:, None], 4, axis=1) if stack_num == 4 else frame
        term = rng.random(E) < 0.1
        trunc = np.full(E, t % 13 == 12) & ~term
        buf.add(Batch(obs=obs, act=rng.integers(0, A, E), rew=rng.standard_normal(E), terminated=term, truncated=trunc,
                      obs_next=obs), buffer_ids=np.arange(E))
    net = ScaledObsInputActionReprNet(DQNet(C, H, W, A)).to(DEV)
    algo = DQN(policy=DiscreteQLearningPolicy(model=net, action_space=_Discrete(A)), optim=AdamOptimizerFactory(lr=1e-3),
               gamma=gamma, n_step_return_horizon=1, target_update_freq=0, is_double=True)
    group = algo._group
    cap = []
    real_step, orig_pre = group.adam_step, algo._preprocess_batch

    def adam_step(optimizer, max_grad_norm):
        cap[-1].update(grad=group.grad.clone(), flat=group.flat.clone())
        real_step(optimizer, max_grad_norm)

    def pre(batch, buffer, indices):
        cap.append(dict(indices=np.asarray(indices).copy()))
        b = orig_pre(batch, buffer, indices)
        cap[-1]["returns"] = b.returns.detach().reshape(-1).cpu().clone()
        return b

    group.adam_step, algo._preprocess_batch = adam_step, pre

    def stacks(idx):
        o = buf.get(idx, "obs") if stack_num == 4 else np.asarray(buf.obs)[idx][:, None]
        assert o.shape == (len(idx), C, H, W) and o.dtype == np.uint8
        return torch.from_numpy((o.astype(np.float64) / 255.0).astype(np.float32).astype(np.float64))

    for u in range(2):
        np.random.seed(300 + u)
        with policy_within_training_step(algo.policy):
            stats = algo.update(buffer=buf, sample_size=Bs)
        c = cap[u]
        idx = c["indices"]
        tag = f"conv_dqn_grad/C{C}_{H}x{W}_stack{stack_num}_u{u}"
        ref = _copy64(net, group, c["flat"])
        with torch.no_grad():
            q_next = ref.module.net(stacks(buf.next(idx)))
            tq = q_next.gather(1, q_next.argmax(1, keepdim=True)).view(-1)
        term = torch.as_tensor(np.asarray(buf.terminated)[idx].astype(np.float64))
        R = torch.as_tensor(np.asarray(buf.rew)[idx].astype(np.float64)) + gamma * (1.0 - term) * tq
        record_parity(f"{tag}/returns", c["returns"].numpy(), R.numpy(), rtol=1e-5, atol=1e-5 * float(R.abs().max()))
        R = c["returns"].to(torch.float64)
        q = ref.module.net(stacks(idx))
        act = torch.as_tensor(np.asarray(buf.act)[idx].astype(np.int64)).view(-1, 1)
        L = (R - q.gather(1, act).view(-1)).pow(2).mean()
        L.backward()
        for (name, p), (_, r) in zip(net.named_parameters(), ref.named_parameters(), strict=True):
            g = r.grad.numpy()
            record_parity(f"{tag}/grad_{name}", _h(group.view(c["grad"], p).view(p.shape)), g, rtol=2e-4,
                          atol=1e-4 * float(np.abs(g).max()) + 1e-12)
        record_parity(f"{tag}/loss", np.array([stats.loss]), np.array([L.item()]), rtol=2e-5, atol=1e-7)


# ---------------------------------------------------------------------------------------------- refusals at build time
class _ConvQ(nn.Module):
    """A Q-network with a conv chain in ``.net`` and its ``input_shape``, as DQNet exposes them."""

    def __init__(self, net, input_shape):
        super().__init__()
        self.net = net
        self.input_shape = input_shape


REFUSED = {
    "input_smaller_than_kernel": (lambda: nn.Sequential(nn.Conv2d(4, 8, 5, 1), nn.ReLU(), nn.Flatten(), nn.Linear(8, 2)), (4, 4, 10)),
    "narrower_than_kernel": (lambda: nn.Sequential(nn.Conv2d(4, 8, 5, 1), nn.ReLU(), nn.Flatten(), nn.Linear(8, 2)), (4, 10, 4)),
    "second_conv_input_too_small": (lambda: nn.Sequential(nn.Conv2d(4, 8, 8, 4), nn.ReLU(), nn.Conv2d(8, 8, 4, 2), nn.ReLU(),
                                                          nn.Flatten(), nn.Linear(8, 2)), (4, 16, 40)),
    "tanh_before_conv": (lambda: nn.Sequential(nn.Conv2d(4, 8, 4, 2), nn.Tanh(), nn.Conv2d(8, 8, 3, 1), nn.ReLU(), nn.Flatten(),
                                               nn.Linear(8 * 5 * 5, 2)), (4, 16, 16)),
    "tanh_before_flatten": (lambda: nn.Sequential(nn.Conv2d(4, 8, 4, 2), nn.ReLU(), nn.Conv2d(8, 8, 3, 1), nn.Tanh(), nn.Flatten(),
                                                  nn.Linear(8 * 5 * 5, 2)), (4, 16, 16)),
    "tanh_before_nested_flatten": (lambda: nn.Sequential(nn.Sequential(nn.Conv2d(4, 8, 4, 2), nn.Tanh()), nn.Flatten(),
                                                         nn.Linear(8 * 7 * 7, 2)), (4, 16, 16)),
}


@pytest.mark.parametrize("case", list(REFUSED))
def test_unsupported_conv_chains_are_refused_when_the_dqn_is_built(case):
    """A convolution whose input is smaller than its kernel (no output pixel) and a Tanh in front of a convolution or a
    flatten (whose backward the fused stack does not provide) raise UnsupportedModelError from ``compile_sequential``,
    i.e. when the DQN is built -- not at the first forward or in the middle of the first ``update()``."""
    from tianshou_b200.algorithm import AdamOptimizerFactory
    from tianshou_b200.algorithm.flat_params import UnsupportedModelError
    from tianshou_b200.algorithm.modelfree.dqn import DQN, DiscreteQLearningPolicy
    from tianshou_b200.algorithm.netgraph import compile_sequential
    make, shape = REFUSED[case]
    with pytest.raises(UnsupportedModelError):
        compile_sequential(list(make()), shape)
    model = _ConvQ(make(), shape).to(DEV)
    with pytest.raises(UnsupportedModelError):
        DQN(policy=DiscreteQLearningPolicy(model=model, action_space=_Discrete(2)), optim=AdamOptimizerFactory(lr=1e-3))


def test_tanh_after_the_flatten_and_one_pixel_convolutions_are_accepted():
    """The refusals stop where the fused stack's backward works: a Tanh Linear after the flatten, a convolution whose
    input is exactly its kernel's size (one output pixel), and a Tanh on the last Linear's input."""
    from tianshou_b200.algorithm.netgraph import compile_sequential
    net = nn.Sequential(nn.Conv2d(4, 8, 5, 1), nn.ReLU(), nn.Flatten(), nn.Linear(8, 6), nn.Tanh(), nn.Linear(6, 2))
    layers = compile_sequential(list(net), (4, 5, 5))
    assert [(L.kind, L.Ho, L.Wo) for L in layers[:1]] == [("conv", 1, 1)]
