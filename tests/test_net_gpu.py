"""Layered-network kernels (csrc/net_gemm.cu, csrc/net_ops.cu) against plain torch references on the same inputs:
the wgmma bf16x3 GEMM in its three operand arrangements (forward / input gradient / weight gradient), im2col /
col2im / flatten permutes, and a full ``FusedStack`` forward + backward vs torch autograd (fp32, tolerance stated)."""
import numpy as np
import pytest
import torch

from ts_testutil import record_parity

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _gemm(a, lda, a_mn, b, ldb, b_mn, c, M, N, K, bias=None, act=0, mask=None, mask_kind=1, accumulate=False, split=True):
    from tianshou_b200._cabi import call, load_library, ptr, stream_ptr
    ws_n = int(load_library().ts_net_gemm_workspace_floats(M, N, K)) if split else 0
    ws = torch.empty(max(ws_n, 1), dtype=torch.float32, device=DEV)
    call("ts_net_gemm", ptr(a), lda, a_mn, ptr(b), ldb, b_mn, ptr(c), c.shape[1], M, N, K, ptr(bias), act,
         ptr(mask), mask.shape[1] if mask is not None else 0, mask_kind, int(accumulate), ptr(ws) if ws_n else None, ws_n, stream_ptr())
    return ws_n


@pytest.mark.parametrize("M,N,K", [(256, 256, 393), (256, 1, 256), (32, 512, 3136), (12800, 32, 256), (1, 7, 5), (130, 129, 65),
                                   (2592, 64, 512), (256, 34, 256)])
def test_net_gemm_forward_vs_fp64(M, N, K):
    g = torch.Generator(device="cpu").manual_seed(M * 7 + N * 3 + K)
    x = torch.randn(M, K, generator=g).to(DEV)
    w = (torch.randn(N, K, generator=g) / K ** 0.5).to(DEV)
    bias = torch.randn(N, generator=g).to(DEV)
    y = torch.full((M, N), float("nan"), device=DEV)
    _gemm(x, K, 0, w, K, 0, y, M, N, K, bias=bias, act=1)
    ref = torch.relu(x.double() @ w.double().T + bias.double())
    fp32 = torch.relu(x @ w.T + bias)
    # bf16x3 = 24 significant bits per operand, pieces obtained by truncation: observed 1e-6 .. 3e-6 of max |C| (r2c run)
    e = record_parity(f"net_gemm_fwd/{M}x{N}x{K}", y.cpu().numpy(), ref.cpu().numpy(), rtol=5e-6, atol=5e-6 * float(ref.abs().max()))
    # fp32-faithful: the same order as torch's own fp32 GEMM against the fp64 product (plus 2e-6 of max |C|: the fp32
    # accumulation inside the tensor core over K / 16 x 6 MMAs; torch's N = 1 case is a gemv with a near-exact sum)
    assert e["max_abs_err"] <= 8.0 * float((fp32.double() - ref).abs().max()) + 2e-6 * float(ref.abs().max())


@pytest.mark.parametrize("M,N,K", [(256, 393, 256), (256, 17, 256), (1568, 576, 64), (100, 40, 33)])
def test_net_gemm_input_gradient_arrangement(M, N, K):
    """dX[M, N] = dY[M, K] W[K, N]  with W given as the layer's [out = K][in = N] matrix (B operand MN-major) + ReLU mask."""
    g = torch.Generator(device="cpu").manual_seed(11)
    dy = torch.randn(M, K, generator=g).to(DEV)
    w = torch.randn(K, N, generator=g).to(DEV)
    src = torch.randn(M, N, generator=g).to(DEV)
    out = torch.zeros(M, N, device=DEV)
    _gemm(dy, K, 0, w, N, 1, out, M, N, K, mask=src)
    ref = (dy.double() @ w.double()) * (src > 0)
    record_parity(f"net_gemm_dx/{M}x{N}x{K}", out.cpu().numpy(), ref.cpu().numpy(), rtol=2e-6, atol=2e-6 * float(ref.abs().max()))
    y = torch.tanh(src)
    _gemm(dy, K, 0, w, N, 1, out, M, N, K, mask=y, mask_kind=2)
    ref = (dy.double() @ w.double()) * (1 - y.double() ** 2)
    record_parity(f"net_gemm_dx_tanh/{M}x{N}x{K}", out.cpu().numpy(), ref.cpu().numpy(), rtol=2e-6, atol=2e-6 * float(ref.abs().max()))


@pytest.mark.parametrize("rows,out_f,in_f", [(256, 256, 393), (12800, 32, 256), (32, 512, 3136), (77, 6, 20)])
def test_net_gemm_weight_gradient_arrangement(rows, out_f, in_f):
    """dW[out, in] = dY^T X (both operands MN-major, reduction over the batch rows; split-K for long reductions)."""
    g = torch.Generator(device="cpu").manual_seed(5)
    dy = torch.randn(rows, out_f, generator=g).to(DEV)
    x = torch.randn(rows, in_f, generator=g).to(DEV)
    for accumulate in (False, True):
        out = torch.ones(out_f, in_f, device=DEV)
        ws_n = _gemm(dy, out_f, 1, x, in_f, 1, out, out_f, in_f, rows, accumulate=accumulate)
        ref = dy.double().T @ x.double() + (1.0 if accumulate else 0.0)
        record_parity(f"net_gemm_dw/{rows}x{out_f}x{in_f}/acc{int(accumulate)}/split{int(ws_n > 0)}", out.cpu().numpy(),
                      ref.cpu().numpy(), rtol=2e-6, atol=3e-6 * float(ref.abs().max()))
    from tianshou_b200._cabi import call, ptr, stream_ptr
    gb = torch.zeros(out_f, device=DEV)
    call("ts_net_colsum", ptr(dy), out_f, rows, out_f, ptr(gb), 0, stream_ptr())
    np.testing.assert_allclose(gb.cpu().numpy(), dy.double().sum(0).cpu().numpy(), rtol=1e-5, atol=1e-4)


# operand arrangements (A MN-major, B MN-major): forward X W^T, input gradient dY W, A MN-major with B K-major, weight
# gradient dY^T X -- with the fp64 tolerance of the existing test of the same arrangement (the A-MN-major-only one has
# none and takes the forward's)
ARRANGEMENTS = {"fwd": (0, 0, 5e-6, 5e-6), "dx": (0, 1, 2e-6, 2e-6), "amn": (1, 0, 5e-6, 5e-6), "dw": (1, 1, 2e-6, 3e-6)}
# M, N around the 128-wide tile edges, K around the 16-deep MMA step and the 64-deep staged chunk; K = 3136 walks the two
# shared-memory stages 49 times (unsplit) -- tiles < 64 and K > 64 split along K when a workspace is given
EDGE_SHAPES = [(1, 1, 1), (63, 64, 15), (64, 63, 16), (127, 129, 17), (128, 127, 64), (129, 257, 65), (257, 128, 3136),
               (1, 257, 3136), (257, 1, 65), (129, 63, 1)]
# epilogues: (bias, act, mask kind (0 = none), accumulate)
EPILOGUES = [(True, 0, 0, False), (True, 1, 1, True), (False, 2, 2, False), (True, 2, 0, True), (False, 0, 1, False)]


def _strided(store, off, rows, cols, ld):
    return store.as_strided((rows, cols), (ld, 1), off)


@pytest.mark.parametrize("arr", list(ARRANGEMENTS))
@pytest.mark.parametrize("M,N,K", EDGE_SHAPES)
def test_net_gemm_arrangements_edges_vs_fp64(M, N, K, arr):
    """Every operand arrangement at tile-edge shapes, split and unsplit (which one ran is asserted), dense operands and
    views (pointers an odd number of floats into the allocation, ld > extent, ldc > N, ld_mask > N: the scalar-load
    fallback and the unpaired epilogue stores), every epilogue; C outside the M x N view must stay untouched, and two
    identical calls must give bit-identical results."""
    from tianshou_b200._cabi import call, load_library, stream_ptr
    a_mn, b_mn, rtol, atol_rel = ARRANGEMENTS[arr]
    g = torch.Generator(device="cpu").manual_seed(M * 131 + N * 17 + K)
    A64 = torch.randn(M, K, generator=g, dtype=torch.float64)
    B64 = torch.randn(N, K, generator=g, dtype=torch.float64) / K ** 0.5
    bias = torch.randn(N, generator=g).to(DEV)
    prod = (A64.float().double() @ B64.float().double().T).to(DEV)      # fp64 product of the fp32 operands
    tiles = ((M + 127) // 128) * ((N + 127) // 128)
    expect_split = (K + 63) // 64 >= 2 and tiles < 64
    lib = load_library()
    for view in (False, True):
        pad, off = (5, 3) if view else (0, 0)
        # A logical [M][K], B logical [N][K]; MN-major storage holds the transpose
        a_rows, a_cols = (K, M) if a_mn else (M, K)
        b_rows, b_cols = (K, N) if b_mn else (N, K)
        lda, ldb, ldc, ldm = a_cols + pad, b_cols + pad, N + (3 if view else 0), N + (2 if view else 0)
        a_st = torch.full((off + a_rows * lda,), float("nan"), device=DEV)
        b_st = torch.full((off + b_rows * ldb,), float("nan"), device=DEV)
        _strided(a_st, off, a_rows, a_cols, lda).copy_((A64.T if a_mn else A64).float())
        _strided(b_st, off, b_rows, b_cols, ldb).copy_((B64.T if b_mn else B64).float())
        # (the padding of the views stays NaN: an element read from outside an operand poisons the result)
        y_st = torch.randn(off + M * ldm, generator=g).to(DEV)
        y = _strided(y_st, off, M, N, ldm)
        for has_bias, act, mask_kind, accumulate in EPILOGUES:
            ref = prod + (bias.double() if has_bias else 0.0)
            ref = torch.relu(ref) if act == 1 else (torch.tanh(ref) if act == 2 else ref)
            if mask_kind == 1:
                ref = ref * (y.double() > 0)
            elif mask_kind == 2:
                ref = ref * (1.0 - y.double() ** 2)
            c0 = torch.randn(off + M * ldc, generator=g).to(DEV)
            if accumulate:
                ref = ref + _strided(c0, off, M, N, ldc).double()
            outs = []
            for split in (False, True):
                ws_n = int(lib.ts_net_gemm_workspace_floats(M, N, K)) if split else 0
                assert (ws_n > 0) == (split and expect_split)
                ws = torch.empty(max(ws_n, 1), device=DEV)
                for _ in range(2):
                    c = c0.clone()
                    call("ts_net_gemm", a_st.data_ptr() + 4 * off, lda, a_mn, b_st.data_ptr() + 4 * off, ldb, b_mn,
                         c.data_ptr() + 4 * off, ldc, M, N, K, bias.data_ptr() if has_bias else None, act,
                         y.data_ptr() if mask_kind else None, ldm if mask_kind else 0, mask_kind or 1, int(accumulate),
                         ws.data_ptr() if ws_n else None, ws_n, stream_ptr())
                    outs.append((split, c))
                key = (f"net_gemm_edges/{arr}/{M}x{N}x{K}/{'view' if view else 'dense'}/b{int(has_bias)}a{act}m{mask_kind}"
                       f"acc{int(accumulate)}/split{int(ws_n > 0)}")
                got = _strided(outs[-1][1], off, M, N, ldc)
                # Unsplit, one register accumulator takes all K / 16 * 6 MMA additions; each may round by up to ~2^-24 of
                # the running sum, so the bound grows with K (at K = 3136: 7e-5 of max |C|, observed 2.7e-5; split-K
                # partials are summed in fp32 and stay within the existing bar)
                acc_bound = 0.0 if ws_n else (K + 15) // 16 * 6 * 2.0 ** -24
                record_parity(key, got.cpu().numpy(), ref.cpu().numpy(), rtol=rtol,
                              atol=max(atol_rel, acc_bound) * float(ref.abs().max()))
                # nothing outside the M x N view is written
                untouched = torch.ones_like(c0, dtype=torch.bool)
                _strided(untouched, off, M, N, ldc).fill_(False)
                assert torch.equal(outs[-1][1][untouched], c0[untouched]), key
                # deterministic: two identical calls, bit-identical output
                assert torch.equal(outs[-2][1], outs[-1][1]), key


def test_conv_stack_forward_backward_vs_torch():
    """NatureCNN-shaped stack (env/atari/atari_network.py:77-96) on uint8 frame stacks: forward and all parameter
    gradients of sum(q * coef) against torch autograd on the same weights."""
    from torch import nn

    from tianshou_b200.algorithm.flat_params import FlatGroup
    from tianshou_b200.algorithm.netgraph import FusedStack, compile_sequential
    torch.manual_seed(0)
    B, A = 6, 5
    net = nn.Sequential(
        nn.Sequential(nn.Conv2d(4, 32, 8, 4), nn.ReLU(inplace=True), nn.Conv2d(32, 64, 4, 2), nn.ReLU(inplace=True),
                      nn.Conv2d(64, 64, 3, 1), nn.ReLU(inplace=True), nn.Flatten()),
        nn.Linear(3136, 512), nn.ReLU(inplace=True), nn.Linear(512, A)).to(DEV)
    ref_net = __import__("copy").deepcopy(net)
    layers = compile_sequential(list(net), (4, 84, 84))
    params = [p for L in layers if L.weight is not None for p in (L.weight, L.bias)]
    group = FlatGroup(params, torch.device(DEV))
    stack = FusedStack(layers, group)
    frames = torch.randint(0, 256, (40, 84, 84), dtype=torch.uint8, device=DEV)
    sidx = torch.randint(0, 40, (B, 4), dtype=torch.int64, device=DEV)
    acts = stack.forward(None, B, "t", frames=(frames, sidx, 255.0))
    q = acts[-1]
    x = (frames[sidx].double() / 255.0).float()          # [B, 4, 84, 84]
    q_ref = ref_net(x)
    # five layers deep with random initial weights the outputs (|q| ~ 0.03) are small differences of O(1) activations: the
    # yardstick is an fp64 evaluation of the same network -- this path must be as close to it as torch's own fp32 forward is
    q64 = __import__("copy").deepcopy(ref_net).double()(x.double()).detach()
    err_torch = float((q_ref.detach().double() - q64).abs().max())
    e = record_parity("conv_stack/q_vs_fp64", q.cpu().numpy(), q64.cpu().numpy(), rtol=1e-4, atol=1e-5)
    assert e["max_abs_err"] <= 8.0 * err_torch + 1e-6, (e["max_abs_err"], err_torch)
    coef = torch.randn(B, A, device=DEV)
    # gradients against autograd in fp64 on the same weights: torch's fp32 convolution backward runs in TF32 on this GPU
    # (cudnn.allow_tf32 defaults to True; observed 2.6 % of max |grad| away from fp64 on the first layer), so it is no yardstick
    net64 = __import__("copy").deepcopy(ref_net).double()
    (net64(x.double()) * coef.double()).sum().backward()
    stack.backward(acts, coef.contiguous(), B, "t")
    ref_params = [p for m in net64.modules() if isinstance(m, (nn.Conv2d, nn.Linear)) for p in (m.weight, m.bias)]
    for i, (p, rp) in enumerate(zip(params, ref_params, strict=True)):
        got = group.view(group.grad, p).view(p.shape)
        record_parity(f"conv_stack/grad{i}", got.cpu().numpy(), rp.grad.float().cpu().numpy(), rtol=1e-4,
                      atol=2e-5 * float(rp.grad.abs().max()))


def test_stack_prev_matches_host_prev_chain():
    from tianshou_b200 import ops
    from tianshou_b200._cabi import call, ptr, stream_ptr
    from tianshou_b200.data import Batch, VectorReplayBuffer
    rng = np.random.default_rng(0)
    E, cap = 5, 12
    buf = VectorReplayBuffer(E * cap, E, device=DEV)
    for t in range(17):
        term = rng.random(E) < 0.15
        buf.add(Batch(obs=rng.standard_normal((E, 2)).astype(np.float32), act=np.zeros((E, 1), np.float32), rew=np.zeros(E),
                      terminated=term, truncated=np.zeros(E, bool), obs_next=np.zeros((E, 2), np.float32)), buffer_ids=np.arange(E))
    idx = buf.sample_indices(0)
    m = buf.device_meta()
    out = torch.empty((len(idx), 4), dtype=torch.int64, device=DEV)
    o, E_, d, l, n = m._args()
    call("ts_stack_prev_indices", ptr(ops._idx(idx, m.device)), len(idx), 4, o, E_, d, l, n, ptr(out), stream_ptr())
    want = [idx]
    for _ in range(3):
        want.insert(0, buf.prev(want[0]))
    assert np.array_equal(out.cpu().numpy(), np.stack(want, axis=1))
