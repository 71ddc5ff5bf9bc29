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


def test_conv_stack_forward_backward_vs_torch():
    """NatureCNN-shaped stack (env/atari/atari_network.py:77-96) on uint8 frame stacks: forward and all parameter
    gradients of sum(q * coef) against torch autograd on the same weights."""
    from torch import nn

    from tianshou_b200.algorithm.netgraph import FlatGroup, FusedStack, compile_sequential
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
