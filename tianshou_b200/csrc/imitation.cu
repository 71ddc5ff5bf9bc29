// Imitation-learning arithmetic (algorithm/imitation/imitation_base.py): the loss and the gradient at the actor's last Linear
// output, between the actor's forward GEMMs and its backward GEMMs.  The GEMMs are the layered-network launches of net_gemm.cu.
//
// Reference: tianshou/algorithm/imitation/imitation_base.py:115-122 (regression: F.mse_loss(actor(s), a); classification:
// F.nll_loss(F.log_softmax(actor(s)), a)), utils/net/continuous.py (ContinuousActorDeterministic: max_action * tanh(last(...))),
// utils/net/discrete.py:87 (DiscreteActor's softmax_output=True default: the classification loss then takes log_softmax of
// probabilities, which is the reference's loss as coded).  The regression follows torch's operation order with __f*_rn, as td3.cu
// does.
#include <math.h>

#include "common.cuh"
#include "row_sums.cuh"

namespace {

using tsb::kRowsPerBlock;
using tsb::kRowThreads;

constexpr int kThreads = 256;

// dz = (2 (pi - act) / n) * max_action * (1 - t^2), t = tanh(z), pi = max_action * t, n = B A: torch's backward of
// F.mse_loss(max_action * tanh(z), act) (mse_loss_backward, mul, tanh_backward).  Grid-stride over the n elements.
__global__ void __launch_bounds__(kThreads) imitation_mse_grad_kernel(const float* __restrict__ z, const float* __restrict__ act,
                                                                      int64_t n, float max_action, float norm, float* __restrict__ dz) {
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
        const float t = tanhf(z[e]);
        const float g = __fmul_rn(norm, __fsub_rn(__fmul_rn(max_action, t), act[e]));
        dz[e] = __fmul_rn(__fmul_rn(g, max_action), __fsub_rn(1.0f, __fmul_rn(t, t)));
    }
}

// loss = sum (pi - act)^2 / n, the sum in row_sums.cuh's fixed order.  One block.
__global__ void __launch_bounds__(tsb::kRowSumThreads) imitation_mse_loss_kernel(const float* __restrict__ z,
                                                                                 const float* __restrict__ act, int64_t n,
                                                                                 float max_action, float* __restrict__ loss) {
    const float s = tsb::block_sum_fixed(n, [&](int64_t e) {
        const float d = __fsub_rn(__fmul_rn(max_action, tanhf(z[e])), act[e]);
        return __fmul_rn(d, d);
    });
    if (threadIdx.x == 0) *loss = __fdiv_rn(s, (float)n);
}

// Per row b of out [B][A], one warp, lanes striding the A columns (any A):
//   softmax_output = 0: out is the last Linear's output z.  rows[b] = logsumexp(z) - z[act],  dz = (softmax(z) - onehot) / B.
//   softmax_output = 1: out is still z, the network's output is p = softmax(z), and the loss takes log_softmax of p.
//                       rows[b] = logsumexp(p) - p[act];  with g = (softmax(p) - onehot) / B,  dz = p (g - sum_k p_k g_k).
// Every log-sum-exp is shifted by the row's maximum; expf / logf at full accuracy.
__global__ void __launch_bounds__(kRowThreads) imitation_nll_rows_kernel(const float* __restrict__ out, const int64_t* __restrict__ act,
                                                                         int64_t B, int A, int softmax_output, float inv_b,
                                                                         float* __restrict__ dz, float* __restrict__ rows) {
    const int lane = tsb::lane_id();
    for (int64_t b = (int64_t)blockIdx.x * kRowsPerBlock + tsb::warp_id(); b < B; b += (int64_t)gridDim.x * kRowsPerBlock) {
        const float* x = out + b * A;
        float* d = dz + b * A;
        const int ab = (int)act[b];
        float m = -INFINITY;
        for (int k = lane; k < A; k += 32) m = fmaxf(m, x[k]);
        m = tsb::warp_max(m);
        float s = 0.0f;
        for (int k = lane; k < A; k += 32) s += expf(x[k] - m);
        s = tsb::warp_sum(s);
        float row;
        if (!softmax_output) {
            for (int k = lane; k < A; k += 32) d[k] = (expf(x[k] - m) / s - (k == ab ? 1.0f : 0.0f)) * inv_b;
            row = logf(s) - (x[ab] - m);
        } else {
            float m2 = -INFINITY;
            for (int k = lane; k < A; k += 32) m2 = fmaxf(m2, expf(x[k] - m) / s);
            m2 = tsb::warp_max(m2);
            float s2 = 0.0f;
            for (int k = lane; k < A; k += 32) s2 += expf(expf(x[k] - m) / s - m2);
            s2 = tsb::warp_sum(s2);
            float spg = 0.0f;
            for (int k = lane; k < A; k += 32) {
                const float p = expf(x[k] - m) / s;
                spg += p * ((expf(p - m2) / s2 - (k == ab ? 1.0f : 0.0f)) * inv_b);
            }
            spg = tsb::warp_sum(spg);
            for (int k = lane; k < A; k += 32) {
                const float p = expf(x[k] - m) / s;
                d[k] = p * ((expf(p - m2) / s2 - (k == ab ? 1.0f : 0.0f)) * inv_b - spg);
            }
            row = logf(s2) - (expf(x[ab] - m) / s - m2);
        }
        if (lane == 0) rows[b] = row;
    }
}

// loss = sum_b rows[b] / B, the sum in row_sums.cuh's fixed order.  One block.
__global__ void __launch_bounds__(tsb::kRowSumThreads) imitation_nll_loss_kernel(const float* __restrict__ rows, int64_t B,
                                                                                 float* __restrict__ loss) {
    const float s = tsb::block_sum_fixed(B, [&](int64_t b) { return rows[b]; });
    if (threadIdx.x == 0) *loss = __fdiv_rn(s, (float)B);
}

inline unsigned grid_for(int64_t items) {
    int64_t b = (items + kThreads - 1) / kThreads;
    const int64_t cap = (int64_t)tsb::num_sms() * 4;
    return (unsigned)(b > cap ? cap : (b < 1 ? 1 : b));
}

}  // namespace

extern "C" int ts_imitation_mse_rows(const float* z, const float* act, int64_t B, int32_t A, float max_action, float* dz, float* loss,
                                     ts_stream_t stream) {
    TS_REQUIRE(z && act && dz && loss && B >= 1 && A >= 1, "ts_imitation_mse_rows: bad argument");
    cudaStream_t st = tsb::as_stream(stream);
    const int64_t n = B * A;
    imitation_mse_grad_kernel<<<grid_for(n), kThreads, 0, st>>>(z, act, n, max_action, 2.0f / (float)n, dz);
    if (tsb::check_launch("ts_imitation_mse_rows")) return 1;
    imitation_mse_loss_kernel<<<1, tsb::kRowSumThreads, 0, st>>>(z, act, n, max_action, loss);
    return tsb::check_launch("ts_imitation_mse_rows/sum");
}

extern "C" int ts_imitation_nll_rows(const float* out, const int64_t* act, int64_t B, int32_t A, int32_t softmax_output, float* dz,
                                     float* rows, float* loss, ts_stream_t stream) {
    TS_REQUIRE(out && act && dz && rows && loss && B >= 1 && A >= 1, "ts_imitation_nll_rows: bad argument");
    cudaStream_t st = tsb::as_stream(stream);
    imitation_nll_rows_kernel<<<tsb::row_grid(B), kRowThreads, 0, st>>>(out, act, B, A, softmax_output ? 1 : 0, 1.0f / (float)B, dz,
                                                                        rows);
    if (tsb::check_launch("ts_imitation_nll_rows")) return 1;
    imitation_nll_loss_kernel<<<1, tsb::kRowSumThreads, 0, st>>>(rows, B, loss);
    return tsb::check_launch("ts_imitation_nll_rows/sum");
}
