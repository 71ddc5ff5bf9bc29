// Intrinsic curiosity module arithmetic (algorithm/modelbased/icm.py): the model inputs built from the feature rows, the per-row
// forward and inverse losses with their gradients, the intrinsic reward, and the feature gradient assembled from the three
// chains' backward passes.  Every GEMM is a layered-network launch of net_gemm.cu.
//
// Reference: tianshou/utils/net/discrete.py:377-428 (IntrinsicCuriosityModule.forward: phi1 = f(s), phi2 = f(s'),
// phi2_hat = forward_model([phi1 | one_hot(act)]), mse = 0.5 * ((phi2_hat - phi2)^2).sum(1), act_hat = inverse_model([phi1 | phi2])),
// tianshou/algorithm/modelbased/icm.py:77-109 (batch.rew += mse * reward_scale; loss = ((1 - w) CE(act_hat, act) + w mean(mse)) *
// lr_scale, phi2 not detached).
#include <math.h>

#include "common.cuh"
#include "row_sums.cuh"

namespace {

using tsb::kRowsPerBlock;
using tsb::kRowThreads;

constexpr int kThreads = 256;

// the action of row b in the dtype the batch holds it: int64 (off-policy device rows) or float32 (the on-policy rollout column)
__device__ __forceinline__ int icm_action(const void* act, int act_f32, int64_t b) {
    return act_f32 ? (int)static_cast<const float*>(act)[b] : (int)static_cast<const int64_t*>(act)[b];
}

// fwd_in [B][F + A] = [phi1 | one_hot(act)], inv_in [B][2F] = [phi1 | phi2], phi [2B][F] = [phi1 ; phi2].  Grid-stride over the
// B (3F + A) outputs.
__global__ void __launch_bounds__(kThreads) icm_inputs_kernel(const float* __restrict__ phi, const void* __restrict__ act, int act_f32,
                                                              int64_t B, int F, int A, float* __restrict__ fwd_in,
                                                              float* __restrict__ inv_in) {
    const int64_t wf = F + A, wr = wf + 2 * (int64_t)F;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < B * wr; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t b = e / wr, c = e - b * wr;
        if (c < wf) {
            fwd_in[b * wf + c] = c < F ? phi[b * F + c] : (c - F == icm_action(act, act_f32, b) ? 1.0f : 0.0f);
        } else {
            const int64_t k = c - wf;
            inv_in[b * 2 * F + k] = k < F ? phi[b * F + k] : phi[(B + b) * F + (k - F)];
        }
    }
}

// Per row b, one warp, lanes striding the F feature columns and the A action columns (any F, A):
//   mse[b] = 0.5 * sum_j (phi2_hat - phi2)^2;    ce[b] = logsumexp(act_hat[b]) - act_hat[b][act], max-shifted;
//   dphi2_hat[b] = gf (phi2_hat - phi2), gf = lr_scale w / B;   dphi[B + b] = -dphi2_hat[b] (phi2's direct term);
//   dact_hat[b] = gi (softmax(act_hat[b]) - onehot), gi = lr_scale (1 - w) / B;
//   rew_out[b] = rew_in[b] + (double)(mse[b] * reward_scale) when rew_out is given (fp32 product, float64 sum).
__global__ void __launch_bounds__(kRowThreads) icm_rows_kernel(const float* __restrict__ phi, const float* __restrict__ phi2_hat,
                                                               const float* __restrict__ act_hat, const void* __restrict__ act,
                                                               int act_f32, int64_t B, int F, int A, float gf, float gi,
                                                               const double* __restrict__ rew_in, float reward_scale,
                                                               double* __restrict__ rew_out, float* __restrict__ dphi,
                                                               float* __restrict__ dphi2_hat, float* __restrict__ dact_hat,
                                                               float* __restrict__ rows) {
    const int lane = tsb::lane_id();
    for (int64_t b = (int64_t)blockIdx.x * kRowsPerBlock + tsb::warp_id(); b < B; b += (int64_t)gridDim.x * kRowsPerBlock) {
        const float* p2 = phi + (B + b) * F;
        const float* ph = phi2_hat + b * F;
        float* dh = dphi2_hat + b * F;
        float* d2 = dphi + (B + b) * F;
        float sq = 0.0f;
        for (int j = lane; j < F; j += 32) {
            const float d = ph[j] - p2[j];
            sq += d * d;
            const float g = gf * d;
            dh[j] = g;
            d2[j] = -g;
        }
        const float mse = 0.5f * tsb::warp_sum(sq);
        const float* x = act_hat + b * A;
        float* dx = dact_hat + b * A;
        const int ab = icm_action(act, act_f32, b);
        float m = -INFINITY;
        for (int k = lane; k < A; k += 32) m = fmaxf(m, x[k]);
        m = tsb::warp_max(m);
        float s = 0.0f;
        for (int k = lane; k < A; k += 32) s += expf(x[k] - m);
        s = tsb::warp_sum(s);
        for (int k = lane; k < A; k += 32) dx[k] = gi * (expf(x[k] - m) / s - (k == ab ? 1.0f : 0.0f));
        if (lane == 0) {
            rows[b] = mse;
            rows[B + b] = logf(s) - (x[ab] - m);
            if (rew_out) rew_out[b] = rew_in[b] + (double)(mse * reward_scale);
        }
    }
}

// losses[1] = mean(mse), losses[2] = mean(ce), losses[0] = ((1 - w) losses[2] + w losses[1]) lr_scale: row_sums.cuh's fixed
// order, one block.
__global__ void __launch_bounds__(tsb::kRowSumThreads) icm_loss_kernel(const float* __restrict__ rows, int64_t B, float w,
                                                                       float lr_scale, float* __restrict__ losses) {
    const float fwd = tsb::block_sum_fixed(B, [&](int64_t b) { return rows[b]; }) / (float)B;    // each sum has its own array
    const float inv = tsb::block_sum_fixed(B, [&](int64_t b) { return rows[B + b]; }) / (float)B;
    if (threadIdx.x == 0) {
        losses[0] = ((1.0f - w) * inv + w * fwd) * lr_scale;
        losses[1] = fwd;
        losses[2] = inv;
    }
}

// dphi [2B][F]: rows b < B get dinv[b][0:F] + dfwd[b]; rows B + b add dinv[b][F:2F] to the direct term already there.  Then
// the derivative of the feature net's last activation (act: TS_ACT_*) at its output phi.  Grid-stride over 2 B F.
__global__ void __launch_bounds__(kThreads) icm_feature_grad_kernel(float* __restrict__ dphi, const float* __restrict__ dinv,
                                                                    const float* __restrict__ dfwd, const float* __restrict__ phi,
                                                                    int act, int64_t B, int F) {
    const int64_t half = B * F;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < 2 * half; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = e / F, j = e - r * F;
        float g = r < B ? dinv[r * 2 * F + j] + dfwd[e] : dphi[e] + dinv[(r - B) * 2 * F + F + j];
        if (act == TS_ACT_RELU) {
            g = phi[e] > 0.0f ? g : 0.0f;
        } else if (act == TS_ACT_TANH) {
            g *= 1.0f - phi[e] * phi[e];
        }
        dphi[e] = g;
    }
}

inline unsigned grid_for(int64_t items) {
    int64_t b = (items + kThreads - 1) / kThreads;
    const int64_t cap = (int64_t)tsb::num_sms() * 4;
    return (unsigned)(b > cap ? cap : (b < 1 ? 1 : b));
}

}  // namespace

extern "C" int ts_icm_inputs(const float* phi, const void* act, int32_t act_f32, int64_t B, int32_t F, int32_t A, float* fwd_in,
                             float* inv_in, ts_stream_t stream) {
    TS_REQUIRE(phi && act && fwd_in && inv_in && B >= 1 && F >= 1 && A >= 1, "ts_icm_inputs: bad argument");
    icm_inputs_kernel<<<grid_for(B * (3 * (int64_t)F + A)), kThreads, 0, tsb::as_stream(stream)>>>(phi, act, act_f32 ? 1 : 0, B, F, A,
                                                                                                   fwd_in, inv_in);
    return tsb::check_launch("ts_icm_inputs");
}

extern "C" int ts_icm_rows(const float* phi, const float* phi2_hat, const float* act_hat, const void* act, int32_t act_f32, int64_t B,
                           int32_t F, int32_t A, float lr_scale, float forward_loss_weight, const double* rew_in, float reward_scale,
                           double* rew_out, float* dphi, float* dphi2_hat, float* dact_hat, float* rows, float* losses,
                           ts_stream_t stream) {
    TS_REQUIRE(phi && phi2_hat && act_hat && act && dphi && dphi2_hat && dact_hat && rows && losses && B >= 1 && F >= 1 && A >= 1,
               "ts_icm_rows: bad argument");
    TS_REQUIRE(!rew_out || rew_in, "ts_icm_rows: rew_out needs rew_in");
    cudaStream_t st = tsb::as_stream(stream);
    const float w = forward_loss_weight;
    icm_rows_kernel<<<tsb::row_grid(B), kRowThreads, 0, st>>>(phi, phi2_hat, act_hat, act, act_f32 ? 1 : 0, B, F, A,
                                                              lr_scale * w / (float)B, lr_scale * (1.0f - w) / (float)B, rew_in,
                                                              reward_scale, rew_out, dphi, dphi2_hat, dact_hat, rows);
    if (tsb::check_launch("ts_icm_rows")) return 1;
    icm_loss_kernel<<<1, tsb::kRowSumThreads, 0, st>>>(rows, B, w, lr_scale, losses);
    return tsb::check_launch("ts_icm_rows/sum");
}

extern "C" int ts_icm_feature_grad(float* dphi, const float* dinv, const float* dfwd, const float* phi, int32_t act, int64_t B,
                                   int32_t F, ts_stream_t stream) {
    TS_REQUIRE(dphi && dinv && dfwd && B >= 1 && F >= 1, "ts_icm_feature_grad: bad argument");
    TS_REQUIRE(act == TS_ACT_NONE || ((act == TS_ACT_RELU || act == TS_ACT_TANH) && phi), "ts_icm_feature_grad: bad activation");
    icm_feature_grad_kernel<<<grid_for(2 * B * (int64_t)F), kThreads, 0, tsb::as_stream(stream)>>>(dphi, dinv, dfwd, phi, act, B, F);
    return tsb::check_launch("ts_icm_feature_grad");
}
