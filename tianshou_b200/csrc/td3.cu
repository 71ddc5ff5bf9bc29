// TD3 / TD3+BC arithmetic (algorithm/modelfree/td3.py, algorithm/imitation/td3_bc.py): the per-row pieces between the GEMMs of
// the deterministic actor and the critics.  The GEMMs themselves are the layered-network launches of net_gemm.cu; the critics'
// squared-loss step reuses ts_critic_mse (net_ops.cu).
//
// Reference: tianshou/utils/net/continuous.py:84 (a = max_action * tanh(last(...))), algorithm/modelfree/td3.py:94-102 (min of
// the lagged critics), :190-202 (target-policy smoothing noise, not clipped back to the action bounds), :214-219 (actor loss
// -mean Q1(s, pi(s))), imitation/td3_bc.py:113-120 (lmbda = alpha / mean|Q|, detached, plus F.mse_loss(pi(s), a)).  Where the
// rounding order matters it follows torch's operation order with __f*_rn, as cql.cu does.
#include <math.h>

#include "common.cuh"

namespace {

constexpr int kThreads = 256;

// x = [s | a] with a = max_action * tanh(z) (+ clamp(noise * policy_noise, +-noise_clip) when noise is given; the clamp is
// skipped when noise_clip <= 0).  One item per element of x, grid-stride.
__global__ void __launch_bounds__(kThreads) td3_act_rows_kernel(
        const float* __restrict__ z, const float* __restrict__ noise, int64_t B, int A, float max_action, float policy_noise,
        float noise_clip, const float* __restrict__ obs, int O, float* __restrict__ x) {
    const int W = O + A;
    const int64_t n = B * W;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) {
        const int64_t b = t / W;
        const int c = (int)(t - b * W);
        if (c < O) {
            x[t] = obs[b * O + c];
            continue;
        }
        const int64_t e = b * A + (c - O);
        float a = __fmul_rn(max_action, tanhf(z[e]));
        if (noise) {
            float d = __fmul_rn(noise[e], policy_noise);
            if (noise_clip > 0.0f) d = fminf(fmaxf(d, -noise_clip), noise_clip);
            a = __fadd_rn(a, d);
        }
        x[t] = a;
    }
}

// torch.min(q1, q2) elementwise (NaN propagates), grid-stride
__global__ void __launch_bounds__(kThreads) td3_target_min_kernel(const float* __restrict__ q1, const float* __restrict__ q2,
                                                                 int64_t B, float* __restrict__ out) {
    for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b < B; b += (int64_t)gridDim.x * blockDim.x) {
        const float u = q1[b], v = q2[b];
        out[b] = (u != u || v != v) ? __fadd_rn(u, v) : fminf(u, v);
    }
}

constexpr int kRowThreads = 1024;
constexpr int kSums = 3;

// One block.  Fixed-order sums of (q, |q|, (pi - a)^2), then
//   TD3    : loss = -(sum q / B);                                     dq = -1 / B
//   TD3+BC : lmbda = alpha * (1 / (sum |q| / B)); loss = -lmbda * (sum q / B) + sum (pi - a)^2 / (B A);  dq = -lmbda / B
// (alpha / t is torch's reciprocal(t) * alpha).  pi = max_action * tanh(z) as td3_act_rows_kernel computes it.  Every row of dq
// is written (block-stride).
__global__ void __launch_bounds__(kRowThreads) td3_actor_rows_kernel(
        const float* __restrict__ q, const float* __restrict__ z, const float* __restrict__ act, int64_t B, int A, float max_action,
        float alpha, float* __restrict__ dq, float* __restrict__ loss) {
    __shared__ float part[kSums][kRowThreads / 32];
    __shared__ float dq_row;
    float acc[kSums] = {0.0f, 0.0f, 0.0f};
    for (int64_t b = threadIdx.x; b < B; b += kRowThreads) {
        acc[0] += q[b];
        acc[1] += fabsf(q[b]);
    }
    if (act) {
        for (int64_t e = threadIdx.x; e < B * A; e += kRowThreads) {
            const float d = __fsub_rn(__fmul_rn(max_action, tanhf(z[e])), act[e]);
            acc[2] = __fadd_rn(acc[2], __fmul_rn(d, d));
        }
    }
#pragma unroll
    for (int k = 0; k < kSums; ++k) {
        const float v = tsb::warp_sum(acc[k]);
        if (tsb::lane_id() == 0) part[k][tsb::warp_id()] = v;
    }
    __syncthreads();
    if (tsb::warp_id() == 0) {
        float tot[kSums];
#pragma unroll
        for (int k = 0; k < kSums; ++k) tot[k] = tsb::warp_sum(part[k][tsb::lane_id()]);
        if (tsb::lane_id() == 0) {
            const float q_mean = __fdiv_rn(tot[0], (float)B);
            if (act) {
                const float lmbda = __fmul_rn(__frcp_rn(__fdiv_rn(tot[1], (float)B)), alpha);
                const float mse = __fdiv_rn(tot[2], (float)(B * A));
                *loss = __fadd_rn(__fmul_rn(-lmbda, q_mean), mse);
                dq_row = __fdiv_rn(-lmbda, (float)B);
            } else {
                *loss = -q_mean;
                dq_row = __fdiv_rn(-1.0f, (float)B);
            }
        }
    }
    __syncthreads();
    const float g = dq_row;
    for (int64_t b = threadIdx.x; b < B; b += kRowThreads) dq[b] = g;
}

// dz = (dact + [act] 2 (pi - a) / (B A)) * max_action * (1 - t^2), t = tanh(z): the backward of pi = max_action * tanh(z) and of
// TD3+BC's F.mse_loss(pi, a).  Grid-stride over B * A.
__global__ void __launch_bounds__(kThreads) td3_actor_head_bwd_kernel(
        const float* __restrict__ z, const float* __restrict__ dact, const float* __restrict__ act, int64_t B, int A,
        float max_action, float* __restrict__ dz) {
    const int64_t n = B * A;
    const float inv_n = __fdiv_rn(2.0f, (float)n);
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
        const float t = tanhf(z[e]);
        float g = dact[e];
        if (act) g = __fadd_rn(g, __fmul_rn(__fsub_rn(__fmul_rn(max_action, t), act[e]), inv_n));
        dz[e] = __fmul_rn(__fmul_rn(g, max_action), __fsub_rn(1.0f, __fmul_rn(t, t)));
    }
}

inline unsigned grid_for(int64_t items) {
    int64_t b = (items + kThreads - 1) / kThreads;
    const int64_t cap = (int64_t)tsb::num_sms() * 4;
    return (unsigned)(b > cap ? cap : (b < 1 ? 1 : b));
}

}  // namespace

extern "C" int ts_td3_act_rows(const float* z, const float* noise, int64_t B, int32_t A, float max_action, float policy_noise,
                               float noise_clip, const float* obs, int32_t O, float* x, ts_stream_t stream) {
    TS_REQUIRE(z && obs && x && B >= 0 && A >= 1 && O >= 0, "ts_td3_act_rows: bad argument");
    if (B == 0) return 0;
    td3_act_rows_kernel<<<grid_for(B * (O + A)), kThreads, 0, tsb::as_stream(stream)>>>(z, noise, B, A, max_action, policy_noise,
                                                                                      noise_clip, obs, O, x);
    return tsb::check_launch("ts_td3_act_rows");
}

extern "C" int ts_td3_target_min(const float* q1, const float* q2, int64_t B, float* out, ts_stream_t stream) {
    TS_REQUIRE(q1 && q2 && out && B >= 0, "ts_td3_target_min: bad argument");
    if (B == 0) return 0;
    td3_target_min_kernel<<<grid_for(B), kThreads, 0, tsb::as_stream(stream)>>>(q1, q2, B, out);
    return tsb::check_launch("ts_td3_target_min");
}

extern "C" int ts_td3_actor_rows(const float* q, const float* z, const float* act, int64_t B, int32_t A, float max_action,
                                 float alpha, float* dq, float* loss, ts_stream_t stream) {
    TS_REQUIRE(q && dq && loss && B >= 1 && A >= 1 && (!act || z), "ts_td3_actor_rows: bad argument");
    td3_actor_rows_kernel<<<1, kRowThreads, 0, tsb::as_stream(stream)>>>(q, z, act, B, A, max_action, alpha, dq, loss);
    return tsb::check_launch("ts_td3_actor_rows");
}

extern "C" int ts_td3_actor_head_bwd(const float* z, const float* dact, const float* act, int64_t B, int32_t A, float max_action,
                                     float* dz, ts_stream_t stream) {
    TS_REQUIRE(z && dact && dz && B >= 0 && A >= 1, "ts_td3_actor_head_bwd: bad argument");
    if (B == 0) return 0;
    td3_actor_head_bwd_kernel<<<grid_for(B * A), kThreads, 0, tsb::as_stream(stream)>>>(z, dact, act, B, A, max_action, dz);
    return tsb::check_launch("ts_td3_actor_head_bwd");
}
