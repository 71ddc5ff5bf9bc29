// Conservative Q-learning arithmetic (algorithm/imitation/cql.py): the per-row pieces between the critics' forward GEMMs and
// their parameter-gradient GEMMs.  The GEMMs themselves are the layered-network launches of net_gemm.cu; the actor step reuses
// SAC's kernels (net_ops.cu).
//
// Reference: tianshou/algorithm/imitation/cql.py:282-292 (one-step target), :295-300 (critic MSE), :303-319 (random,
// current-pi and next-pi blocks), :331-346 (calibration max), :348-365 (log-sum-exp penalty), :367-384 (Lagrange multiplier,
// critic losses).  torch.logsumexp (max-shifted, an infinite max replaced by 0), its backward exp(x - lse), and
// torch.maximum's backward (half the gradient to each side at a tie) are followed operation by operation.
#include <math.h>

#include "common.cuh"

namespace {

constexpr int kThreads = 256;

// torch.clamp(exp(log_alpha), alpha_min, alpha_max) (cql.py:370-374); 1 when there is no multiplier
__device__ __forceinline__ float multiplier(const float* log_alpha, float alpha_min, float alpha_max) {
    return log_alpha ? fminf(fmaxf(expf(*log_alpha), alpha_min), alpha_max) : 1.0f;
}

// One item per data row (t < B) or per block row (t - B < N = B * R).  q1 / q2: [B + 3N] critic outputs in the row order
// [data | random | current-pi | next-pi].
//   data row b   : sq_rows[k][b] = (q - y)^2;  dq = 2 (q - y) / B - scale w / B
//   block row i  : v_j = q_j - c_j (c = rand_logp, logp_cur[i], logp_next[i]); calibrated: v_j = max(v_j, cal_ret[i / R]);
//                  x_j = v_j / T; lse_rows[k][i] = logsumexp_j x_j;
//                  dq_j = (scale T w / N) exp(x_j - lse) / T * (1 | 1/2 | 0 by v_j >/==/< cal_ret)
// Every item is written when the grid is smaller than B + N (grid-stride loop).
__global__ void __launch_bounds__(kThreads) cql_rows_kernel(
        const float* __restrict__ q1, const float* __restrict__ q2, const float* __restrict__ target, int64_t B, int R,
        const float* __restrict__ logp_cur, const float* __restrict__ logp_next, float rand_logp, const float* __restrict__ cal_ret,
        float temperature, float cql_weight, const float* __restrict__ log_alpha, float alpha_min, float alpha_max,
        float* __restrict__ dq1, float* __restrict__ dq2, float* __restrict__ sq_rows, float* __restrict__ lse_rows) {
    const int64_t N = B * R;
    const float scale = multiplier(log_alpha, alpha_min, alpha_max);
    const float g_data = __fdiv_rn(__fmul_rn(scale, cql_weight), (float)B);
    const float g_lse = __fdiv_rn(__fmul_rn(__fmul_rn(scale, temperature), cql_weight), (float)N);
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < B + N; t += (int64_t)gridDim.x * blockDim.x) {
        if (t < B) {
            const float y = target[t];
            const float d1 = __fsub_rn(q1[t], y), d2 = __fsub_rn(q2[t], y);
            sq_rows[t] = __fmul_rn(d1, d1);
            sq_rows[B + t] = __fmul_rn(d2, d2);
            dq1[t] = __fsub_rn(__fdiv_rn(__fmul_rn(2.0f, d1), (float)B), g_data);
            dq2[t] = __fsub_rn(__fdiv_rn(__fmul_rn(2.0f, d2), (float)B), g_data);
            continue;
        }
        const int64_t i = t - B;
        const float c[3] = {rand_logp, logp_cur[i], logp_next[i]};
        const float r = cal_ret ? cal_ret[i / R] : 0.0f;
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            const float* q = k == 0 ? q1 : q2;
            float* dq = k == 0 ? dq1 : dq2;
            float x[3], mask[3];
#pragma unroll
            for (int j = 0; j < 3; ++j) {
                float v = __fsub_rn(q[B + j * N + i], c[j]);
                mask[j] = 1.0f;
                if (cal_ret) {
                    mask[j] = v > r ? 1.0f : (v == r ? 0.5f : 0.0f);
                    v = v < r ? r : v;
                }
                x[j] = __fdiv_rn(v, temperature);
            }
            const float mx = fmaxf(fmaxf(x[0], x[1]), x[2]);
            const float m = isinf(mx) ? 0.0f : mx;
            const float s = __fadd_rn(__fadd_rn(expf(__fsub_rn(x[0], m)), expf(__fsub_rn(x[1], m))), expf(__fsub_rn(x[2], m)));
            const float lse = __fadd_rn(logf(s), m);
            lse_rows[k * N + i] = lse;
#pragma unroll
            for (int j = 0; j < 3; ++j)
                dq[B + j * N + i] = __fmul_rn(__fdiv_rn(__fmul_rn(g_lse, expf(__fsub_rn(x[j], lse))), temperature), mask[j]);
        }
    }
}

constexpr int kLossThreads = 1024;
constexpr int kSums = 6;

// One block.  Fixed-order sums of (sq1, sq2, q1 data, q2 data, lse1, lse2), then per critic
//   penalty_k = mean(lse_k) * w * T - mean(q_k data) * w
//   Lagrange  : a = clamp(exp(log_alpha)); c_k = a (penalty_k - threshold); cql_alpha_loss = -(c1 + c2) * 0.5;
//               d cql_alpha_loss / d log_alpha = (-0.5 (penalty_1 - thr) - 0.5 (penalty_2 - thr)) * [min <= e <= max] * e
//   loss_k    = mean(sq_k) + (c_k or penalty_k)
// out[0..3] = (critic1 loss, critic2 loss, a, cql_alpha_loss); out[2..3] are left alone without a multiplier.
__global__ void __launch_bounds__(kLossThreads) cql_losses_kernel(
        const float* __restrict__ q1, const float* __restrict__ q2, const float* __restrict__ sq_rows,
        const float* __restrict__ lse_rows, int64_t B, int64_t N, float temperature, float cql_weight,
        const float* __restrict__ log_alpha, float alpha_min, float alpha_max, float threshold, float* __restrict__ grad_log_alpha,
        float* __restrict__ out) {
    __shared__ float part[kSums][kLossThreads / 32];
    float acc[kSums] = {0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f};
    for (int64_t b = threadIdx.x; b < B; b += kLossThreads) {
        acc[0] += sq_rows[b];
        acc[1] += sq_rows[B + b];
        acc[2] += q1[b];
        acc[3] += q2[b];
    }
    for (int64_t i = threadIdx.x; i < N; i += kLossThreads) {
        acc[4] += lse_rows[i];
        acc[5] += lse_rows[N + i];
    }
#pragma unroll
    for (int k = 0; k < kSums; ++k) {
        const float v = tsb::warp_sum(acc[k]);
        if (tsb::lane_id() == 0) part[k][tsb::warp_id()] = v;
    }
    __syncthreads();
    if (tsb::warp_id() != 0) return;
    float tot[kSums];
#pragma unroll
    for (int k = 0; k < kSums; ++k) tot[k] = tsb::warp_sum(part[k][tsb::lane_id()]);
    if (tsb::lane_id() != 0) return;
    float pen[2], loss[2];
    for (int k = 0; k < 2; ++k) {
        const float lse_mean = __fdiv_rn(tot[4 + k], (float)N), q_mean = __fdiv_rn(tot[2 + k], (float)B);
        pen[k] = __fsub_rn(__fmul_rn(__fmul_rn(lse_mean, cql_weight), temperature), __fmul_rn(q_mean, cql_weight));
        loss[k] = __fdiv_rn(tot[k], (float)B);
    }
    if (log_alpha) {
        const float e = expf(*log_alpha);
        const float a = fminf(fmaxf(e, alpha_min), alpha_max);
        const float p1 = __fsub_rn(pen[0], threshold), p2 = __fsub_rn(pen[1], threshold);
        const float c1 = __fmul_rn(a, p1), c2 = __fmul_rn(a, p2);
        loss[0] = __fadd_rn(loss[0], c1);
        loss[1] = __fadd_rn(loss[1], c2);
        out[2] = a;
        out[3] = __fmul_rn(-__fadd_rn(c1, c2), 0.5f);
        const float ga = __fadd_rn(__fmul_rn(-0.5f, p1), __fmul_rn(-0.5f, p2));
        *grad_log_alpha = (e >= alpha_min && e <= alpha_max) ? __fmul_rn(ga, e) : 0.0f;
    } else {
        loss[0] = __fadd_rn(loss[0], pen[0]);
        loss[1] = __fadd_rn(loss[1], pen[1]);
    }
    out[0] = loss[0];
    out[1] = loss[1];
}

// y = rew + logical_not(done) * gamma * (min(q1', q2') - alpha * logp)   (cql.py:282-292).  rew / done are the batch's fp32
// rows: to_torch(batch, dtype=torch.float) narrows the float64 rewards and turns the bool flags into 0 / 1.
__global__ void __launch_bounds__(kThreads) cql_target_kernel(
        const float* __restrict__ q1, const float* __restrict__ q2, const float* __restrict__ logp, float alpha,
        const float* __restrict__ rew, const float* __restrict__ done, float gamma, int64_t B, float* __restrict__ out) {
    for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b < B; b += (int64_t)gridDim.x * blockDim.x) {
        const float v = __fsub_rn(fminf(q1[b], q2[b]), __fmul_rn(alpha, logp[b]));
        const float nd = done[b] != 0.0f ? 0.0f : 1.0f;
        out[b] = __fadd_rn(rew[b], __fmul_rn(__fmul_rn(nd, gamma), v));
    }
}

inline unsigned grid_for(int64_t items) {
    int64_t b = (items + kThreads - 1) / kThreads;
    const int64_t cap = (int64_t)tsb::num_sms() * 4;
    return (unsigned)(b > cap ? cap : (b < 1 ? 1 : b));
}

}  // namespace

extern "C" int ts_cql_rows(const float* q1, const float* q2, const float* target, int64_t B, int32_t R, const float* logp_cur,
                           const float* logp_next, float rand_logp, const float* cal_ret, float temperature, float cql_weight,
                           const float* log_alpha, float alpha_min, float alpha_max, float* dq1, float* dq2, float* sq_rows,
                           float* lse_rows, ts_stream_t stream) {
    TS_REQUIRE(q1 && q2 && target && logp_cur && logp_next && dq1 && dq2 && sq_rows && lse_rows && B >= 1 && R >= 1,
               "ts_cql_rows: bad argument");
    cql_rows_kernel<<<grid_for(B + B * R), kThreads, 0, tsb::as_stream(stream)>>>(
        q1, q2, target, B, R, logp_cur, logp_next, rand_logp, cal_ret, temperature, cql_weight, log_alpha, alpha_min, alpha_max, dq1,
        dq2, sq_rows, lse_rows);
    return tsb::check_launch("ts_cql_rows");
}

extern "C" int ts_cql_losses(const float* q1, const float* q2, const float* sq_rows, const float* lse_rows, int64_t B, int64_t N,
                             float temperature, float cql_weight, const float* log_alpha, float alpha_min, float alpha_max,
                             float threshold, float* grad_log_alpha, float* out, ts_stream_t stream) {
    TS_REQUIRE(q1 && q2 && sq_rows && lse_rows && out && B >= 1 && N >= 1 && (!log_alpha || grad_log_alpha),
               "ts_cql_losses: bad argument");
    cql_losses_kernel<<<1, kLossThreads, 0, tsb::as_stream(stream)>>>(q1, q2, sq_rows, lse_rows, B, N, temperature, cql_weight,
                                                                       log_alpha, alpha_min, alpha_max, threshold, grad_log_alpha, out);
    return tsb::check_launch("ts_cql_losses");
}

extern "C" int ts_cql_target(const float* q1, const float* q2, const float* logp, float alpha, const float* rew, const float* done,
                             float gamma, int64_t B, float* out, ts_stream_t stream) {
    TS_REQUIRE(q1 && q2 && logp && rew && done && out && B >= 0, "ts_cql_target: bad argument");
    if (B == 0) return 0;
    cql_target_kernel<<<grid_for(B), kThreads, 0, tsb::as_stream(stream)>>>(q1, q2, logp, alpha, rew, done, gamma, B, out);
    return tsb::check_launch("ts_cql_target");
}
