// Discrete CRR arithmetic (algorithm/imitation/discrete_crr.py): the per-row pieces between the actor / critic head GEMMs of
// the forward and their backward GEMMs.  The GEMMs themselves are the layered-network launches of net_gemm.cu.
//
// Reference: tianshou/algorithm/imitation/discrete_crr.py:131-143 (one-step target from the lagged actor and critic, critic
// loss), :145-155 (advantage, improvement coefficient, actor loss), :157-158 (CQL regulariser and the total).
#include <float.h>
#include <math.h>

#include "common.cuh"
#include "row_sums.cuh"

namespace {

using tsb::kRowsPerBlock;
using tsb::kRowThreads;

struct Softmax {
    float mx, sum, lse;
};

// max, sum exp(x - max) and torch.logsumexp (an infinite max replaced by 0 in the final add) of one row, over the warp
__device__ __forceinline__ Softmax row_softmax(const float* __restrict__ x, int A, int lane) {
    Softmax r;
    r.mx = -INFINITY;
    for (int a = lane; a < A; a += 32) r.mx = fmaxf(r.mx, x[a]);
    r.mx = tsb::warp_max(r.mx);
    float s = 0.0f;
    for (int a = lane; a < A; a += 32) s += expf(x[a] - r.mx);
    r.sum = tsb::warp_sum(s);
    r.lse = logf(r.sum) + (isinf(r.mx) ? 0.0f : r.mx);
    return r;
}

// Pass 0, per row b, with p = softmax(logits[b]), p' = softmax(logits_old[b]), qa = q[b][act[b]]:
//   target = rew[b] + gamma * (done[b] > 0 ? 0 : sum_a p'_a q_old[b][a])
//   S = sum_a p_a q_a, adv = qa - S
//   rows[0][b] = -log p[act];  rows[1][b] = coef = exp mode: clamp(exp(adv / beta), 0, bound); binary: 1[adv > 0]; all: 1
//   rows[2][b] = 0.5 (qa - target)^2;  rows[3][b] = logsumexp(q[b]) - qa
// The reference multiplies -log_prob [B] by the coefficient [B, 1] (discrete_crr.py:155): the product broadcasts to [B, B], so
// its actor loss is mean_b(-log p[act]) * mean_b(coef), not the mean of the per-row products.  Pass 1 therefore runs after the
// sums (means[0] = mean -log p[act], means[1] = mean coef) and writes the gradient of
// (means[0] * means[1] + mean rows[2] + cql_weight * mean rows[3]) as autograd takes it: the advantage is NOT detached, so in exp
// mode, where the clamp passes (0 <= exp(adv / beta) <= bound), g = means[0] * exp(adv / beta) / beta reaches q through
// d adv / d q_a = 1[a == act] - p_a and the logits through d adv / d z_a = -p_a (q_a - S).
template <bool kGrad>
__global__ void __launch_bounds__(kRowThreads) discrete_crr_rows_kernel(
        const float* __restrict__ q, const float* __restrict__ logits, const int64_t* __restrict__ act, const float* __restrict__ q_old,
        const float* __restrict__ logits_old, const float* __restrict__ rew, const float* __restrict__ done, int64_t B, int A, float gamma,
        int mode, float beta, float bound, float cql_weight, float inv_b, const float* __restrict__ means, float* __restrict__ dq,
        float* __restrict__ dlogits, float* __restrict__ rows) {
    const int lane = tsb::lane_id();
    for (int64_t b = (int64_t)blockIdx.x * kRowsPerBlock + tsb::warp_id(); b < B; b += (int64_t)gridDim.x * kRowsPerBlock) {
        const float* z = logits + b * A;
        const float* qr = q + b * A;
        const float* zo = logits_old + b * A;
        const float* qo = q_old + b * A;
        const int ab = (int)act[b];
        const float qa = qr[ab];

        const Softmax so = row_softmax(zo, A, lane);
        float eq = 0.0f;
        for (int a = lane; a < A; a += 32) eq += qo[a] * (expf(zo[a] - so.mx) / so.sum);
        eq = tsb::warp_sum(eq);
        if (done[b] > 0.0f) eq = 0.0f;
        const float err = qa - (rew[b] + gamma * eq);

        const Softmax sp = row_softmax(z, A, lane);
        const Softmax sq = row_softmax(qr, A, lane);
        float S = 0.0f;
        for (int a = lane; a < A; a += 32) S += qr[a] * (expf(z[a] - sp.mx) / sp.sum);
        S = tsb::warp_sum(S);
        const float adv = qa - S;
        float coef = 1.0f, dcoef = 0.0f;          // the coefficient and d coef / d adv
        if (mode == TS_CRR_BINARY) {
            coef = adv > 0.0f ? 1.0f : 0.0f;
        } else if (mode == TS_CRR_EXP) {
            const float e = expf(adv / beta);
            coef = fminf(fmaxf(e, 0.0f), bound);
            if (e >= 0.0f && e <= bound) dcoef = e / beta;
        }
        if (!kGrad) {
            if (lane == 0) {
                rows[b] = -(z[ab] - sp.lse);
                rows[B + b] = coef;
                rows[2 * B + b] = 0.5f * err * err;
                rows[3 * B + b] = sq.lse - qa;
            }
        } else {
            const float g = means[0] * dcoef, cbar = means[1];
            for (int a = lane; a < A; a += 32) {
                const float hit = a == ab ? 1.0f : 0.0f;
                const float p = expf(z[a] - sp.mx) / sp.sum;
                const float pq = expf(qr[a] - sq.mx) / sq.sum;
                dq[b * A + a] = (hit * err + g * (hit - p) + cql_weight * (pq - hit)) * inv_b;
                dlogits[b * A + a] = (cbar * (p - hit) - g * p * (qr[a] - S)) * inv_b;
            }
        }
    }
}

// rows [4][B] -> means[0..1] = mean rows[0], mean rows[1]; losses = (loss, actor, critic, cql).  One block, each thread sums its
// stride of rows in order, then a shared-memory tree: fixed order, bit-identical from run to run.
__global__ void __launch_bounds__(tsb::kRowSumThreads) discrete_crr_sums_kernel(const float* __restrict__ rows, int64_t B, float inv_b,
                                                                               float cql_weight, float* __restrict__ means,
                                                                               float* __restrict__ losses) {
    __shared__ float s[4][tsb::kRowSumThreads];
    float acc[4] = {0.0f, 0.0f, 0.0f, 0.0f};
    for (int64_t i = threadIdx.x; i < B; i += tsb::kRowSumThreads) {
#pragma unroll
        for (int k = 0; k < 4; ++k) acc[k] += rows[k * B + i];
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) s[k][threadIdx.x] = acc[k];
    __syncthreads();
    for (int off = tsb::kRowSumThreads / 2; off > 0; off >>= 1) {
        if ((int)threadIdx.x < off) {
#pragma unroll
            for (int k = 0; k < 4; ++k) s[k][threadIdx.x] += s[k][threadIdx.x + off];
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        const float nbar = s[0][0] * inv_b, cbar = s[1][0] * inv_b, critic = s[2][0] * inv_b, cql = s[3][0] * inv_b;
        means[0] = nbar;
        means[1] = cbar;
        losses[1] = nbar * cbar;
        losses[2] = critic;
        losses[3] = cql;
        losses[0] = nbar * cbar + critic + cql_weight * cql;
    }
}

}  // namespace

extern "C" int ts_discrete_crr_rows(const float* q, const float* logits, const int64_t* act, const float* q_old,
                                    const float* logits_old, const float* rew, const float* done, int64_t B, int32_t A, float gamma,
                                    int32_t mode, float beta, float ratio_upper_bound, float min_q_weight, float* dq, float* dlogits,
                                    float* rows, float* losses, ts_stream_t stream) {
    TS_REQUIRE(q && logits && act && q_old && logits_old && rew && done && dq && dlogits && rows && losses && B >= 1 && A >= 1,
               "ts_discrete_crr_rows: bad argument");
    TS_REQUIRE(mode == TS_CRR_EXP || mode == TS_CRR_BINARY || mode == TS_CRR_ALL, "ts_discrete_crr_rows: unknown mode %d", (int)mode);
    cudaStream_t st = tsb::as_stream(stream);
    const float inv_b = 1.0f / (float)B;
    const unsigned grid = tsb::row_grid(B);
    float* means = rows + 4 * B;
    discrete_crr_rows_kernel<false><<<grid, kRowThreads, 0, st>>>(q, logits, act, q_old, logits_old, rew, done, B, A, gamma, mode, beta,
                                                                 ratio_upper_bound, min_q_weight, inv_b, nullptr, dq, dlogits, rows);
    if (tsb::check_launch("ts_discrete_crr_rows")) return 1;
    discrete_crr_sums_kernel<<<1, tsb::kRowSumThreads, 0, st>>>(rows, B, inv_b, min_q_weight, means, losses);
    if (tsb::check_launch("ts_discrete_crr_rows/sums")) return 1;
    discrete_crr_rows_kernel<true><<<grid, kRowThreads, 0, st>>>(q, logits, act, q_old, logits_old, rew, done, B, A, gamma, mode, beta,
                                                                ratio_upper_bound, min_q_weight, inv_b, means, dq, dlogits, rows);
    return tsb::check_launch("ts_discrete_crr_rows/grad");
}
