// Discrete soft actor-critic arithmetic (algorithm/modelfree/discrete_sac.py): the per-row categorical pieces between the
// actor / critic forward GEMMs and the actor's backward GEMMs.  The GEMMs themselves are the layered-network launches of
// net_gemm.cu; the critics' squared loss is ts_dqn_loss (net_ops.cu).
//
// Reference: tianshou/algorithm/modelfree/discrete_sac.py:147-155 (target value sum_a pi(a|s') min(Q1', Q2')(s', a) +
// alpha H(pi(.|s'))), :176-184 (actor loss -(alpha H + sum_a pi(a|s) min(Q1, Q2)(s, a)).mean() and its gradient), torch's
// Categorical(logits=...) (distributions/categorical.py: logits - logsumexp, softmax probs, entropy
// -sum(clamp(logits, finfo.min) * probs)).
#include <float.h>
#include <math.h>

#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kRowsPerBlock = kThreads / 32;      // one warp per row

// Per row b, with z = logits[b], m = min(q1[b], q2[b]), p = softmax(z), log p = z - logsumexp(z):
//   probs[b]   = p
//   entropy[b] = H = -sum_a clamp(log p_a, -FLT_MAX) * p_a
//   v[b]       = sum_a p_a m_a + alpha H
//   dlogits[b] = scale * d(-v[b]) / dz = scale * (alpha p (log p + H) - p (m - sum_a p_a m_a))      (when not NULL)
// A row whose p_a underflows to 0 contributes 0 * finite = 0 for that action, never NaN.  Lanes stride over the A actions, so
// any A >= 1 works; warps stride over the rows, so every row is written when B exceeds the launch grid.
__global__ void __launch_bounds__(kThreads) discrete_sac_rows_kernel(
        const float* __restrict__ logits, const float* __restrict__ q1, const float* __restrict__ q2, float alpha, int64_t B, int A,
        float* __restrict__ v, float* __restrict__ entropy, float* __restrict__ probs, float* __restrict__ dlogits, float scale) {
    const int lane = tsb::lane_id();
    for (int64_t b = (int64_t)blockIdx.x * kRowsPerBlock + tsb::warp_id(); b < B; b += (int64_t)gridDim.x * kRowsPerBlock) {
        const float* z = logits + b * A;
        const float* qa = q1 + b * A;
        const float* qb = q2 + b * A;
        float* p_out = probs + b * A;
        float mx = -INFINITY;
        for (int a = lane; a < A; a += 32) mx = fmaxf(mx, z[a]);
        mx = tsb::warp_max(mx);
        float s = 0.0f;
        for (int a = lane; a < A; a += 32) s += expf(z[a] - mx);
        s = tsb::warp_sum(s);
        // torch.logsumexp: log(sum(exp(z - max))) + max, with an infinite max replaced by 0 in the final add
        const float lse = logf(s) + (isinf(mx) ? 0.0f : mx);
        float plogp = 0.0f, pm = 0.0f;
        for (int a = lane; a < A; a += 32) {
            const float p = expf(z[a] - mx) / s;
            const float lp = fmaxf(z[a] - lse, -FLT_MAX);
            p_out[a] = p;
            plogp += lp * p;
            pm += p * fminf(qa[a], qb[a]);
        }
        const float H = -tsb::warp_sum(plogp);
        const float S = tsb::warp_sum(pm);
        if (lane == 0) {
            entropy[b] = H;
            v[b] = S + alpha * H;
        }
        if (dlogits) {
            float* d = dlogits + b * A;
            for (int a = lane; a < A; a += 32) {
                const float p = p_out[a];          // written by this lane above
                const float lp = fmaxf(z[a] - lse, -FLT_MAX);
                d[a] = scale * (alpha * p * (lp + H) - p * (fminf(qa[a], qb[a]) - S));
            }
        }
    }
}

inline unsigned row_grid(int64_t rows) {
    int64_t b = (rows + kRowsPerBlock - 1) / kRowsPerBlock;
    const int64_t cap = (int64_t)tsb::num_sms() * 16;
    return (unsigned)(b > cap ? cap : (b < 1 ? 1 : b));
}

}  // namespace

extern "C" int ts_discrete_sac_rows(const float* logits, const float* q1, const float* q2, float alpha, int64_t B, int32_t A, float* v,
                                    float* entropy, float* probs, float* dlogits, float dlogit_scale, ts_stream_t stream) {
    TS_REQUIRE(logits && q1 && q2 && v && entropy && probs && B >= 0 && A >= 1, "ts_discrete_sac_rows: bad argument");
    if (B == 0) return 0;
    discrete_sac_rows_kernel<<<row_grid(B), kThreads, 0, tsb::as_stream(stream)>>>(logits, q1, q2, alpha, B, A, v, entropy, probs,
                                                                                    dlogits, dlogit_scale);
    return tsb::check_launch("ts_discrete_sac_rows");
}
