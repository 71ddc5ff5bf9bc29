// FQF arithmetic (algorithm/modelfree/fqf.py, utils/net/discrete.py FractionProposalNetwork / FullQuantileFunction): the per-row
// pieces of the fraction proposal and the fraction loss that no IQN or layered-network launch provides -- the softmax, cumulative
// sum and entropy of the proposed fractions, the target at the arg-max of the fraction-weighted quantile mean, and the W1 fraction
// gradient back through the cumsum, the softmax and the entropy.  The quantile network itself runs on iqn.cu's kernels and the
// GEMMs of net_gemm.cu; the quantile-Huber rows are ts_iqn_rows with tau_hats as the per-row fractions.
//
// Reference: tianshou/utils/net/discrete.py:219-252 (FractionProposalNetwork.forward), :288-314 (FullQuantileFunction.forward),
// algorithm/modelfree/fqf.py:94-98 (the fraction-weighted action), :178-193 (the target), :221-247 (the fraction loss).
#include <float.h>
#include <math.h>

#include "common.cuh"
#include "quantile.cuh"
#include "row_sums.cuh"

namespace {

using tsb::argmax_before;
using tsb::kRowsPerBlock;
using tsb::kRowThreads;

constexpr int kFqfThreads = 128;
constexpr int kFqfWarps = kFqfThreads / 32;
constexpr int kFqfSmemFloats = 48 * 1024 / 4;     // the default dynamic shared-memory limit: one row's N fractions

unsigned fqf_row_grid(int64_t B) {
    const int64_t cap = (int64_t)tsb::num_sms() * 8;
    return (unsigned)(B < cap ? B : cap);
}

// fixed-order max over a CTA, every thread returns it (max is order-free, the fixed order only matters for a NaN)
__device__ __forceinline__ float block_max(float v, float* __restrict__ red) {
    v = tsb::warp_max(v);
    __syncthreads();
    if (tsb::lane_id() == 0) red[tsb::warp_id()] = v;
    __syncthreads();
    float m = red[0];
#pragma unroll
    for (int w = 1; w < kFqfWarps; ++w) m = fmaxf(m, red[w]);
    return m;
}

// One CTA per row b (grid-stride), threads over j = 0 .. N - 1.  With m = max_j z_j, e_j = exp(z_j - m), s = sum_j e_j:
//   logp[b][j] = max(z_j - (m + log s), -FLT_MAX)     (Categorical's normalised logits, clamped as its entropy clamps them)
//   p[b][j] = e_j / s                                  H[b] = -sum_j logp[b][j] * p[b][j]
//   taus[b][0] = 0, taus[b][k + 1] = fl32(sum_{j <= k} p_j)   (one thread, in order, accumulated in double as torch's CPU cumsum)
//   tau_hats[b][k] = (taus[b][k] + taus[b][k + 1]) / 2       inner[b][k] = taus[b][k + 1], k < N - 1
__global__ void __launch_bounds__(kFqfThreads) fqf_fractions_kernel(const float* __restrict__ z, int64_t B, int N,
                                                                    float* __restrict__ taus, float* __restrict__ tau_hats,
                                                                    float* __restrict__ inner, float* __restrict__ p,
                                                                    float* __restrict__ logp, float* __restrict__ H) {
    extern __shared__ float cum[];          // [N] this row's probabilities, then its cumulative sums
    __shared__ float red[kFqfWarps];
    const int tid = threadIdx.x;
    for (int64_t b = blockIdx.x; b < B; b += gridDim.x) {
        const float* zb = z + b * N;
        float m = -INFINITY;
        for (int j = tid; j < N; j += kFqfThreads) m = fmaxf(m, zb[j]);
        m = block_max(m, red);
        float se = 0.0f;
        for (int j = tid; j < N; j += kFqfThreads) se += expf(zb[j] - m);
        const float s = tsb::block_sum<kFqfWarps>(se, red);
        const float lse = m + logf(s);
        float h = 0.0f;
        for (int j = tid; j < N; j += kFqfThreads) {
            const float zj = zb[j];
            const float l = fmaxf(zj - lse, -FLT_MAX);
            const float pj = expf(zj - m) / s;
            p[b * N + j] = pj;
            logp[b * N + j] = l;
            cum[j] = pj;
            h += l * pj;
        }
        const float ent = -tsb::block_sum<kFqfWarps>(h, red);      // its barriers also publish cum
        if (tid == 0) {
            H[b] = ent;
            double acc = 0.0;
            for (int j = 0; j < N; ++j) {
                acc += (double)cum[j];
                cum[j] = (float)acc;
            }
        }
        __syncthreads();
        float* tb = taus + b * (N + 1);
        if (tid == 0) tb[0] = 0.0f;
        for (int j = tid; j < N; j += kFqfThreads) {
            const float hi = cum[j], lo = j > 0 ? cum[j - 1] : 0.0f;
            tb[j + 1] = hi;
            tau_hats[b * N + j] = (lo + hi) / 2.0f;
            if (j < N - 1) inner[b * (N - 1) + j] = hi;
        }
        __syncthreads();                    // the next row overwrites cum
    }
}

// Per row b: m_a = sum_n (taus[b][n + 1] - taus[b][n]) * q_online[b][n][a] (each width and product rounded in fp32, lanes over
// n, then the butterfly), a* = the first arg-max of m (NaN the maximum), out[b][n] = q_next[b][n][a*].  One warp per row.
__global__ void __launch_bounds__(kRowThreads) fqf_target_kernel(const float* __restrict__ q_online, const float* __restrict__ taus,
                                                                 const float* __restrict__ q_next, int64_t B, int A, int N,
                                                                 float* __restrict__ out, int64_t* __restrict__ act_out) {
    const int lane = tsb::lane_id();
    for (int64_t b = (int64_t)blockIdx.x * kRowsPerBlock + tsb::warp_id(); b < B; b += (int64_t)gridDim.x * kRowsPerBlock) {
        const float* qb = q_online + b * N * (int64_t)A;
        const float* tb = taus + b * (N + 1);
        float bv = 0.0f;
        int bi = -1;
        for (int a = 0; a < A; ++a) {
            float s = 0.0f;
            for (int n = lane; n < N; n += 32) s += __fmul_rn(__fsub_rn(tb[n + 1], tb[n]), qb[(int64_t)n * A + a]);
            const float m = tsb::warp_sum(s);
            if (argmax_before(m, a, bv, bi)) { bv = m; bi = a; }
        }
        const float* src = q_next + b * N * (int64_t)A + bi;
        for (int n = lane; n < N; n += 32) out[b * N + n] = src[(int64_t)n * A];
        if (lane == 0 && act_out) act_out[b] = bi;
    }
}

// One CTA per row b (grid-stride).  With h_n = q_hat[b][n][act] (at tau_hats) and c_i = q_tau[b][i][act] (at taus[i + 1]),
// i = 0 .. N - 2, the reference's strict sign tests give
//   g_i = (c_i > (i ? c_{i-1} : h_0) ? 1 : -1) (c_i - h_i) + (c_i < (i < N - 2 ? c_{i+1} : h_{N-1}) ? 1 : -1) (c_i - h_{i+1})
//   rows[0][b] = sum_i g_i taus[b][i + 1]     rows[1][b] = H[b]     rows[2][b] = 0
// and with G_j = sum_{i >= j} g_i (one thread, from the end, in double; G_{N-1} = 0), S = sum_j p_j G_j:
//   dz[b][j] = (1/B) p_j ((G_j - S) + ent_coef (logp_j + H[b]))      (0 where p_j == 0)
// the gradient of fraction_loss - ent_coef * mean_b H with respect to the fraction net's output z.
__global__ void __launch_bounds__(kFqfThreads) fqf_fraction_rows_kernel(
        const float* __restrict__ q_hat, const float* __restrict__ q_tau, const int64_t* __restrict__ act,
        const float* __restrict__ taus, const float* __restrict__ p, const float* __restrict__ logp, const float* __restrict__ H,
        int64_t B, int A, int N, float ent_coef, float inv_b, float* __restrict__ dz, float* __restrict__ rows) {
    extern __shared__ float gs[];           // [N] the row's g_i, then G_j
    __shared__ float red[kFqfWarps];
    const int tid = threadIdx.x;
    for (int64_t b = blockIdx.x; b < B; b += gridDim.x) {
        const int ab = (int)act[b];
        const float* hb = q_hat + b * N * (int64_t)A + ab;
        const float* cb = q_tau + b * (N - 1) * (int64_t)A + ab;
        const float* tb = taus + b * (N + 1);
        float fr = 0.0f;
        for (int i = tid; i < N - 1; i += kFqfThreads) {
            const float c = cb[(int64_t)i * A];
            const float hl = hb[(int64_t)i * A], hr = hb[(int64_t)(i + 1) * A];
            const float prev = i > 0 ? cb[(int64_t)(i - 1) * A] : hl;
            const float next = i < N - 2 ? cb[(int64_t)(i + 1) * A] : hr;
            const float v1 = c - hl, v2 = c - hr;
            const float g = (c > prev ? v1 : -v1) + (c < next ? v2 : -v2);
            gs[i] = g;
            fr += __fmul_rn(g, tb[i + 1]);
        }
        const float frac = tsb::block_sum<kFqfWarps>(fr, red);        // its barriers also publish gs
        const float hrow = H[b];
        if (tid == 0) {
            double acc = 0.0;
            gs[N - 1] = 0.0f;
            for (int j = N - 2; j >= 0; --j) {
                acc += (double)gs[j];
                gs[j] = (float)acc;
            }
            rows[b] = frac;
            rows[B + b] = hrow;
            rows[2 * B + b] = 0.0f;
        }
        __syncthreads();
        const float* pb = p + b * N;
        float sp = 0.0f;
        for (int j = tid; j < N; j += kFqfThreads) sp += pb[j] * gs[j];
        const float S = tsb::block_sum<kFqfWarps>(sp, red);
        const float* lb = logp + b * N;
        for (int j = tid; j < N; j += kFqfThreads) {
            const float pj = pb[j];
            dz[b * N + j] = pj > 0.0f ? inv_b * pj * ((gs[j] - S) + ent_coef * (lb[j] + hrow)) : 0.0f;
        }
        __syncthreads();                    // the next row overwrites gs
    }
}

}  // namespace

extern "C" int ts_fqf_fractions(const float* z, int64_t B, int32_t N, float* taus, float* tau_hats, float* inner, float* p,
                                float* logp, float* H, ts_stream_t stream) {
    TS_REQUIRE(z && taus && tau_hats && inner && p && logp && H && B >= 0 && N >= 2, "ts_fqf_fractions: bad argument");
    TS_REQUIRE(N <= kFqfSmemFloats, "ts_fqf_fractions: N = %d fractions need %d floats of shared memory, more than the %d a block "
               "holds", N, N, kFqfSmemFloats);
    if (B == 0) return 0;
    fqf_fractions_kernel<<<fqf_row_grid(B), kFqfThreads, (size_t)N * sizeof(float), tsb::as_stream(stream)>>>(
        z, B, N, taus, tau_hats, inner, p, logp, H);
    return tsb::check_launch("ts_fqf_fractions");
}

extern "C" int ts_fqf_target(const float* q_online, const float* taus, const float* q_next, int64_t B, int32_t A, int32_t N,
                             float* out, int64_t* act_out, ts_stream_t stream) {
    TS_REQUIRE(q_online && taus && q_next && out && B >= 0 && A >= 1 && N >= 1, "ts_fqf_target: bad argument");
    if (B == 0) return 0;
    fqf_target_kernel<<<tsb::row_grid(B), kRowThreads, 0, tsb::as_stream(stream)>>>(q_online, taus, q_next, B, A, N, out, act_out);
    return tsb::check_launch("ts_fqf_target");
}

extern "C" int ts_fqf_fraction_rows(const float* q_hat, const float* q_tau, const int64_t* act, const float* taus, const float* p,
                                    const float* logp, const float* H, int64_t B, int32_t A, int32_t N, float ent_coef, float* dz,
                                    float* rows, float* losses, ts_stream_t stream) {
    TS_REQUIRE(q_hat && q_tau && act && taus && p && logp && H && dz && rows && losses && B >= 1 && A >= 1 && N >= 2,
               "ts_fqf_fraction_rows: bad argument");
    TS_REQUIRE(N <= kFqfSmemFloats, "ts_fqf_fraction_rows: N = %d fractions need %d floats of shared memory, more than the %d a "
               "block holds", N, N, kFqfSmemFloats);
    TS_REQUIRE(isfinite(ent_coef), "ts_fqf_fraction_rows: ent_coef must be finite");
    cudaStream_t st = tsb::as_stream(stream);
    const float inv_b = 1.0f / (float)B;
    fqf_fraction_rows_kernel<<<fqf_row_grid(B), kFqfThreads, (size_t)N * sizeof(float), st>>>(q_hat, q_tau, act, taus, p, logp, H,
                                                                                              B, A, N, ent_coef, inv_b, dz, rows);
    if (tsb::check_launch("ts_fqf_fraction_rows")) return 1;
    tsb::row_sums3_kernel<<<1, tsb::kRowSumThreads, 0, st>>>(rows, B, inv_b, inv_b, inv_b, 1.0f, -ent_coef, 0.0f, losses);
    return tsb::check_launch("ts_fqf_fraction_rows/sums");
}
