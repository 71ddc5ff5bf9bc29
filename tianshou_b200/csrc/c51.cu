// C51 arithmetic (algorithm/modelfree/c51.py): the per-row pieces between the categorical network's forward GEMMs and its
// backward GEMMs.  The GEMMs are the layered-network launches of net_gemm.cu; the network's last Linear has A * N outputs, read
// here as raw logits [B][A][N] (action-major, atom-minor).  The softmax over each action's N atoms, which the reference's
// model applies, belongs to these kernels.
//
// Reference: tianshou/algorithm/modelfree/c51.py:62-63 (the action value is sum_k p_k z_k), :113-136 (the target distribution at
// the online arg-max, the clamp and the dense projection), :143-160 (the cross-entropy with 1e-8 inside the log, the weighted
// mean, the unweighted priority).
#include <float.h>
#include <math.h>

#include "common.cuh"
#include "quantile.cuh"
#include "row_sums.cuh"

namespace {

using tsb::argmax_before;
using tsb::kRowsPerBlock;
using tsb::kRowThreads;

constexpr int kC51Threads = 128;
constexpr int kC51Warps = kC51Threads / 32;
constexpr int kC51SmemFloats = 48 * 1024 / 4;     // the default dynamic shared-memory limit: 4 arrays of N floats

// softmax over x[0..N) on one warp: (max, sum_k exp(x_k - max)); every lane returns the same pair
__device__ __forceinline__ void warp_softmax_stats(const float* __restrict__ x, int N, int lane, float& mx, float& s) {
    float m = -INFINITY;
    for (int k = lane; k < N; k += 32) m = fmaxf(m, x[k]);
    mx = tsb::warp_max(m);
    float a = 0.0f;
    for (int k = lane; k < N; k += 32) a += expf(x[k] - mx);
    s = tsb::warp_sum(a);
}

// Per row b: p_a = softmax(logits_online[b][a]), Q_a = sum_k p_ak z_k, a* = the first arg-max of Q (NaN the maximum),
// next_dist[b] = softmax(logits_next[b][a*]).  One warp per row.
__global__ void __launch_bounds__(kRowThreads) c51_target_kernel(const float* __restrict__ lo, const float* __restrict__ ln,
                                                                 const float* __restrict__ z, int64_t B, int A, int N,
                                                                 float* __restrict__ next_dist, int64_t* __restrict__ act_out) {
    const int lane = tsb::lane_id();
    const int64_t AN = (int64_t)A * N;
    for (int64_t b = (int64_t)blockIdx.x * kRowsPerBlock + tsb::warp_id(); b < B; b += (int64_t)gridDim.x * kRowsPerBlock) {
        float bv = 0.0f;
        int bi = -1;
        for (int a = 0; a < A; ++a) {
            const float* x = lo + b * AN + (int64_t)a * N;
            float mx, s;
            warp_softmax_stats(x, N, lane, mx, s);
            float q = 0.0f;
            for (int k = lane; k < N; k += 32) q += (expf(x[k] - mx) / s) * z[k];
            q = tsb::warp_sum(q);
            if (argmax_before(q, a, bv, bi)) { bv = q; bi = a; }
        }
        const float* x = ln + b * AN + (int64_t)bi * N;
        float mx, s;
        warp_softmax_stats(x, N, lane, mx, s);
        for (int k = lane; k < N; k += 32) next_dist[b * N + k] = expf(x[k] - mx) / s;
        if (lane == 0 && act_out) act_out[b] = bi;
    }
}

// fixed-order max over a CTA of kWarps warps (the companion of tsb::block_sum); red holds kWarps floats
__device__ __forceinline__ float block_max(float v, float* __restrict__ red) {
    v = tsb::warp_max(v);
    __syncthreads();
    if (tsb::lane_id() == 0) red[tsb::warp_id()] = v;
    __syncthreads();
    float m = red[0];
#pragma unroll
    for (int w = 1; w < kC51Warps; ++w) m = fmaxf(m, red[w]);
    return m;
}

// One CTA per row b (grid-stride), threads over the atoms j.  With t_k = clamp(returns[b][k], v_min, v_max),
// target_j = sum_k clamp(1 - |t_k - z_j| / delta_z, 0, 1) next_dist[b][k]   (k in order), p = softmax(logits[b][act_b]):
//   CE_b = -sum_j target_j log(p_j + 1e-8)        rows[0][b] = w_b CE_b, rows[1][b] = prio[b] = CE_b, rows[2][b] = 0
//   pg_j = -(w_b / B) target_j p_j / (p_j + 1e-8)  (= p_j g_j with g_j = d loss / d p_j)
//   dlogits[b][act_b][j] = pg_j - p_j sum_i pg_i, every other block of the row 0.
__global__ void __launch_bounds__(kC51Threads) c51_rows_kernel(
        const float* __restrict__ logits, const int64_t* __restrict__ act, const float* __restrict__ returns,
        const float* __restrict__ z, float v_min, float v_max, float delta_z, const float* __restrict__ next_dist,
        const float* __restrict__ weight, int64_t B, int A, int N, float inv_b, float* __restrict__ dlogits,
        float* __restrict__ prio, float* __restrict__ rows) {
    extern __shared__ float smem[];
    float* t = smem;                // [N] clamped returns
    float* nd = smem + N;           // [N] next_dist
    float* tg = smem + 2 * N;       // [N] projected target
    float* p = smem + 3 * N;        // [N] current probabilities
    __shared__ float red[kC51Warps];
    const int tid = threadIdx.x;
    const int64_t AN = (int64_t)A * N;
    for (int64_t b = blockIdx.x; b < B; b += gridDim.x) {
        const int ab = (int)act[b];
        const float* x = logits + b * AN + (int64_t)ab * N;
        float* db = dlogits + b * AN;
        const float wb = weight ? weight[b] : 1.0f;
        __syncthreads();                    // the previous row is done with the shared arrays
        float m = -INFINITY;
        for (int k = tid; k < N; k += kC51Threads) {
            t[k] = fminf(fmaxf(returns[b * N + k], v_min), v_max);
            nd[k] = next_dist[b * N + k];
            m = fmaxf(m, x[k]);
        }
        for (int64_t e = tid; e < AN; e += kC51Threads)
            if ((int)(e / N) != ab) db[e] = 0.0f;
        const float mx = block_max(m, red);         // its barriers also publish t and nd
        float se = 0.0f;
        for (int j = tid; j < N; j += kC51Threads) {
            const float zj = z[j];
            float acc = 0.0f;
            for (int k = 0; k < N; ++k) acc += fminf(fmaxf(1.0f - fabsf(t[k] - zj) / delta_z, 0.0f), 1.0f) * nd[k];
            tg[j] = acc;
            const float e = expf(x[j] - mx);
            p[j] = e;
            se += e;
        }
        const float s = tsb::block_sum<kC51Warps>(se, red);
        const float gs = -wb * inv_b;
        float ce = 0.0f, spg = 0.0f;
        for (int j = tid; j < N; j += kC51Threads) {
            const float pj = p[j] / s;
            p[j] = pj;
            const float pe = pj + 1e-8f;
            ce -= tg[j] * logf(pe);
            spg += gs * tg[j] * (pj / pe);
        }
        const float ce_b = tsb::block_sum<kC51Warps>(ce, red);
        const float sum_pg = tsb::block_sum<kC51Warps>(spg, red);
        for (int j = tid; j < N; j += kC51Threads) {
            const float pj = p[j];
            db[(int64_t)ab * N + j] = gs * tg[j] * (pj / (pj + 1e-8f)) - pj * sum_pg;
        }
        if (tid == 0) {
            rows[b] = wb * ce_b;
            rows[B + b] = ce_b;
            rows[2 * B + b] = 0.0f;
            prio[b] = ce_b;
        }
    }
}

}  // namespace

extern "C" int ts_c51_target(const float* logits_online, const float* logits_next, const float* support, int64_t B, int32_t A,
                             int32_t N, float* next_dist, int64_t* act_out, ts_stream_t stream) {
    TS_REQUIRE(logits_online && logits_next && support && next_dist && B >= 0 && A >= 1 && N >= 2, "ts_c51_target: bad argument");
    if (B == 0) return 0;
    c51_target_kernel<<<tsb::row_grid(B), kRowThreads, 0, tsb::as_stream(stream)>>>(logits_online, logits_next, support, B, A, N,
                                                                                      next_dist, act_out);
    return tsb::check_launch("ts_c51_target");
}

extern "C" int ts_c51_rows(const float* logits, const int64_t* act, const float* returns, const float* support, float v_min,
                           float v_max, float delta_z, const float* next_dist, const float* weight, int64_t B, int32_t A, int32_t N,
                           float* dlogits, float* prio, float* rows, float* losses, ts_stream_t stream) {
    TS_REQUIRE(logits && act && returns && support && next_dist && dlogits && prio && rows && losses && B >= 1 && A >= 1 && N >= 2 &&
               delta_z > 0.0f && v_min <= v_max, "ts_c51_rows: bad argument");
    const int64_t smem_floats = 4 * (int64_t)N;
    TS_REQUIRE(smem_floats <= kC51SmemFloats, "ts_c51_rows: N = %d atoms need %lld floats of shared memory, more than the %d a "
               "block holds", N, (long long)smem_floats, kC51SmemFloats);
    cudaStream_t st = tsb::as_stream(stream);
    const float inv_b = 1.0f / (float)B;
    const int64_t cap = (int64_t)tsb::num_sms() * 8;
    const unsigned grid = (unsigned)(B < cap ? B : cap);
    c51_rows_kernel<<<grid, kC51Threads, smem_floats * sizeof(float), st>>>(logits, act, returns, support, v_min, v_max, delta_z,
                                                                            next_dist, weight, B, A, N, inv_b, dlogits, prio, rows);
    if (tsb::check_launch("ts_c51_rows")) return 1;
    tsb::row_sums3_kernel<<<1, tsb::kRowSumThreads, 0, st>>>(rows, B, inv_b, inv_b, inv_b, 1.0f, 0.0f, 0.0f, losses);
    return tsb::check_launch("ts_c51_rows/sums");
}
