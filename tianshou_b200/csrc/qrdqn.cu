// QR-DQN and discrete CQL arithmetic (algorithm/modelfree/qrdqn.py, algorithm/imitation/discrete_cql.py): the per-row pieces
// between the quantile network's forward GEMMs and its backward GEMMs.  The GEMMs themselves are the layered-network launches of
// net_gemm.cu; the network's last Linear has A * N outputs, read here as [B][A][N] (action-major, quantile-minor).
//
// Reference: tianshou/algorithm/modelfree/qrdqn.py:18-20 (the action value is the quantile mean), :94-106 (the target
// distribution at the online arg-max), :108-131 (quantile-Huber loss, the priority); imitation/discrete_cql.py:80-113 (the
// same loss plus the log-sum-exp penalty over the quantile means).
#include <float.h>
#include <math.h>

#include "common.cuh"
#include "row_sums.cuh"

namespace {

using tsb::kRowsPerBlock;
using tsb::kRowThreads;

constexpr int kQrThreads = 256;
constexpr int kQrWarps = kQrThreads / 32;
constexpr int kQrSmemFloats = 48 * 1024 / 4;     // the default dynamic shared-memory limit: N targets, N taus, A means

// torch.argmax's order on (value, index): a NaN is the maximum, ties go to the lowest index (as in discrete_bcq.cu)
__device__ __forceinline__ bool argmax_before(float v, int i, float bv, int bi) {
    if (bi < 0) return true;
    const bool vn = isnan(v), bn = isnan(bv);
    if (vn || bn) return vn && (!bn || i < bi);
    return v > bv || (v == bv && i < bi);
}

// mean of x[0 .. N) over one warp: every lane adds its stride in order, then the butterfly; every lane returns the same value,
// and two equal rows give equal means
__device__ __forceinline__ float quantile_mean(const float* __restrict__ x, int N, int lane) {
    float s = 0.0f;
    for (int k = lane; k < N; k += 32) s += x[k];
    return tsb::warp_sum(s) / (float)N;
}

// Per row b: m_a = mean_k q_online[b][a][k], a* = the first arg-max of m (NaN the maximum), out[b][k] = q_next[b][a*][k].
// One warp per row.
__global__ void __launch_bounds__(kRowThreads) qrdqn_target_kernel(const float* __restrict__ q_online, const float* __restrict__ q_next,
                                                                   int64_t B, int A, int N, float* __restrict__ out,
                                                                   int64_t* __restrict__ act_out) {
    const int lane = tsb::lane_id();
    const int64_t AN = (int64_t)A * N;
    for (int64_t b = (int64_t)blockIdx.x * kRowsPerBlock + tsb::warp_id(); b < B; b += (int64_t)gridDim.x * kRowsPerBlock) {
        float bv = 0.0f;
        int bi = -1;
        for (int a = 0; a < A; ++a) {
            const float m = quantile_mean(q_online + b * AN + (int64_t)a * N, N, lane);
            if (argmax_before(m, a, bv, bi)) { bv = m; bi = a; }
        }
        const float* src = q_next + b * AN + (int64_t)bi * N;
        for (int k = lane; k < N; k += 32) out[b * N + k] = src[k];
        if (lane == 0 && act_out) act_out[b] = bi;
    }
}

// fixed-order sum over the CTA: the warp butterfly, then warp 0 adds the per-warp values in order.  Every thread returns it.
__device__ __forceinline__ float block_sum(float v, float* __restrict__ red) {
    v = tsb::warp_sum(v);
    __syncthreads();                         // red may still be read by the previous call
    if (tsb::lane_id() == 0) red[tsb::warp_id()] = v;
    __syncthreads();
    float s = 0.0f;
#pragma unroll
    for (int w = 0; w < kQrWarps; ++w) s += red[w];
    return s;
}

// One CTA per row b (grid-stride), threads over the current quantiles i.  With c_i = q[b][act][i], t = returns[b],
// u_ij = t_j - c_i, h_ij = smooth_l1(u_ij) (beta 1) and w_ij = |tau_i - 1[u_ij <= 0]|:
//   rows[0][b] = weight_b * (1/N) sum_i sum_j h_ij w_ij          rows[2][b] = prio[b] = (1/N) sum_i sum_j h_ij
//   rows[1][b] = logsumexp_a m_a - m_act  (m_a = mean_k q[b][a][k]; only with cql_scale != 0, else 0)
//   dq[b][a][k] = cql_scale (softmax(m)_a - 1[a == act])  +  1[a == act] * (-qr_scale weight_b sum_j w_kj clip(u_kj, -1, 1))
// qr_scale = 1 / (B N), cql_scale = min_q_weight / (B N).  The indicator carries no gradient (the reference detaches it).
__global__ void __launch_bounds__(kQrThreads) qrdqn_rows_kernel(
        const float* __restrict__ q, const int64_t* __restrict__ act, const float* __restrict__ returns, const float* __restrict__ tau_hat,
        const float* __restrict__ weight, int64_t B, int A, int N, float qr_scale, float cql_scale, float* __restrict__ dq,
        float* __restrict__ prio, float* __restrict__ rows) {
    extern __shared__ float smem[];
    float* t = smem;                // [N] this row's target quantiles
    float* tau = smem + N;          // [N]
    float* m = smem + 2 * N;        // [A] quantile means (CQL only)
    __shared__ float red[kQrWarps];
    __shared__ float soft[2];       // max_a m_a, sum_a exp(m_a - max)
    const int tid = threadIdx.x, lane = tsb::lane_id(), warp = tsb::warp_id();
    const int64_t AN = (int64_t)A * N;
    const bool cql = cql_scale != 0.0f;
    for (int k = tid; k < N; k += kQrThreads) tau[k] = tau_hat[k];
    for (int64_t b = blockIdx.x; b < B; b += gridDim.x) {
        const float* qb = q + b * AN;
        float* db = dq + b * AN;
        const int ab = (int)act[b];
        const float wb = weight ? weight[b] : 1.0f;
        __syncthreads();                    // the previous row is done with t, m and soft
        for (int k = tid; k < N; k += kQrThreads) t[k] = returns[b * N + k];
        float cql_row = 0.0f, p_act = 0.0f;
        if (cql) {
            for (int a = warp; a < A; a += kQrWarps) {
                const float ma = quantile_mean(qb + (int64_t)a * N, N, lane);
                if (lane == 0) m[a] = ma;
            }
            __syncthreads();
            if (warp == 0) {
                float mx = -INFINITY;
                for (int a = lane; a < A; a += 32) mx = fmaxf(mx, m[a]);
                mx = tsb::warp_max(mx);
                float s = 0.0f;
                for (int a = lane; a < A; a += 32) s += expf(m[a] - mx);
                s = tsb::warp_sum(s);
                if (lane == 0) { soft[0] = mx; soft[1] = s; }
            }
            __syncthreads();
            const float mx = soft[0], s = soft[1];
            cql_row = logf(s) + (isinf(mx) ? 0.0f : mx) - m[ab];
            p_act = expf(m[ab] - mx) / s;
            for (int64_t e = tid; e < AN; e += kQrThreads) {           // every block but the taken action's
                const int a = (int)(e / N);
                if (a != ab) db[e] = cql_scale * (expf(m[a] - mx) / s);
            }
        } else {
            __syncthreads();
            for (int64_t e = tid; e < AN; e += kQrThreads)
                if ((int)(e / N) != ab) db[e] = 0.0f;
        }
        const float cql_act = cql ? cql_scale * (p_act - 1.0f) : 0.0f;
        const float g_scale = -qr_scale * wb;
        float acc_qr = 0.0f, acc_p = 0.0f;
        for (int i = tid; i < N; i += kQrThreads) {
            const float c = qb[(int64_t)ab * N + i];
            const float ti = tau[i];
            float sq = 0.0f, sp = 0.0f, sg = 0.0f;
            for (int j = 0; j < N; ++j) {
                const float u = t[j] - c;
                const float au = fabsf(u);
                const float h = au < 1.0f ? 0.5f * au * au : au - 0.5f;
                const float w = fabsf(ti - (u <= 0.0f ? 1.0f : 0.0f));
                sq += h * w;
                sp += h;
                sg += w * fminf(fmaxf(u, -1.0f), 1.0f);
            }
            acc_qr += sq;
            acc_p += sp;
            db[(int64_t)ab * N + i] = g_scale * sg + cql_act;
        }
        const float inv_n = 1.0f / (float)N;
        const float qr = block_sum(acc_qr, red) * inv_n;
        const float pr = block_sum(acc_p, red) * inv_n;
        if (tid == 0) {
            rows[b] = wb * qr;
            rows[B + b] = cql_row;
            rows[2 * B + b] = pr;
            prio[b] = pr;
        }
    }
}

}  // namespace

extern "C" int ts_qrdqn_target(const float* q_online, const float* q_next, int64_t B, int32_t A, int32_t N, float* out,
                               int64_t* act_out, ts_stream_t stream) {
    TS_REQUIRE(q_online && q_next && out && B >= 0 && A >= 1 && N >= 1, "ts_qrdqn_target: bad argument");
    if (B == 0) return 0;
    qrdqn_target_kernel<<<tsb::row_grid(B), kRowThreads, 0, tsb::as_stream(stream)>>>(q_online, q_next, B, A, N, out, act_out);
    return tsb::check_launch("ts_qrdqn_target");
}

extern "C" int ts_qrdqn_rows(const float* q, const int64_t* act, const float* returns, const float* tau_hat, const float* weight,
                             int64_t B, int32_t A, int32_t N, float min_q_weight, float* dq, float* prio, float* rows, float* losses,
                             ts_stream_t stream) {
    TS_REQUIRE(q && act && returns && tau_hat && dq && prio && rows && losses && B >= 1 && A >= 1 && N >= 2 && min_q_weight >= 0.0f,
               "ts_qrdqn_rows: bad argument");
    const int64_t smem_floats = 2 * (int64_t)N + (min_q_weight > 0.0f ? A : 0);
    TS_REQUIRE(smem_floats <= kQrSmemFloats, "ts_qrdqn_rows: N = %d quantiles and A = %d actions need %lld floats of shared memory, "
               "more than the %d a block holds", N, A, (long long)smem_floats, kQrSmemFloats);
    cudaStream_t st = tsb::as_stream(stream);
    const double bn = (double)B * (double)N;
    const float qr_scale = (float)(1.0 / bn), cql_scale = (float)(min_q_weight / bn);
    const int64_t cap = (int64_t)tsb::num_sms() * 8;
    const unsigned grid = (unsigned)(B < cap ? B : cap);
    qrdqn_rows_kernel<<<grid, kQrThreads, smem_floats * sizeof(float), st>>>(q, act, returns, tau_hat, weight, B, A, N, qr_scale,
                                                                            cql_scale, dq, prio, rows);
    if (tsb::check_launch("ts_qrdqn_rows")) return 1;
    const float inv_b = 1.0f / (float)B;
    tsb::row_sums3_kernel<<<1, tsb::kRowSumThreads, 0, st>>>(rows, B, inv_b, inv_b, inv_b, 1.0f, min_q_weight, 0.0f, losses);
    return tsb::check_launch("ts_qrdqn_rows/sums");
}
