// IQN arithmetic (algorithm/modelfree/iqn.py, utils/net/discrete.py ImplicitQuantileNetwork): the per-row pieces between the
// network's GEMMs that no layered-network launch provides -- the cosine features of the sampled fractions, the product of the
// trunk's features with their embedding and its backward, the target at the arg-max of the sample means and the quantile-Huber
// rows with a fraction per row and sample.  The GEMMs themselves are the launches of net_gemm.cu.  The head runs on B * S rows
// in sample-major order, so its output is q[B][S][A].
//
// Reference: tianshou/utils/net/discrete.py:126-160 (CosineEmbeddingNetwork), :163-216 (ImplicitQuantileNetwork.forward: the
// fractions, the product, the head), algorithm/modelfree/qrdqn.py:94-106 (the target at the online arg-max of the quantile
// means), algorithm/modelfree/iqn.py:156-183 (the quantile-Huber loss with per-sample fractions, the priority).
#include <math.h>

#include "common.cuh"
#include "quantile.cuh"
#include "row_sums.cuh"

namespace {

using tsb::argmax_before;
using tsb::kRowsPerBlock;
using tsb::kRowThreads;

constexpr int kIqnThreads = 256;
constexpr int kIqnWarps = kIqnThreads / 32;
constexpr int kIqnSmemFloats = 48 * 1024 / 4;     // the default dynamic shared-memory limit: the row's S_t target quantiles
constexpr int kEwThreads = 256;

// as many blocks of kEwThreads as n elements need, at most 8 per SM: the element-wise kernels stride over the rest
unsigned ew_grid(int64_t n) {
    const int64_t b = (n + kEwThreads - 1) / kEwThreads, cap = (int64_t)tsb::num_sms() * 8;
    return (unsigned)(b > cap ? cap : (b < 1 ? 1 : b));
}

// out[r][c] = cos(tau[r] * (pi_f * (c + 1))) with pi_f = fl32(pi): both products rounded on their own (no contraction, as the
// reference's two fp32 tensor multiplications), cosf at full accuracy.  One warp per row, lanes over c.
__global__ void __launch_bounds__(kRowThreads) iqn_cos_kernel(const float* __restrict__ taus, int64_t R, int C, float* __restrict__ out) {
    for (int64_t r = (int64_t)blockIdx.x * kRowsPerBlock + tsb::warp_id(); r < R; r += (int64_t)gridDim.x * kRowsPerBlock) {
        const float t = taus[r];
        for (int c = tsb::lane_id(); c < C; c += 32) {
            const float i_pi = __fmul_rn(3.14159265358979323846f, (float)(c + 1));
            out[r * C + c] = cosf(__fmul_rn(t, i_pi));
        }
    }
}

// h[b * S + s][d] = feat[b][d] * e[b * S + s][d]
__global__ void __launch_bounds__(kEwThreads) iqn_mix_kernel(const float* __restrict__ feat, const float* __restrict__ e, int64_t B,
                                                             int S, int D, float* __restrict__ h) {
    const int64_t n = B * S * (int64_t)D, SD = (int64_t)S * D;
    for (int64_t k = (int64_t)blockIdx.x * kEwThreads + threadIdx.x; k < n; k += (int64_t)gridDim.x * kEwThreads) {
        const int64_t b = k / SD, d = k % D;
        h[k] = feat[b * D + d] * e[k];
    }
}

// One thread per (b, d): over s = 0 .. S - 1 in order, dfeat accumulates dh * e and de_pre = dh * feat * 1[e > 0] (the
// embedding's ReLU, whose output e is); dfeat then takes the derivative of the trunk's last activation at its output y, the
// rule of ts_net_gemm's mask (ReLU: * 1[y > 0], tanh: * (1 - y^2)).
__global__ void __launch_bounds__(kEwThreads) iqn_mix_backward_kernel(const float* __restrict__ dh, const float* __restrict__ feat,
                                                                      const float* __restrict__ e, int64_t B, int S, int D, int trunk_act,
                                                                      const float* __restrict__ trunk_out, float* __restrict__ dfeat,
                                                                      float* __restrict__ de_pre) {
    const int64_t n = B * (int64_t)D;
    for (int64_t k = (int64_t)blockIdx.x * kEwThreads + threadIdx.x; k < n; k += (int64_t)gridDim.x * kEwThreads) {
        const int64_t b = k / D, d = k - b * D;
        const float f = feat[k];
        float acc = 0.0f;
        for (int s = 0; s < S; ++s) {
            const int64_t r = (b * S + s) * D + d;
            const float g = dh[r], es = e[r];
            acc += g * es;
            de_pre[r] = es > 0.0f ? g * f : 0.0f;
        }
        if (trunk_act == TS_ACT_RELU) {
            acc = trunk_out[k] > 0.0f ? acc : 0.0f;
        } else if (trunk_act == TS_ACT_TANH) {
            const float y = trunk_out[k];
            acc = acc * fmaf(-y, y, 1.0f);
        }
        dfeat[k] = acc;
    }
}

// Per row b: m_a = mean_s q_online[b][s][a] over the S_on online samples, a* = the first arg-max of m (NaN the maximum),
// out[b][s] = q_next[b][s][a*] for the S_next samples of q_next.  One warp per row.
__global__ void __launch_bounds__(kRowThreads) iqn_target_kernel(const float* __restrict__ q_online, const float* __restrict__ q_next,
                                                                 int64_t B, int A, int S_on, int S_next, float* __restrict__ out,
                                                                 int64_t* __restrict__ act_out) {
    const int lane = tsb::lane_id();
    for (int64_t b = (int64_t)blockIdx.x * kRowsPerBlock + tsb::warp_id(); b < B; b += (int64_t)gridDim.x * kRowsPerBlock) {
        const float* qb = q_online + b * S_on * (int64_t)A;
        float bv = 0.0f;
        int bi = -1;
        for (int a = 0; a < A; ++a) {
            const float m = tsb::quantile_mean(qb + a, S_on, A, lane);
            if (argmax_before(m, a, bv, bi)) { bv = m; bi = a; }
        }
        const float* src = q_next + b * S_next * (int64_t)A + bi;
        for (int s = lane; s < S_next; s += 32) out[b * S_next + s] = src[(int64_t)s * A];
        if (lane == 0 && act_out) act_out[b] = bi;
    }
}

// One CTA per row b (grid-stride), threads over the current quantiles i.  With c_i = q[b][i][act], tau_i = taus[b][i],
// t_j = returns[b][j] (in shared memory), u_ij = t_j - c_i:
//   rows[0][b] = weight_b * (1/S_on) sum_i sum_j h_ij w_ij       rows[2][b] = prio[b] = (1/S_on) sum_i sum_j h_ij
//   rows[1][b] = 0                                               dq[b][i][a] = 1[a == act] * (-scale weight_b sum_j w_ij clip(u_ij))
// with h, w the pair terms of quantile_huber_pair and scale = 1 / (B S_on).
__global__ void __launch_bounds__(kIqnThreads) iqn_rows_kernel(
        const float* __restrict__ q, const int64_t* __restrict__ act, const float* __restrict__ returns, const float* __restrict__ taus,
        const float* __restrict__ weight, int64_t B, int A, int S_on, int S_t, float scale, float* __restrict__ dq,
        float* __restrict__ prio, float* __restrict__ rows) {
    extern __shared__ float t[];            // [S_t] this row's target quantiles
    __shared__ float red[kIqnWarps];
    const int tid = threadIdx.x;
    const int64_t SA = (int64_t)S_on * A;
    for (int64_t b = blockIdx.x; b < B; b += gridDim.x) {
        const float* qb = q + b * SA;
        float* db = dq + b * SA;
        const int ab = (int)act[b];
        const float wb = weight ? weight[b] : 1.0f;
        __syncthreads();                    // the previous row is done with t
        for (int j = tid; j < S_t; j += kIqnThreads) t[j] = returns[b * S_t + j];
        for (int64_t e = tid; e < SA; e += kIqnThreads)
            if ((int)(e % A) != ab) db[e] = 0.0f;
        __syncthreads();
        const float g_scale = -scale * wb;
        float acc_qr = 0.0f, acc_p = 0.0f;
        for (int i = tid; i < S_on; i += kIqnThreads) {
            const float c = qb[(int64_t)i * A + ab];
            const float ti = taus[b * S_on + i];
            float sq = 0.0f, sp = 0.0f, sg = 0.0f;
            for (int j = 0; j < S_t; ++j) tsb::quantile_huber_pair(t[j], c, ti, sq, sp, sg);
            acc_qr += sq;
            acc_p += sp;
            db[(int64_t)i * A + ab] = g_scale * sg;
        }
        const float inv_s = 1.0f / (float)S_on;
        const float qr = tsb::block_sum<kIqnWarps>(acc_qr, red) * inv_s;
        const float pr = tsb::block_sum<kIqnWarps>(acc_p, red) * inv_s;
        if (tid == 0) {
            rows[b] = wb * qr;
            rows[B + b] = 0.0f;
            rows[2 * B + b] = pr;
            prio[b] = pr;
        }
    }
}

}  // namespace

extern "C" int ts_iqn_cos(const float* taus, int64_t R, int32_t C, float* out, ts_stream_t stream) {
    TS_REQUIRE(taus && out && R >= 0 && C >= 1, "ts_iqn_cos: bad argument");
    if (R == 0) return 0;
    iqn_cos_kernel<<<tsb::row_grid(R), kRowThreads, 0, tsb::as_stream(stream)>>>(taus, R, C, out);
    return tsb::check_launch("ts_iqn_cos");
}

extern "C" int ts_iqn_mix(const float* feat, const float* e, int64_t B, int32_t S, int32_t D, float* h, ts_stream_t stream) {
    TS_REQUIRE(feat && e && h && B >= 0 && S >= 1 && D >= 1, "ts_iqn_mix: bad argument");
    if (B == 0) return 0;
    iqn_mix_kernel<<<ew_grid(B * S * (int64_t)D), kEwThreads, 0, tsb::as_stream(stream)>>>(feat, e, B, S, D, h);
    return tsb::check_launch("ts_iqn_mix");
}

extern "C" int ts_iqn_mix_backward(const float* dh, const float* feat, const float* e, int64_t B, int32_t S, int32_t D,
                                   int32_t trunk_act, const float* trunk_out, float* dfeat, float* de_pre, ts_stream_t stream) {
    TS_REQUIRE(dh && feat && e && dfeat && de_pre && B >= 0 && S >= 1 && D >= 1, "ts_iqn_mix_backward: bad argument");
    TS_REQUIRE(trunk_act == TS_ACT_NONE || ((trunk_act == TS_ACT_RELU || trunk_act == TS_ACT_TANH) && trunk_out),
               "ts_iqn_mix_backward: trunk activation %d needs its output", trunk_act);
    if (B == 0) return 0;
    iqn_mix_backward_kernel<<<ew_grid(B * (int64_t)D), kEwThreads, 0, tsb::as_stream(stream)>>>(dh, feat, e, B, S, D, trunk_act,
                                                                                              trunk_out, dfeat, de_pre);
    return tsb::check_launch("ts_iqn_mix_backward");
}

extern "C" int ts_iqn_target(const float* q_online, const float* q_next, int64_t B, int32_t A, int32_t S_on, int32_t S_next,
                             float* out, int64_t* act_out, ts_stream_t stream) {
    TS_REQUIRE(q_online && q_next && out && B >= 0 && A >= 1 && S_on >= 1 && S_next >= 1, "ts_iqn_target: bad argument");
    if (B == 0) return 0;
    iqn_target_kernel<<<tsb::row_grid(B), kRowThreads, 0, tsb::as_stream(stream)>>>(q_online, q_next, B, A, S_on, S_next, out,
                                                                                     act_out);
    return tsb::check_launch("ts_iqn_target");
}

extern "C" int ts_iqn_rows(const float* q, const int64_t* act, const float* returns, const float* taus, const float* weight,
                           int64_t B, int32_t A, int32_t S_on, int32_t S_t, float* dq, float* prio, float* rows, float* losses,
                           ts_stream_t stream) {
    TS_REQUIRE(q && act && returns && taus && dq && prio && rows && losses && B >= 1 && A >= 1 && S_on >= 1 && S_t >= 1,
               "ts_iqn_rows: bad argument");
    TS_REQUIRE(S_t <= kIqnSmemFloats, "ts_iqn_rows: S_t = %d target quantiles need %d floats of shared memory, more than the %d a "
               "block holds", S_t, S_t, kIqnSmemFloats);
    cudaStream_t st = tsb::as_stream(stream);
    const float scale = (float)(1.0 / ((double)B * (double)S_on));
    const int64_t cap = (int64_t)tsb::num_sms() * 8;
    const unsigned grid = (unsigned)(B < cap ? B : cap);
    iqn_rows_kernel<<<grid, kIqnThreads, (size_t)S_t * sizeof(float), st>>>(q, act, returns, taus, weight, B, A, S_on, S_t, scale,
                                                                           dq, prio, rows);
    if (tsb::check_launch("ts_iqn_rows")) return 1;
    const float inv_b = 1.0f / (float)B;
    tsb::row_sums3_kernel<<<1, tsb::kRowSumThreads, 0, st>>>(rows, B, inv_b, inv_b, inv_b, 1.0f, 0.0f, 0.0f, losses);
    return tsb::check_launch("ts_iqn_rows/sums");
}
