// BDQN arithmetic (algorithm/modelfree/bdqn.py): the dueling combine Q = V + (S - mean_a S) of a branching network and the
// per-row pieces of its 1-step target and loss, between the GEMMs of the trunk, the value head and the branch ensemble
// (ts_net_gemm / ts_net_gemm_batched, net_gemm.cu).  The value head's output is V [B][1]; the branch ensemble's is S [nb][B][A]
// (member k's rows back to back), so Q[b][k][a] = V[b] + (S[k][b][a] - mean_a S[k][b][:]).
//
// Reference: tianshou/utils/net/common.py:661-674 (the dueling combine), tianshou/algorithm/modelfree/bdqn.py:126-224 (the target
// r + gamma * mean_k Q'_k(s', a*_k) * (1 - end) formed in numpy, the loss over the chosen action of every branch, the prioritised
// buffer's signed sum over branches).  Every sum runs in a fixed order, so updates repeat bit for bit.
#include <math.h>

#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kRedThreads = 1024;

inline unsigned grid_for(int64_t items) {
    int64_t b = (items + kThreads - 1) / kThreads;
    const int64_t cap = (int64_t)tsb::num_sms() * 4;
    return (unsigned)(b > cap ? cap : (b < 1 ? 1 : b));
}

// mean_a s[a] of one branch row: in index order, then / A
__device__ __forceinline__ float row_mean(const float* __restrict__ s, int A) {
    float acc = s[0];
    for (int a = 1; a < A; ++a) acc = __fadd_rn(acc, s[a]);
    return __fdiv_rn(acc, (float)A);
}

// Q'_k(s', a*_k) of row b, branch k: a*_k = the first arg-max of the selecting network's Q (NaN counts as the maximum, as in
// torch's argmax), read from the evaluating network's Q.
__device__ __forceinline__ float branch_target(const float* __restrict__ v_sel, const float* __restrict__ s_sel,
                                               const float* __restrict__ v_val, const float* __restrict__ s_val, int64_t B,
                                               int A, int64_t b, int k) {
    const int64_t row = ((int64_t)k * B + b) * A;
    const float* ss = s_sel + row;
    const float vs = v_sel[b], ms = row_mean(ss, A);
    float best = __fadd_rn(vs, __fsub_rn(ss[0], ms));
    int arg = 0;
    for (int a = 1; a < A; ++a) {
        const float q = __fadd_rn(vs, __fsub_rn(ss[a], ms));
        if (best == best && (q > best || q != q)) { best = q; arg = a; }
    }
    const float* sv = s_val + row;
    return __fadd_rn(v_val[b], __fsub_rn(sv[arg], row_mean(sv, A)));
}

// y[b] = fp32(rew[i] + fp32(gamma * m) * (1 - end[i])) with i = idx[b] and m the fp32 mean over the branches, summed in numpy's
// order for a float32 row (np.mean in bdqn.py:157): fewer than 8 values in sequence; otherwise eight running sums over the
// values in blocks of 8, combined pairwise, then the tail in sequence (numpy's pairwise_sum for up to 128 values; beyond 128
// branches the same blocks run over the whole row).  y_branch (nullable) [B][nb]: the per-branch targets fp32(rew[i] +
// fp32(gamma * Q'_k) * (1 - end[i])) that the reference's B = 1 loss broadcasts.  Grid-stride over rows.
__global__ void __launch_bounds__(kThreads) bdqn_target_kernel(const float* __restrict__ v_sel, const float* __restrict__ s_sel,
                                                              const float* __restrict__ v_val, const float* __restrict__ s_val,
                                                              int64_t B, int nb, int A, float gamma, const double* __restrict__ rew,
                                                              const uint8_t* __restrict__ end, const int64_t* __restrict__ idx,
                                                              float* __restrict__ y, float* __restrict__ y_branch) {
    for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b < B; b += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i = idx[b];
        const double r = rew[i], live = end[i] ? 0.0 : 1.0;
        float s;
        if (nb < 8) {
            s = branch_target(v_sel, s_sel, v_val, s_val, B, A, b, 0);
            for (int k = 1; k < nb; ++k) s = __fadd_rn(s, branch_target(v_sel, s_sel, v_val, s_val, B, A, b, k));
        } else {
            float p[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) p[j] = branch_target(v_sel, s_sel, v_val, s_val, B, A, b, j);
            const int full = nb - nb % 8;
            for (int k0 = 8; k0 < full; k0 += 8) {
#pragma unroll
                for (int j = 0; j < 8; ++j) p[j] = __fadd_rn(p[j], branch_target(v_sel, s_sel, v_val, s_val, B, A, b, k0 + j));
            }
            s = __fadd_rn(__fadd_rn(__fadd_rn(p[0], p[1]), __fadd_rn(p[2], p[3])), __fadd_rn(__fadd_rn(p[4], p[5]), __fadd_rn(p[6], p[7])));
            for (int k = full; k < nb; ++k) s = __fadd_rn(s, branch_target(v_sel, s_sel, v_val, s_val, B, A, b, k));
        }
        const float m = __fdiv_rn(s, (float)nb);
        y[b] = __double2float_rn(__dadd_rn(r, __dmul_rn((double)__fmul_rn(gamma, m), live)));
        if (y_branch) {
            for (int k = 0; k < nb; ++k) {
                const float q = branch_target(v_sel, s_sel, v_val, s_val, B, A, b, k);
                y_branch[b * nb + k] = __double2float_rn(__dadd_rn(r, __dmul_rn((double)__fmul_rn(gamma, q), live)));
            }
        }
    }
}

// Per row b: td[b][k] = y[b] - Q[b][k][act[b][k]], rows[b] = w mean_k td^2 (scratch), td_sum[b] = sum_k td (signed: the
// prioritised buffer's batch.weight), dV[b] = sum_k g[b][k] with g = dL/dQ at the chosen action = -2 w td / (nb B), branches in
// index order.  Grid-stride over rows.
__global__ void __launch_bounds__(kThreads) bdqn_rows_kernel(const float* __restrict__ v, const float* __restrict__ s,
                                                            const int64_t* __restrict__ act, const float* __restrict__ y,
                                                            const float* __restrict__ weight, int64_t B, int nb, int A,
                                                            float* __restrict__ td, float* __restrict__ rows,
                                                            float* __restrict__ td_sum, float* __restrict__ dv) {
    const float inv_n = __fdiv_rn(1.0f, (float)((int64_t)nb * B));
    for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b < B; b += (int64_t)gridDim.x * blockDim.x) {
        const float w = weight ? weight[b] : 1.0f, vb = v[b], yb = y[b];
        float sq = 0.0f, sum = 0.0f, gsum = 0.0f;
        for (int k = 0; k < nb; ++k) {
            const float* sr = s + ((int64_t)k * B + b) * A;
            const float q = __fadd_rn(vb, __fsub_rn(sr[act[b * nb + k]], row_mean(sr, A)));
            const float d = __fsub_rn(yb, q);
            td[b * nb + k] = d;
            sq = __fadd_rn(sq, __fmul_rn(d, d));
            sum = __fadd_rn(sum, d);
            gsum = __fadd_rn(gsum, __fmul_rn(__fmul_rn(-2.0f, d), __fmul_rn(inv_n, w)));
        }
        rows[b] = __fmul_rn(__fdiv_rn(sq, (float)nb), w);
        td_sum[b] = sum;
        dv[b] = gsum;
    }
}

// dS[k][b][a] = g[b][k][a] - mean_a g[b][k][:]: g is -2 w td / (nb B) at the chosen action and 0 elsewhere.  blockIdx.y = branch
// k, grid-stride over rows.
__global__ void __launch_bounds__(kThreads) bdqn_dscore_kernel(const float* __restrict__ td, const int64_t* __restrict__ act,
                                                              const float* __restrict__ weight, int64_t B, int nb, int A,
                                                              float* __restrict__ ds) {
    const float inv_n = __fdiv_rn(1.0f, (float)((int64_t)nb * B));
    const int k = (int)blockIdx.y;
    for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b < B; b += (int64_t)gridDim.x * blockDim.x) {
        const float w = weight ? weight[b] : 1.0f;
        const float g = __fmul_rn(__fmul_rn(-2.0f, td[b * nb + k]), __fmul_rn(inv_n, w));
        const float ga = __fdiv_rn(g, (float)A);
        const int64_t chosen = act[b * nb + k];
        float* out = ds + ((int64_t)k * B + b) * A;
        for (int a = 0; a < A; ++a) out[a] = a == chosen ? __fsub_rn(g, ga) : -ga;
    }
}

// *loss = sum(rows[0 .. B)) / B: one block, strided partial sums then a pairwise tree (fixed order).  With y_branch (B = 1):
// plus the population variance of the nb per-branch targets, the term the reference's broadcast [nb, nb, A] returns add.
__global__ void __launch_bounds__(kRedThreads) bdqn_sum_kernel(const float* __restrict__ rows, int64_t B,
                                                              const float* __restrict__ y_branch, int nb, float* __restrict__ loss) {
    __shared__ float sh[kRedThreads];
    float acc = 0.0f;
    for (int64_t i = threadIdx.x; i < B; i += kRedThreads) acc = __fadd_rn(acc, rows[i]);
    sh[threadIdx.x] = acc;
    __syncthreads();
    for (int off = kRedThreads / 2; off > 0; off >>= 1) {
        if ((int)threadIdx.x < off) sh[threadIdx.x] = __fadd_rn(sh[threadIdx.x], sh[threadIdx.x + off]);
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        float l = __fdiv_rn(sh[0], (float)B);
        if (y_branch) {
            float m = 0.0f;
            for (int k = 0; k < nb; ++k) m = __fadd_rn(m, y_branch[k]);
            m = __fdiv_rn(m, (float)nb);
            float var = 0.0f;
            for (int k = 0; k < nb; ++k) {
                const float d = __fsub_rn(y_branch[k], m);
                var = __fadd_rn(var, __fmul_rn(d, d));
            }
            l = __fadd_rn(l, __fdiv_rn(var, (float)nb));
        }
        *loss = l;
    }
}

}  // namespace

extern "C" int ts_bdqn_target(const float* v_sel, const float* s_sel, const float* v_val, const float* s_val, int64_t B, int32_t nb,
                              int32_t A, float gamma, const double* rew, const uint8_t* end, const int64_t* idx, float* y,
                              float* y_branch, ts_stream_t stream) {
    TS_REQUIRE(v_sel && s_sel && v_val && s_val && rew && end && idx && y && B >= 0 && nb >= 1 && A >= 1,
               "ts_bdqn_target: bad argument");
    if (B == 0) return 0;
    bdqn_target_kernel<<<grid_for(B), kThreads, 0, tsb::as_stream(stream)>>>(v_sel, s_sel, v_val, s_val, B, nb, A, gamma, rew, end,
                                                                            idx, y, y_branch);
    return tsb::check_launch("ts_bdqn_target");
}

extern "C" int ts_bdqn_rows(const float* v, const float* s, const int64_t* act, const float* y, const float* weight,
                            const float* y_branch, int64_t B, int32_t nb, int32_t A, float* td, float* rows, float* td_sum,
                            float* ds, float* dv, float* loss, ts_stream_t stream) {
    TS_REQUIRE(v && s && act && y && td && rows && td_sum && ds && dv && loss && B >= 1 && nb >= 1 && A >= 1,
               "ts_bdqn_rows: bad argument");
    TS_REQUIRE(!y_branch || B == 1, "ts_bdqn_rows: the per-branch targets enter the loss at B = 1 only, got B = %lld", (long long)B);
    const cudaStream_t st = tsb::as_stream(stream);
    bdqn_rows_kernel<<<grid_for(B), kThreads, 0, st>>>(v, s, act, y, weight, B, nb, A, td, rows, td_sum, dv);
    if (tsb::check_launch("ts_bdqn_rows")) return 1;
    TS_REQUIRE(nb <= 65535, "ts_bdqn_rows: %d branches exceed the grid", nb);
    bdqn_dscore_kernel<<<dim3(grid_for(B), (unsigned)nb), kThreads, 0, st>>>(td, act, weight, B, nb, A, ds);
    if (tsb::check_launch("ts_bdqn_rows/dscore")) return 1;
    bdqn_sum_kernel<<<1, kRedThreads, 0, st>>>(rows, B, y_branch, nb, loss);
    return tsb::check_launch("ts_bdqn_rows/sum");
}
