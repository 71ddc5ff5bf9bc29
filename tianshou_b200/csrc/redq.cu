// REDQ arithmetic (algorithm/modelfree/redq.py): the per-row pieces between the batched GEMMs of the critic ensemble
// (ts_net_gemm_batched, net_gemm.cu).  Member e's q-values are q[e * B + b], the ensemble stack's [E][B][1] output.
//
// Reference: tianshou/algorithm/modelfree/redq.py:254-269 (the target over a random subset of the lagged ensemble, min or mean,
// minus alpha * log pi), :273-279 (the ensemble's weighted squared loss and the prioritised buffer's batch.weight = mean_e td),
// :285-289 (the actor loss mean(alpha * log pi - mean_e Q)).  Every sum runs in a fixed order, so updates repeat bit for bit.
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

// out[b] = {min | mean} over the members in `subset` of q[e][b], minus alpha * logp[b].  Grid-stride over rows.
__global__ void __launch_bounds__(kThreads) redq_target_kernel(const float* __restrict__ q, int E, int64_t B, uint64_t subset,
                                                              int mode, float alpha, const float* __restrict__ logp,
                                                              float* __restrict__ out) {
    const int count = __popcll(subset);
    for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b < B; b += (int64_t)gridDim.x * blockDim.x) {
        float acc = 0.0f;
        bool first = true;
        for (int e = 0; e < E; ++e) {
            if (!((subset >> e) & 1ull)) continue;
            const float v = q[(int64_t)e * B + b];
            if (mode == TS_REDQ_MEAN) acc = first ? v : __fadd_rn(acc, v);
            else acc = first ? v : ((acc != acc || v != v) ? __fadd_rn(acc, v) : fminf(acc, v));
            first = false;
        }
        if (mode == TS_REDQ_MEAN) acc = __fdiv_rn(acc, (float)count);
        out[b] = __fsub_rn(acc, __fmul_rn(alpha, logp[b]));
    }
}

// td / dq / row_mean / rows of the critic loss, one row per item (members in order).  Grid-stride over rows.
__global__ void __launch_bounds__(kThreads) redq_critic_rows_kernel(const float* __restrict__ q, const float* __restrict__ target,
                                                                   const float* __restrict__ weight, int E, int64_t B,
                                                                   float* __restrict__ td, float* __restrict__ dq,
                                                                   float* __restrict__ row_mean, float* __restrict__ rows) {
    const float inv_n = __fdiv_rn(1.0f, (float)((int64_t)E * B));
    for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b < B; b += (int64_t)gridDim.x * blockDim.x) {
        const float w = weight ? weight[b] : 1.0f, t = target[b];
        float s = 0.0f, r = 0.0f;
        for (int e = 0; e < E; ++e) {
            const int64_t i = (int64_t)e * B + b;
            const float d = __fsub_rn(q[i], t);
            td[i] = d;
            dq[i] = __fmul_rn(__fmul_rn(2.0f, d), __fmul_rn(inv_n, w));
            s = __fadd_rn(s, d);
            r = __fadd_rn(r, __fmul_rn(__fmul_rn(d, d), w));
        }
        row_mean[b] = __fdiv_rn(s, (float)E);
        rows[b] = r;
    }
}

// rows [B] of the actor loss: alpha * logp - mean_e q (members in order), and dq = -1 / (E B).  Grid-stride over rows.
__global__ void __launch_bounds__(kThreads) redq_actor_rows_kernel(const float* __restrict__ q, const float* __restrict__ logp,
                                                                  int E, int64_t B, float alpha, float* __restrict__ dq,
                                                                  float* __restrict__ rows) {
    const float g = __fdiv_rn(-1.0f, (float)((int64_t)E * B));
    for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b < B; b += (int64_t)gridDim.x * blockDim.x) {
        float s = 0.0f;
        for (int e = 0; e < E; ++e) {
            s = __fadd_rn(s, q[(int64_t)e * B + b]);
            dq[(int64_t)e * B + b] = g;
        }
        rows[b] = __fsub_rn(__fmul_rn(alpha, logp[b]), __fdiv_rn(s, (float)E));
    }
}

// *out = sum(x[0 .. n)) / denom: one block, strided partial sums then a pairwise tree (fixed order)
__global__ void __launch_bounds__(kRedThreads) redq_sum_kernel(const float* __restrict__ x, int64_t n, float denom,
                                                              float* __restrict__ out) {
    __shared__ float s[kRedThreads];
    float acc = 0.0f;
    for (int64_t i = threadIdx.x; i < n; i += kRedThreads) acc = __fadd_rn(acc, x[i]);
    s[threadIdx.x] = acc;
    __syncthreads();
    for (int off = kRedThreads / 2; off > 0; off >>= 1) {
        if ((int)threadIdx.x < off) s[threadIdx.x] = __fadd_rn(s[threadIdx.x], s[threadIdx.x + off]);
        __syncthreads();
    }
    if (threadIdx.x == 0) *out = __fdiv_rn(s[0], denom);
}

}  // namespace

extern "C" int ts_redq_target(const float* q, int32_t E, int64_t B, uint64_t subset, int32_t target_mode, float alpha,
                              const float* logp, float* out, ts_stream_t stream) {
    TS_REQUIRE(q && logp && out && B >= 0, "ts_redq_target: bad argument");
    TS_REQUIRE(E >= 1 && E <= 64, "ts_redq_target: the subset mask holds 1 .. 64 members, got E = %d", E);
    TS_REQUIRE(subset != 0 && (E == 64 || (subset >> E) == 0), "ts_redq_target: subset mask names no member or one past E = %d", E);
    TS_REQUIRE(target_mode == TS_REDQ_MIN || target_mode == TS_REDQ_MEAN, "ts_redq_target: unknown target_mode %d", target_mode);
    if (B == 0) return 0;
    redq_target_kernel<<<grid_for(B), kThreads, 0, tsb::as_stream(stream)>>>(q, E, B, subset, target_mode, alpha, logp, out);
    return tsb::check_launch("ts_redq_target");
}

extern "C" int ts_redq_critic_rows(const float* q, const float* target, const float* weight, int32_t E, int64_t B, float* td,
                                   float* dq, float* row_mean, float* rows, float* loss, ts_stream_t stream) {
    TS_REQUIRE(q && target && td && dq && row_mean && rows && loss && E >= 1 && B >= 1, "ts_redq_critic_rows: bad argument");
    const cudaStream_t st = tsb::as_stream(stream);
    redq_critic_rows_kernel<<<grid_for(B), kThreads, 0, st>>>(q, target, weight, E, B, td, dq, row_mean, rows);
    if (tsb::check_launch("ts_redq_critic_rows")) return 1;
    redq_sum_kernel<<<1, kRedThreads, 0, st>>>(rows, B, (float)((int64_t)E * B), loss);
    return tsb::check_launch("ts_redq_critic_rows/sum");
}

extern "C" int ts_redq_actor_rows(const float* q, const float* logp, int32_t E, int64_t B, float alpha, float* dq, float* rows,
                                  float* loss, ts_stream_t stream) {
    TS_REQUIRE(q && logp && dq && rows && loss && E >= 1 && B >= 1, "ts_redq_actor_rows: bad argument");
    const cudaStream_t st = tsb::as_stream(stream);
    redq_actor_rows_kernel<<<grid_for(B), kThreads, 0, st>>>(q, logp, E, B, alpha, dq, rows);
    if (tsb::check_launch("ts_redq_actor_rows")) return 1;
    redq_sum_kernel<<<1, kRedThreads, 0, st>>>(rows, B, (float)B, loss);
    return tsb::check_launch("ts_redq_actor_rows/sum");
}
