// n-step return: windowed gather-reduce over VectorReplayBuffer index rows, sm_90a.
//
// Reference: numba `_nstep_return` (tianshou/algorithm/algorithm_base.py:1160-1222):
//   gammas = N; acc = 0
//   for n = N-1 .. 0:  now = idx[n][i]
//        if end_flag[now]: gammas = n+1; acc = 0
//        acc = rew[now] + gamma * acc
//   out[i][a] = target_q[i][a] * gamma^gammas + acc
// f64 throughout, gamma powers built by repeated multiplication (:1204-1206).  The kernel keeps
// that exact operation order (explicit __dmul_rn/__dadd_rn: no FMA contraction) so the f64 result
// is bit-identical to the reference; the f32 output variant rounds once at the store.
//
// One thread per sampled index i: the N index loads are coalesced across i (row-major [N][I]),
// rew / end_flag are random 8 B / 1 B gathers into a buffer of millions of slots -> latency bound;
// all N gathers of a thread are independent of the recurrence and are issued before it is folded.
#include "common.cuh"

namespace {

constexpr int kMaxUnroll = 8;

template <typename TO>
__global__ void nstep_kernel(const double* __restrict__ rew, const uint8_t* __restrict__ end_flag,
                             const float* __restrict__ target_q, const int64_t* __restrict__ idx,
                             int64_t I, int64_t A, int n_step, double gamma, TO* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= I) return;
    double acc = 0.0;
    int gammas = n_step;
    int n = n_step - 1;
    // chunks of up to kMaxUnroll steps: gather first, then fold
    while (n >= 0) {
        double r[kMaxUnroll];
        uint8_t e[kMaxUnroll];
        const int cnt = (n + 1 < kMaxUnroll) ? n + 1 : kMaxUnroll;
#pragma unroll
        for (int k = 0; k < kMaxUnroll; ++k) {
            if (k < cnt) {
                const int64_t now = idx[(int64_t)(n - k) * I + i];
                r[k] = __ldg(rew + now);
                e[k] = __ldg(end_flag + now);
            }
        }
#pragma unroll
        for (int k = 0; k < kMaxUnroll; ++k) {
            if (k < cnt) {
                if (e[k]) { gammas = n - k + 1; acc = 0.0; }
                acc = __dadd_rn(r[k], __dmul_rn(gamma, acc));
            }
        }
        n -= cnt;
    }
    double gpow = 1.0;
    for (int k = 0; k < gammas; ++k) gpow = __dmul_rn(gpow, gamma);
    for (int64_t a = 0; a < A; ++a) {
        const double q = (double)target_q[i * A + a];
        out[i * A + a] = (TO)__dadd_rn(__dmul_rn(q, gpow), acc);
    }
}

}  // namespace

extern "C" int ts_nstep_return(const double* rew, const uint8_t* end_flag, const float* target_q,
                               const int64_t* stacked_idx, int64_t I, int64_t A, int32_t n_step,
                               double gamma, void* out, int out_dtype, ts_stream_t stream) {
    TS_REQUIRE(n_step >= 1, "ts_nstep_return: n_step must be >= 1");
    TS_REQUIRE(out_dtype == TS_F32 || out_dtype == TS_F64, "ts_nstep_return: bad out_dtype");
    if (I == 0 || A == 0) return 0;
    TS_REQUIRE(rew && end_flag && target_q && stacked_idx && out, "ts_nstep_return: null pointer");
    const unsigned grid = (unsigned)((I + 127) / 128);
    cudaStream_t st = tsb::as_stream(stream);
    if (out_dtype == TS_F32)
        nstep_kernel<float><<<grid, 128, 0, st>>>(rew, end_flag, target_q, stacked_idx, I, A, n_step, gamma, static_cast<float*>(out));
    else
        nstep_kernel<double><<<grid, 128, 0, st>>>(rew, end_flag, target_q, stacked_idx, I, A, n_step, gamma, static_cast<double*>(out));
    return tsb::check_launch("ts_nstep_return");
}
