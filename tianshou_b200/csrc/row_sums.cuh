// The closing reduction of the three-term offline discrete losses (discrete_bcq.cu, discrete_crr.cu): three series of per-row
// partials -> the three loss terms and their weighted total, in one block with a fixed summation order (bit-identical from
// run to run, no atomics).
#pragma once
#include "common.cuh"

namespace tsb {

constexpr int kRowSumThreads = 1024;

// rows [3][B]; out[1 + k] = scale[k] * sum_b rows[k][b]; out[0] = sum_k weight[k] * out[1 + k].
// Each thread sums its stride of rows in order, then a shared-memory tree: a term's error is bounded by
// ~(B / 1024 + 10) eps times the sum of the magnitudes of its rows.
static __global__ void __launch_bounds__(kRowSumThreads) row_sums3_kernel(const float* __restrict__ rows, int64_t B, float s0, float s1,
                                                                         float s2, float w0, float w1, float w2,
                                                                         float* __restrict__ out) {
    __shared__ float s[3][kRowSumThreads];
    float a0 = 0.0f, a1 = 0.0f, a2 = 0.0f;
    for (int64_t i = threadIdx.x; i < B; i += kRowSumThreads) {
        a0 += rows[i];
        a1 += rows[B + i];
        a2 += rows[2 * B + i];
    }
    s[0][threadIdx.x] = a0;
    s[1][threadIdx.x] = a1;
    s[2][threadIdx.x] = a2;
    __syncthreads();
    for (int off = kRowSumThreads / 2; off > 0; off >>= 1) {
        if ((int)threadIdx.x < off) {
            s[0][threadIdx.x] += s[0][threadIdx.x + off];
            s[1][threadIdx.x] += s[1][threadIdx.x + off];
            s[2][threadIdx.x] += s[2][threadIdx.x + off];
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        const float t0 = s[0][0] * s0, t1 = s[1][0] * s1, t2 = s[2][0] * s2;
        out[1] = t0;
        out[2] = t1;
        out[3] = t2;
        out[0] = w0 * t0 + w1 * t1 + w2 * t2;
    }
}

// The same fixed order for one series computed on the fly, inside a one-block kernel of kRowSumThreads threads: thread t sums
// term(i) for i = t, t + 1024, ... < n in order, then a shared-memory tree.  Every thread returns the total.
template <class Term>
__device__ __forceinline__ float block_sum_fixed(int64_t n, Term term) {
    __shared__ float s[kRowSumThreads];
    float a = 0.0f;
    for (int64_t i = threadIdx.x; i < n; i += kRowSumThreads) a += term(i);
    s[threadIdx.x] = a;
    __syncthreads();
    for (int off = kRowSumThreads / 2; off > 0; off >>= 1) {
        if ((int)threadIdx.x < off) s[threadIdx.x] += s[threadIdx.x + off];
        __syncthreads();
    }
    return s[0];
}

// one warp per row, warps stride over the rows: the grid of the per-row kernels
constexpr int kRowThreads = 256;
constexpr int kRowsPerBlock = kRowThreads / 32;
inline unsigned row_grid(int64_t rows) {
    int64_t b = (rows + kRowsPerBlock - 1) / kRowsPerBlock;
    const int64_t cap = (int64_t)num_sms() * 16;
    return (unsigned)(b > cap ? cap : (b < 1 ? 1 : b));
}

}  // namespace tsb
