// What the quantile-regression kernels share (qrdqn.cu, iqn.cu, discrete_bcq.cu): torch.argmax's order, the warp mean of one
// action's quantiles, the fixed-order CTA sum and the quantile-Huber pair term of the reference's loss expression.
//
// Reference: tianshou/algorithm/modelfree/qrdqn.py:114-121 and iqn.py:164-176 (smooth_l1(t_j - c_i) times
// |tau_i - 1[t_j - c_i <= 0]|, the indicator detached).
#pragma once
#include <math.h>

#include "common.cuh"

namespace tsb {

// torch.argmax's order on (value, index): a NaN is the maximum, ties go to the lowest index
__device__ __forceinline__ bool argmax_before(float v, int i, float bv, int bi) {
    if (bi < 0) return true;
    const bool vn = isnan(v), bn = isnan(bv);
    if (vn || bn) return vn && (!bn || i < bi);
    return v > bv || (v == bv && i < bi);
}

// mean of x[k * stride] over k in [0, N) on one warp: every lane adds its stride of k in order, then the butterfly; every lane
// returns the same value, and two equal rows give equal means
__device__ __forceinline__ float quantile_mean(const float* __restrict__ x, int N, int64_t stride, int lane) {
    float s = 0.0f;
    for (int k = lane; k < N; k += 32) s += x[(int64_t)k * stride];
    return warp_sum(s) / (float)N;
}

// fixed-order sum over a CTA of kWarps warps: the warp butterfly, then every thread adds the per-warp values in order and
// returns the same value.  red holds kWarps floats.
template <int kWarps>
__device__ __forceinline__ float block_sum(float v, float* __restrict__ red) {
    v = warp_sum(v);
    __syncthreads();                         // red may still be read by the previous call
    if (lane_id() == 0) red[warp_id()] = v;
    __syncthreads();
    float s = 0.0f;
#pragma unroll
    for (int w = 0; w < kWarps; ++w) s += red[w];
    return s;
}

// One (current quantile c at fraction tau, target quantile t) pair of the quantile-Huber loss, u = t - c:
//   sq += smooth_l1(u) * |tau - 1[u <= 0]|      (the loss term)
//   sp += smooth_l1(u)                          (the priority term)
//   sg += |tau - 1[u <= 0]| * clip(u, -1, 1)    (minus d term / d c: the indicator carries no gradient)
// smooth_l1 with beta 1: 0.5 u^2 below |u| = 1, |u| - 0.5 from there on.
__device__ __forceinline__ void quantile_huber_pair(float t, float c, float tau, float& sq, float& sp, float& sg) {
    const float u = t - c;
    const float au = fabsf(u);
    const float h = au < 1.0f ? 0.5f * au * au : au - 0.5f;
    const float w = fabsf(tau - (u <= 0.0f ? 1.0f : 0.0f));
    sq += h * w;
    sp += h;
    sg += w * fminf(fmaxf(u, -1.0f), 1.0f);
}

}  // namespace tsb
