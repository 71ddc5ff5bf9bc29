// torch's optimiser step for one element, the one statement shared by every device update: the per-step SIMT step
// (mlp.cu), the fused epoch kernel (mlp_tc.cu) and the layer-wise / off-policy steps (net_ops.cu).
// Reference: torch/nn/utils/clip_grad.py clip_grad_norm_, torch/optim/adam.py and rmsprop.py (_single_tensor_*).
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

namespace optim {

// clip_grad_norm_'s coefficient: min(max_norm / (total_norm + 1e-6), 1); callers pass it only when clipping is on
__device__ __forceinline__ float clip_coef(float max_norm, float total_norm) {
    return fminf(max_norm / (total_norm + 1e-6f), 1.0f);
}

// Adam's step size lr / (1 - beta1^step) and sqrt(1 - beta2^step), formed in double and rounded once.  The host and the
// device pow may differ in the last bit, so each caller keeps computing it where it always has.
struct AdamBias { float step_size, bc2_sqrt; };
__host__ __device__ inline AdamBias adam_bias(double lr, double beta1, double beta2, int64_t step) {
    return AdamBias{(float)(lr / (1.0 - pow(beta1, (double)step))), (float)sqrt(1.0 - pow(beta2, (double)step))};
}

// Second moment v * decay + (w * g) * g (exp_avg_sq.mul_(beta2).addcmul_(grad, grad, 1 - beta2) and RMSprop's square_avg
// update).  Of the two products one is fused into the add; which one sets the last bit of every later step, so it is
// stated here rather than left to the compiler: FUSE_DECAY rounds (w g) g and fuses v * decay, otherwise v * decay is
// rounded and (w g) * g fused.  The fused epoch kernel and RMSprop fuse the decay, the other Adam steps the square.
template <bool FUSE_DECAY>
__device__ __forceinline__ float second_moment(float v, float decay, float w, float g) {
    return FUSE_DECAY ? __fmaf_rn(v, decay, __fmul_rn(__fmul_rn(w, g), g)) : __fmaf_rn(__fmul_rn(w, g), g, __fmul_rn(v, decay));
}

// torch.optim.Adam single-tensor step of one element on the clipped gradient g.  w1 = 1 - beta1 and w2 = 1 - beta2 are
// formed in double and rounded once, as torch passes them (lerp weight, addcmul value): 1.0f - (float)0.999 would be
// 1.3e-5 off in relative terms.
template <bool FUSE_DECAY = false>
__device__ __forceinline__ void adam_elem(float g, float& p, float& m, float& v, float step_size, float bc2_sqrt, float beta2,
                                          float w1, float w2, float eps, float wd) {
    if (wd != 0.0f) g = fmaf(wd, p, g);         // grad.add(param, alpha=weight_decay)
    m = m + w1 * (g - m);                       // exp_avg.lerp_(grad, 1 - beta1)
    v = second_moment<FUSE_DECAY>(v, beta2, w2, g);
    const float denom = sqrtf(v) / bc2_sqrt + eps;
    p = p - step_size * (m / denom);            // param.addcdiv_(exp_avg, denom, -step_size)
}

// torch.optim.RMSprop single-tensor step of one element without momentum / centering; w_sq = 1 - alpha formed in double
// and rounded once, as torch passes addcmul's value
__device__ __forceinline__ void rmsprop_elem(float g, float& p, float& v, float lr, float alpha, float w_sq, float eps, float wd) {
    if (wd != 0.0f) g = fmaf(wd, p, g);
    v = second_moment<true>(v, alpha, w_sq, g); // square_avg.mul_(alpha).addcmul_(grad, grad, 1 - alpha)
    p = p - lr * (g / (sqrtf(v) + eps));        // param.addcdiv_(grad, square_avg.sqrt().add_(eps), -lr)
}

}  // namespace optim
