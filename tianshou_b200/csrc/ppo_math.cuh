// Per-row PPO loss arithmetic shared by the tensor-core kernels (csrc/mlp_tc.cu).
// Reference: tianshou/algorithm/modelfree/ppo.py:183-211 with torch's backward tie rules for
// minimum / maximum / clamp (derivatives.yaml: equal operands split the gradient in halves).
#pragma once
#include <cuda_runtime.h>

#include "../../include/ts_b200.h"

namespace ppo {

struct Scalars {  // hyper-parameters narrowed to f32 where torch would narrow them
    float eps_clip, lo_c, hi_c, vf_coef, ent_coef, adv_eps, dual_clip, inv_b, adv_mean, adv_std;
    int value_clip, adv_norm, a2c;
};

__device__ __forceinline__ Scalars make_scalars(const ts_ppo_hparams& hp, int64_t global_rows,
                                                const float* __restrict__ adv_moments) {
    Scalars s;
    s.eps_clip = (float)hp.eps_clip;
    s.lo_c = (float)(1.0 - hp.eps_clip);
    s.hi_c = (float)(1.0 + hp.eps_clip);
    s.vf_coef = (float)hp.vf_coef;
    s.ent_coef = (float)hp.ent_coef;
    s.adv_eps = (float)hp.adv_eps;
    s.dual_clip = (float)hp.dual_clip;
    s.inv_b = 1.0f / (float)global_rows;
    s.value_clip = hp.value_clip;
    s.a2c = hp.loss_kind == TS_LOSS_A2C;
    s.adv_norm = hp.advantage_normalization && adv_moments != nullptr;
    s.adv_mean = s.adv_norm ? adv_moments[0] : 0.0f;
    s.adv_std = s.adv_norm ? adv_moments[1] : 1.0f;
    return s;
}

// value loss of one row and d(total loss)/d(value)            (ppo.py:198-208)
__device__ __forceinline__ void critic_row(const Scalars& s, float value, float R, float vs, float& vf_row, float& dv) {
    float g;
    if (s.value_clip) {
        const float dlt = value - vs;
        const float dcl = fminf(fmaxf(dlt, -s.eps_clip), s.eps_clip);
        const float v_clip = vs + dcl;
        const float e1 = R - value, e2 = R - v_clip;
        const float vf1 = e1 * e1, vf2 = e2 * e2;
        vf_row = fmaxf(vf1, vf2);
        const float in_range = (dlt >= -s.eps_clip && dlt <= s.eps_clip) ? 1.0f : 0.0f;
        const float g1 = -2.0f * e1, g2 = -2.0f * e2 * in_range;
        g = (vf1 > vf2) ? g1 : ((vf1 < vf2) ? g2 : 0.5f * (g1 + g2));
    } else {
        const float e1 = R - value;
        vf_row = e1 * e1;
        g = -2.0f * e1;
    }
    dv = s.vf_coef * s.inv_b * g;
}

// clipped surrogate of one row: objective value and d(total loss)/d(logp)   (ppo.py:183-196)
__device__ __forceinline__ void actor_row(const Scalars& s, float logp, float logp_old, float adv_raw, float& obj, float& gl) {
    float Adv = adv_raw;
    if (s.a2c) {     // a2c.py:262-266: actor_loss = -(log_prob * adv).mean()
        obj = logp * Adv;
        gl = -s.inv_b * Adv;
        return;
    }
    if (s.adv_norm) Adv = (Adv - s.adv_mean) / (s.adv_std + s.adv_eps);
    const float ratio = expf(logp - logp_old);
    const float rc = fminf(fmaxf(ratio, s.lo_c), s.hi_c);
    const bool in_range = (ratio >= s.lo_c) && (ratio <= s.hi_c);
    const float surr1 = ratio * Adv, surr2 = rc * Adv;
    float g_ratio;
    if (surr1 < surr2) g_ratio = Adv;
    else if (surr1 > surr2) g_ratio = in_range ? Adv : 0.0f;
    else g_ratio = in_range ? Adv : 0.5f * Adv;
    const float clip1 = fminf(surr1, surr2);
    obj = clip1;
    if (s.dual_clip > 0.0f && Adv < 0.0f) {   // ppo.py:191-194
        const float c2 = s.dual_clip * Adv;
        obj = fmaxf(clip1, c2);
        if (clip1 < c2) g_ratio = 0.0f; else if (clip1 == c2) g_ratio *= 0.5f;
    }
    gl = -s.inv_b * g_ratio * ratio;
}

// log N(x; mu, sigma) of one action dim, torch.distributions.Normal.log_prob order
__device__ __forceinline__ float normal_logp_term(float x, float mu, float sigma) {
    const float var = sigma * sigma;
    const float diff = x - mu;
    return -(diff * diff) / (2.0f * var) - logf(sigma) - 0.9189385332046727f;
}

// Categorical(probs = softmax(z)) of one row (utils/net/discrete.py:69-92 + torch.distributions.Categorical), shared by
// the PPO loss rows (ppo_rows.cu) and the NPG / TRPO rows (npg.cu).
constexpr int kCatMaxA = 64;
struct Cat { float p[kCatMaxA], pn[kCatMaxA], lg[kCatMaxA]; float s2; };
// p = softmax(z); Categorical renormalises (pn = p / sum p), logits = log(clamp(pn, eps, 1 - eps)); entropy = -sum pn * logits
__device__ __forceinline__ void cat_forward(const float* z, int A, int action, Cat& c, float& logp, float& ent) {
    constexpr float eps = 1.1920928955078125e-07f;
    float m = z[0];
    for (int a = 1; a < A; ++a) m = fmaxf(m, z[a]);
    float s = 0.0f;
    for (int a = 0; a < A; ++a) { c.p[a] = expf(z[a] - m); s += c.p[a]; }
    float s2 = 0.0f;
    for (int a = 0; a < A; ++a) { c.p[a] = c.p[a] / s; s2 += c.p[a]; }
    c.s2 = s2;
    ent = 0.0f;
    for (int a = 0; a < A; ++a) {
        c.pn[a] = c.p[a] / s2;
        c.lg[a] = logf(fminf(fmaxf(c.pn[a], eps), 1.0f - eps));
        ent -= c.pn[a] * c.lg[a];
    }
    logp = (action >= 0 && action < A) ? c.lg[action] : 0.0f;
}
// autograd's chain: gather + entropy -> log o clamp -> renormalisation -> softmax
__device__ __forceinline__ void cat_backward(const Cat& c, int A, int action, float gl, float ge, float* dz) {
    constexpr float eps = 1.1920928955078125e-07f;
    float dot = 0.0f;
    for (int a = 0; a < A; ++a) {
        const float dlg = (a == action ? gl : 0.0f) - ge * c.pn[a];
        const bool pass = c.pn[a] >= eps && c.pn[a] <= 1.0f - eps;
        dz[a] = -ge * c.lg[a] + (pass ? dlg / c.pn[a] : 0.0f);
        dot += dz[a] * c.pn[a];
    }
    float dot2 = 0.0f;
    for (int a = 0; a < A; ++a) { dz[a] = (dz[a] - dot) / c.s2; dot2 += dz[a] * c.p[a]; }
    for (int a = 0; a < A; ++a) dz[a] = c.p[a] * (dz[a] - dot2);
}

}  // namespace ppo
