// Rainbow arithmetic (algorithm/modelfree/rainbow.py): the noisy layers' effective weights and the split of their gradient, and
// the dueling combine of the categorical heads.  The GEMMs are the layered-network launches of net_gemm.cu; C51's kernels
// (c51.cu) run unchanged on the combined logits.
//
// Reference: tianshou/utils/net/discrete.py NoisyLinear (the train-mode weight mu_W + sigma_W * ger(eps_q, eps_p) and bias
// mu_bias + sigma_bias * eps_q, formed by three separate fp32 ops), tianshou/utils/net/common.py:355-364 and
// tianshou/env/atari/atari_network.py:196-206 (logits = q - q.mean(dim=1, keepdim=True) + v over [B][A][N]).
#include <math.h>

#include "common.cuh"

namespace {

constexpr int kThreads = 256;

inline unsigned grid_for(int64_t items) {
    int64_t b = (items + kThreads - 1) / kThreads;
    const int64_t cap = (int64_t)tsb::num_sms() * 8;
    return (unsigned)(b > cap ? cap : (b < 1 ? 1 : b));
}

// w_eff[o][i] = mu_w + sigma_w * (eps_q[o] * eps_p[i]) and b_eff[o] = mu_b + sigma_b * eps_q[o], each product and sum rounded on
// its own (no FMA contraction): bit for bit torch's outer product, then *, then +.  Grid-stride over out * in + out elements.
__global__ void __launch_bounds__(kThreads) noisy_weight_kernel(
        const float* __restrict__ mu_w, const float* __restrict__ sigma_w, const float* __restrict__ mu_b,
        const float* __restrict__ sigma_b, const float* __restrict__ eps_p, const float* __restrict__ eps_q, int out, int in,
        float* __restrict__ w_eff, float* __restrict__ b_eff) {
    const int64_t nw = (int64_t)out * in;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < nw + out; e += (int64_t)gridDim.x * blockDim.x) {
        if (e < nw) {
            const int o = (int)(e / in), i = (int)(e - (int64_t)o * in);
            w_eff[e] = __fadd_rn(mu_w[e], __fmul_rn(sigma_w[e], __fmul_rn(eps_q[o], eps_p[i])));
        } else {
            const int o = (int)(e - nw);
            b_eff[o] = __fadd_rn(mu_b[o], __fmul_rn(sigma_b[o], eps_q[o]));
        }
    }
}

// The gradients of the four trainable tensors from the effective weight's and bias's: d mu_w = dw, d sigma_w = dw * (eps_q[o] *
// eps_p[i]), d mu_b = db, d sigma_b = db * eps_q[o] (autograd of the forward above: mul's gradient times the other operand).
__global__ void __launch_bounds__(kThreads) noisy_grad_kernel(
        const float* __restrict__ dw, const float* __restrict__ db, const float* __restrict__ eps_p, const float* __restrict__ eps_q,
        int out, int in, float* __restrict__ g_mu_w, float* __restrict__ g_sigma_w, float* __restrict__ g_mu_b,
        float* __restrict__ g_sigma_b) {
    const int64_t nw = (int64_t)out * in;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < nw + out; e += (int64_t)gridDim.x * blockDim.x) {
        if (e < nw) {
            const int o = (int)(e / in), i = (int)(e - (int64_t)o * in);
            const float g = dw[e];
            g_mu_w[e] = g;
            g_sigma_w[e] = __fmul_rn(g, __fmul_rn(eps_q[o], eps_p[i]));
        } else {
            const int o = (int)(e - nw);
            const float g = db[o];
            g_mu_b[o] = g;
            g_sigma_b[o] = __fmul_rn(g, eps_q[o]);
        }
    }
}

// logits[b][a][n] = (q[b][a][n] - m) + v[b][n] with m = (sum_a q[b][a][n] in index order) / A.  One thread per (b, n).
__global__ void __launch_bounds__(kThreads) dueling_atoms_kernel(const float* __restrict__ q, const float* __restrict__ v, int64_t B,
                                                                int A, int N, float* __restrict__ logits) {
    const int64_t AN = (int64_t)A * N;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < B * N; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t b = e / N;
        const int n = (int)(e - b * N);
        const float* qb = q + b * AN + n;
        float acc = qb[0];
        for (int a = 1; a < A; ++a) acc = __fadd_rn(acc, qb[(int64_t)a * N]);
        const float m = __fdiv_rn(acc, (float)A), vb = v[e];
        float* lb = logits + b * AN + n;
        for (int a = 0; a < A; ++a) lb[(int64_t)a * N] = __fadd_rn(__fsub_rn(qb[(int64_t)a * N], m), vb);
    }
}

// dv[b][n] = s = sum_a dl[b][a][n] (index order), dq[b][a][n] = dl[b][a][n] - s / A.  One thread per (b, n), no atomics.
__global__ void __launch_bounds__(kThreads) dueling_atoms_bwd_kernel(const float* __restrict__ dl, int64_t B, int A, int N,
                                                                    float* __restrict__ dq, float* __restrict__ dv) {
    const int64_t AN = (int64_t)A * N;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < B * N; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t b = e / N;
        const int n = (int)(e - b * N);
        const float* db = dl + b * AN + n;
        float s = db[0];
        for (int a = 1; a < A; ++a) s = __fadd_rn(s, db[(int64_t)a * N]);
        dv[e] = s;
        const float sa = __fdiv_rn(s, (float)A);
        float* qb = dq + b * AN + n;
        for (int a = 0; a < A; ++a) qb[(int64_t)a * N] = __fsub_rn(db[(int64_t)a * N], sa);
    }
}

}  // namespace

extern "C" int ts_noisy_weight(const float* mu_w, const float* sigma_w, const float* mu_b, const float* sigma_b, const float* eps_p,
                               const float* eps_q, int32_t out, int32_t in, float* w_eff, float* b_eff, ts_stream_t stream) {
    TS_REQUIRE(mu_w && sigma_w && mu_b && sigma_b && eps_p && eps_q && w_eff && b_eff && out >= 1 && in >= 1,
               "ts_noisy_weight: bad argument");
    const int64_t n = (int64_t)out * in + out;
    noisy_weight_kernel<<<grid_for(n), kThreads, 0, tsb::as_stream(stream)>>>(mu_w, sigma_w, mu_b, sigma_b, eps_p, eps_q, out, in,
                                                                              w_eff, b_eff);
    return tsb::check_launch("ts_noisy_weight");
}

extern "C" int ts_noisy_grad(const float* dw, const float* db, const float* eps_p, const float* eps_q, int32_t out, int32_t in,
                             float* g_mu_w, float* g_sigma_w, float* g_mu_b, float* g_sigma_b, ts_stream_t stream) {
    TS_REQUIRE(dw && db && eps_p && eps_q && g_mu_w && g_sigma_w && g_mu_b && g_sigma_b && out >= 1 && in >= 1,
               "ts_noisy_grad: bad argument");
    const int64_t n = (int64_t)out * in + out;
    noisy_grad_kernel<<<grid_for(n), kThreads, 0, tsb::as_stream(stream)>>>(dw, db, eps_p, eps_q, out, in, g_mu_w, g_sigma_w, g_mu_b,
                                                                            g_sigma_b);
    return tsb::check_launch("ts_noisy_grad");
}

extern "C" int ts_dueling_atoms(const float* q, const float* v, int64_t B, int32_t A, int32_t N, float* logits, ts_stream_t stream) {
    TS_REQUIRE(q && v && logits && B >= 0 && A >= 1 && N >= 1, "ts_dueling_atoms: bad argument");
    if (B == 0) return 0;
    dueling_atoms_kernel<<<grid_for(B * N), kThreads, 0, tsb::as_stream(stream)>>>(q, v, B, A, N, logits);
    return tsb::check_launch("ts_dueling_atoms");
}

extern "C" int ts_dueling_atoms_bwd(const float* dlogits, int64_t B, int32_t A, int32_t N, float* dq, float* dv, ts_stream_t stream) {
    TS_REQUIRE(dlogits && dq && dv && B >= 0 && A >= 1 && N >= 1, "ts_dueling_atoms_bwd: bad argument");
    if (B == 0) return 0;
    dueling_atoms_bwd_kernel<<<grid_for(B * N), kThreads, 0, tsb::as_stream(stream)>>>(dlogits, B, A, N, dq, dv);
    return tsb::check_launch("ts_dueling_atoms_bwd");
}
