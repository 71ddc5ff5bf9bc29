// Natural policy gradient / TRPO update arithmetic on a LAYERED actor (algorithm/modelfree/npg.py, trpo.py): the per-row
// kernels sit between the forward / tangent GEMMs and the backward GEMMs of net_gemm.cu, the vector kernels run the conjugate
// gradient and the parameter steps with every scalar in device memory, so a minibatch needs no host round trip.
//
// Reference: tianshou/algorithm/modelfree/npg.py:123-224 (preprocessing, vanilla gradient, Fisher-vector product with
// damping 0.1, conjugate gradient, natural step), trpo.py:132-191 (ratio surrogate, step size from s . MVP(s), backtracking
// line search), torch.distributions.kl (Normal / Independent / Categorical kl_divergence).
#include <math.h>

#include "common.cuh"
#include "ppo_math.cuh"

namespace {

constexpr int kMaxA = ppo::kCatMaxA;
constexpr float kProbEps = 1.1920928955078125e-07f;     // torch.finfo(float32).eps of clamp_probs
constexpr int kVecThreads = 1024;                       // one block: the reductions below have a fixed order

// Fixed-order sum over one block (blockDim.x a multiple of 32); every thread gets the result.
__device__ double block_sum(double v, double* sh /* [33] */) {
    for (int o = 16; o > 0; o >>= 1) v += tsb::shfl_down_f64(v, o);
    if (tsb::lane_id() == 0) sh[tsb::warp_id()] = v;
    __syncthreads();
    if (tsb::warp_id() == 0) {
        double t = tsb::lane_id() < (int)(blockDim.x >> 5) ? sh[tsb::lane_id()] : 0.0;
        for (int o = 16; o > 0; o >>= 1) t += tsb::shfl_down_f64(t, o);
        if (threadIdx.x == 0) sh[32] = t;
    }
    __syncthreads();
    const double r = sh[32];
    __syncthreads();
    return r;
}

// Gauss-Newton rows of the Fisher-vector product: out = H(head) . tangent(head) / B, H = Hessian of the row's
// KL(old || new) w.r.t. the head outputs at old = new.
//   Gaussian Independent(Normal(mu, exp(logstd))): H = diag(1 / sigma^2) for mu, 2 per action for logstd (mean over rows: the
//   logstd part is 2 * tangent(logstd), written once to out_logstd).
//   Categorical(probs = softmax(z)): KL = -sum_b p_old_b log clamp(pn_b) + const, d^2 log pn_b / dz^2 = -(diag(pn) - pn pn^T)
//   for every b inside the clamp and 0 outside, so H = c (diag(pn) - pn pn^T), c = sum of pn_b inside [eps, 1 - eps].
__global__ void fvp_rows_kernel(const float* __restrict__ head, const float* __restrict__ tangent, const float* __restrict__ logstd,
                                const float* __restrict__ tangent_logstd, int64_t B, int A, int categorical, float* __restrict__ out,
                                float* __restrict__ out_logstd) {
    const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const float inv_b = 1.0f / (float)B;
    if (!categorical && b < A) out_logstd[b] = 2.0f * tangent_logstd[b];
    if (b >= B) return;
    if (categorical) {
        float z[kMaxA];
        for (int a = 0; a < A; ++a) z[a] = head[b * A + a];
        ppo::Cat c;
        float lp, ent;
        ppo::cat_forward(z, A, -1, c, lp, ent);
        float mass = 0.0f, dot = 0.0f;
        for (int a = 0; a < A; ++a) {
            if (c.pn[a] >= kProbEps && c.pn[a] <= 1.0f - kProbEps) mass += c.pn[a];
            dot += c.pn[a] * tangent[b * A + a];
        }
        for (int a = 0; a < A; ++a) out[b * A + a] = mass * c.pn[a] * (tangent[b * A + a] - dot) * inv_b;
    } else {
        for (int a = 0; a < A; ++a) {
            const float sg = expf(logstd[a]);
            out[b * A + a] = tangent[b * A + a] / (sg * sg) * inv_b;
        }
    }
}

// Surrogate rows: log-prob, loss row (-logp * adv for NPG, -exp(logp - logp_old) * adv for TRPO; their mean is the actor
// loss) and, with dhead != NULL, d actor_loss / d head (+ per-row d / d logstd for a Gaussian head).
__global__ void npg_rows_kernel(const float* __restrict__ head, const float* __restrict__ logstd, const float* __restrict__ act,
                                const float* __restrict__ adv, const float* __restrict__ logp_old, int64_t B, int A, int categorical,
                                int ratio_surrogate, float* __restrict__ loss_rows, float* __restrict__ dhead,
                                float* __restrict__ dlogstd_rows) {
    const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const float inv_b = 1.0f / (float)B;
    float lp = 0.0f;
    if (categorical) {
        float z[kMaxA];
        for (int a = 0; a < A; ++a) z[a] = head[b * A + a];
        const int action = (int)act[b];
        ppo::Cat c;
        float ent;
        ppo::cat_forward(z, A, action, c, lp, ent);
        const float w = ratio_surrogate ? expf(lp - logp_old[b]) : 1.0f;
        loss_rows[b] = -(ratio_surrogate ? w : lp) * adv[b];
        if (dhead) {
            float dz[kMaxA];
            ppo::cat_backward(c, A, action, -w * adv[b] * inv_b, 0.0f, dz);
            for (int a = 0; a < A; ++a) dhead[b * A + a] = dz[a];
        }
    } else {
        for (int a = 0; a < A; ++a) lp += ppo::normal_logp_term(act[b * A + a], head[b * A + a], expf(logstd[a]));
        const float w = ratio_surrogate ? expf(lp - logp_old[b]) : 1.0f;
        loss_rows[b] = -(ratio_surrogate ? w : lp) * adv[b];
        if (dhead) {
            const float gl = -w * adv[b] * inv_b;
            for (int a = 0; a < A; ++a)
                ppo::normal_backward(act[b * A + a], head[b * A + a], expf(logstd[a]), gl, dhead[b * A + a], dlogstd_rows[b * A + a]);
        }
    }
}

// Row KL(old || new) in torch's formulas: Normal 0.5 (r + t1 - 1 - log r), r = (s_old / s_new)^2, t1 = ((mu_old - mu_new) /
// s_new)^2, summed over actions; Categorical sum p_old (logits_old - logits_new) with inf where p_new == 0 and 0 where
// p_old == 0 (kl.py _kl_categorical_categorical).
__global__ void kl_rows_kernel(const float* __restrict__ head_old, const float* __restrict__ logstd_old, const float* __restrict__ head_new,
                               const float* __restrict__ logstd_new, int64_t B, int A, int categorical, float* __restrict__ kl_rows) {
    const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    float kl = 0.0f;
    if (categorical) {
        float z[kMaxA];
        ppo::Cat co, cn;
        float lp, ent;
        for (int a = 0; a < A; ++a) z[a] = head_old[b * A + a];
        ppo::cat_forward(z, A, -1, co, lp, ent);
        for (int a = 0; a < A; ++a) z[a] = head_new[b * A + a];
        ppo::cat_forward(z, A, -1, cn, lp, ent);
        for (int a = 0; a < A; ++a) {
            float t = co.pn[a] * (co.lg[a] - cn.lg[a]);
            if (cn.pn[a] == 0.0f) t = INFINITY;
            if (co.pn[a] == 0.0f) t = 0.0f;
            kl += t;
        }
    } else {
        for (int a = 0; a < A; ++a) {
            const float so = expf(logstd_old[a]), sn = expf(logstd_new[a]);
            const float q = so / sn;
            const float r = q * q;
            const float d = (head_old[b * A + a] - head_new[b * A + a]) / sn;
            kl += 0.5f * (r + d * d - 1.0f - logf(r));
        }
    }
    kl_rows[b] = kl;
}

__global__ void mean_rows_kernel(const float* __restrict__ rows, int64_t B, float* __restrict__ out) {
    __shared__ double sh[33];
    double s = 0.0;
    for (int64_t i = threadIdx.x; i < B; i += blockDim.x) s += (double)rows[i];
    s = block_sum(s, sh);
    if (threadIdx.x == 0) *out = (float)(s / (double)B);
}

// state: [0] r.r, [1] done flag, [2] iterations run
__global__ void cg_init_kernel(const float* __restrict__ g, float* __restrict__ x, float* __restrict__ r, float* __restrict__ p,
                               int64_t n, double* __restrict__ state) {
    __shared__ double sh[33];
    double s = 0.0;
    for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
        const float v = g[i];
        x[i] = 0.0f; r[i] = v; p[i] = v;
        s += (double)v * v;
    }
    s = block_sum(s, sh);
    if (threadIdx.x == 0) { state[0] = s; state[1] = 0.0; state[2] = 0.0; }
}

// One iteration of npg.py:212-223 with z = F p on entry (damping folded in here: z += damping p).
__global__ void cg_step_kernel(float* __restrict__ x, float* __restrict__ r, float* __restrict__ p, float* __restrict__ z, int64_t n,
                               float damping, double residual_tol, double* __restrict__ state, float* __restrict__ iters_out) {
    __shared__ double sh[33];
    if (state[1] != 0.0) return;
    double pz = 0.0;
    for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
        const float zi = z[i] + p[i] * damping;
        z[i] = zi;
        pz += (double)p[i] * zi;
    }
    pz = block_sum(pz, sh);
    const double rdotr = state[0];
    const float alpha = (float)(rdotr / pz);
    double rr = 0.0;
    for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
        x[i] += alpha * p[i];
        const float ri = r[i] - alpha * z[i];
        r[i] = ri;
        rr += (double)ri * ri;
    }
    rr = block_sum(rr, sh);
    const double iters = state[2] + 1.0;
    if (rr < residual_tol) {
        if (threadIdx.x == 0) { state[1] = 1.0; state[2] = iters; if (iters_out) *iters_out = (float)iters; }
        return;
    }
    const float beta = (float)(rr / rdotr);
    for (int64_t i = threadIdx.x; i < n; i += blockDim.x) p[i] = r[i] + beta * p[i];
    if (threadIdx.x == 0) { state[0] = rr; state[2] = iters; if (iters_out) *iters_out = (float)iters; }
}

// trpo.py:152-159: z = F s on entry; step = sqrt(2 max_kl / (s . (z + damping s))).  stats_row[2] (kl) = 0 and
// stats_row[3] (step size) = step: what the reference reports when no candidate is evaluated.
__global__ void trpo_step_size_kernel(const float* __restrict__ s, const float* __restrict__ z, int64_t n, float damping, float two_max_kl,
                                      float* __restrict__ step, float* __restrict__ stats_row) {
    __shared__ double sh[33];
    double d = 0.0;
    for (int64_t i = threadIdx.x; i < n; i += blockDim.x) d += (double)s[i] * (z[i] + s[i] * damping);
    d = block_sum(d, sh);
    if (threadIdx.x == 0) {
        const float st = sqrtf(two_max_kl / (float)d);
        *step = st;
        stats_row[2] = 0.0f;
        stats_row[3] = st;
        stats_row[5] = -1.0f;
        stats_row[6] = 0.0f;
    }
}

__global__ void axpy_kernel(float* __restrict__ out, const float* __restrict__ theta, const float* __restrict__ dir, float coef,
                            const float* __restrict__ scale, int64_t n) {
    const float c = scale ? *scale * coef : coef;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        out[i] = theta[i] + c * dir[i];
}

// trpo.py:170-186 for candidate i: new loss / kl means, acceptance, step shrink or failure.
// flag: 0 rejected (another candidate follows), 1 accepted, 2 every candidate rejected.
__global__ void trpo_decide_kernel(const float* __restrict__ loss_rows, const float* __restrict__ kl_rows, int64_t B, int i,
                                   int max_backtracks, float max_kl, float backtrack_coeff, float* __restrict__ step,
                                   float* __restrict__ stats_row, int32_t* __restrict__ flag) {
    __shared__ double sh[33];
    double sl = 0.0, sk = 0.0;
    for (int64_t b = threadIdx.x; b < B; b += blockDim.x) { sl += (double)loss_rows[b]; sk += (double)kl_rows[b]; }
    sl = block_sum(sl, sh);
    sk = block_sum(sk, sh);
    if (threadIdx.x != 0) return;
    const float new_loss = (float)(sl / (double)B), kl = (float)(sk / (double)B);
    stats_row[2] = kl;
    if (kl < max_kl && new_loss < stats_row[0]) {
        *flag = 1;
        stats_row[3] = *step;
        stats_row[5] = (float)i;
    } else if (i < max_backtracks - 1) {
        *flag = 0;
        *step = *step * backtrack_coeff;
    } else {
        *flag = 2;
        stats_row[3] = 0.0f;
        stats_row[6] = 1.0f;
    }
}

// npg.py:136-137: whole-batch (adv - mean) / std, unbiased std, no epsilon.
__global__ void normalize_adv_kernel(float* __restrict__ adv, int64_t n) {
    __shared__ double sh[33];
    double s = 0.0;
    for (int64_t i = threadIdx.x; i < n; i += blockDim.x) s += (double)adv[i];
    const double mean = block_sum(s, sh) / (double)n;
    double q = 0.0;
    for (int64_t i = threadIdx.x; i < n; i += blockDim.x) { const double d = (double)adv[i] - mean; q += d * d; }
    const double var = block_sum(q, sh) / (double)(n - 1);
    const float m = (float)mean, sd = (float)sqrt(var);
    for (int64_t i = threadIdx.x; i < n; i += blockDim.x) adv[i] = (adv[i] - m) / sd;
}

unsigned row_blocks(int64_t B) { return (unsigned)((B + 127) / 128); }

}  // namespace

extern "C" int ts_npg_fvp_rows(const float* head, const float* tangent, const float* logstd, const float* tangent_logstd, int64_t B,
                               int32_t A, int32_t categorical, float* out, float* out_logstd, ts_stream_t stream) {
    TS_REQUIRE(head && tangent && out && A >= 1 && A <= kMaxA && B > 0, "ts_npg_fvp_rows: bad argument (act_dim <= %d)", kMaxA);
    TS_REQUIRE(categorical || (logstd && tangent_logstd && out_logstd), "ts_npg_fvp_rows: Gaussian head needs logstd");
    const int64_t threads = B > A ? B : A;
    fvp_rows_kernel<<<row_blocks(threads), 128, 0, tsb::as_stream(stream)>>>(head, tangent, logstd, tangent_logstd, B, A, categorical, out,
                                                                          out_logstd);
    return tsb::check_launch("ts_npg_fvp_rows");
}

extern "C" int ts_npg_rows(const float* head, const float* logstd, const float* act, const float* adv, const float* logp_old, int64_t B,
                           int32_t A, int32_t categorical, int32_t ratio_surrogate, float* loss_rows, float* dhead, float* dlogstd_rows,
                           ts_stream_t stream) {
    TS_REQUIRE(head && act && adv && loss_rows && A >= 1 && A <= kMaxA && B > 0, "ts_npg_rows: bad argument (act_dim <= %d)", kMaxA);
    TS_REQUIRE(categorical || logstd, "ts_npg_rows: Gaussian head needs logstd");
    TS_REQUIRE(!ratio_surrogate || logp_old, "ts_npg_rows: the ratio surrogate needs logp_old");
    TS_REQUIRE(!dhead || categorical || dlogstd_rows, "ts_npg_rows: Gaussian gradient needs dlogstd_rows");
    npg_rows_kernel<<<row_blocks(B), 128, 0, tsb::as_stream(stream)>>>(head, logstd, act, adv, logp_old, B, A, categorical, ratio_surrogate,
                                                                    loss_rows, dhead, dlogstd_rows);
    return tsb::check_launch("ts_npg_rows");
}

extern "C" int ts_npg_kl_rows(const float* head_old, const float* logstd_old, const float* head_new, const float* logstd_new, int64_t B,
                              int32_t A, int32_t categorical, float* kl_rows, ts_stream_t stream) {
    TS_REQUIRE(head_old && head_new && kl_rows && A >= 1 && A <= kMaxA && B > 0, "ts_npg_kl_rows: bad argument (act_dim <= %d)", kMaxA);
    TS_REQUIRE(categorical || (logstd_old && logstd_new), "ts_npg_kl_rows: Gaussian head needs logstd");
    kl_rows_kernel<<<row_blocks(B), 128, 0, tsb::as_stream(stream)>>>(head_old, logstd_old, head_new, logstd_new, B, A, categorical,
                                                                   kl_rows);
    return tsb::check_launch("ts_npg_kl_rows");
}

extern "C" int ts_npg_mean_rows(const float* rows, int64_t B, float* out, ts_stream_t stream) {
    TS_REQUIRE(rows && out && B > 0, "ts_npg_mean_rows: bad argument");
    mean_rows_kernel<<<1, kVecThreads, 0, tsb::as_stream(stream)>>>(rows, B, out);
    return tsb::check_launch("ts_npg_mean_rows");
}

extern "C" int ts_cg_init(const float* g, float* x, float* r, float* p, int64_t n, double* state, ts_stream_t stream) {
    TS_REQUIRE(g && x && r && p && state && n > 0, "ts_cg_init: bad argument");
    cg_init_kernel<<<1, kVecThreads, 0, tsb::as_stream(stream)>>>(g, x, r, p, n, state);
    return tsb::check_launch("ts_cg_init");
}

extern "C" int ts_cg_step(float* x, float* r, float* p, float* z, int64_t n, double damping, double residual_tol, double* state,
                          float* iters_out, ts_stream_t stream) {
    TS_REQUIRE(x && r && p && z && state && n > 0, "ts_cg_step: bad argument");
    cg_step_kernel<<<1, kVecThreads, 0, tsb::as_stream(stream)>>>(x, r, p, z, n, (float)damping, residual_tol, state, iters_out);
    return tsb::check_launch("ts_cg_step");
}

extern "C" int ts_trpo_step_size(const float* s, const float* z, int64_t n, double damping, double max_kl, float* step, float* stats_row,
                                 ts_stream_t stream) {
    TS_REQUIRE(s && z && step && stats_row && n > 0, "ts_trpo_step_size: bad argument");
    trpo_step_size_kernel<<<1, kVecThreads, 0, tsb::as_stream(stream)>>>(s, z, n, (float)damping, (float)(2.0 * max_kl), step, stats_row);
    return tsb::check_launch("ts_trpo_step_size");
}

extern "C" int ts_npg_axpy(float* out, const float* theta, const float* dir, double coef, const float* scale, int64_t n,
                           ts_stream_t stream) {
    TS_REQUIRE(out && theta && dir && n > 0, "ts_npg_axpy: bad argument");
    const int64_t blocks = tsb::imin((n + 255) / 256, (int64_t)tsb::num_sms() * 8);
    axpy_kernel<<<(unsigned)blocks, 256, 0, tsb::as_stream(stream)>>>(out, theta, dir, (float)coef, scale, n);
    return tsb::check_launch("ts_npg_axpy");
}

extern "C" int ts_trpo_decide(const float* loss_rows, const float* kl_rows, int64_t B, int32_t i, int32_t max_backtracks, double max_kl,
                              double backtrack_coeff, float* step, float* stats_row, int32_t* flag, ts_stream_t stream) {
    TS_REQUIRE(loss_rows && kl_rows && step && stats_row && flag && B > 0 && i >= 0 && i < max_backtracks, "ts_trpo_decide: bad argument");
    trpo_decide_kernel<<<1, kVecThreads, 0, tsb::as_stream(stream)>>>(loss_rows, kl_rows, B, i, max_backtracks, (float)max_kl,
                                                                     (float)backtrack_coeff, step, stats_row, flag);
    return tsb::check_launch("ts_trpo_decide");
}

extern "C" int ts_npg_normalize_adv(float* adv, int64_t n, ts_stream_t stream) {
    TS_REQUIRE(adv && n > 1, "ts_npg_normalize_adv: needs at least two rows");
    normalize_adv_kernel<<<1, kVecThreads, 0, tsb::as_stream(stream)>>>(adv, n);
    return tsb::check_launch("ts_npg_normalize_adv");
}
