// BCQ arithmetic (algorithm/imitation/bcq.py): the per-row pieces between the GEMMs of the VAE, the perturbation network and the
// critics.  The GEMMs themselves are the layered-network launches of net_gemm.cu; the critics' squared-loss step reuses
// ts_critic_mse (net_ops.cu) and the actor loss -mean Q1 reuses ts_td3_actor_rows (td3.cu).
//
// Reference: tianshou/utils/net/continuous.py:407-412 (Perturbation: clamp(a + phi * max_action * tanh(logits), +-max_action)),
// :455-490 (VAE: log_std clamped to [-4, 15], z = mean + std * eps, decode = max_action * tanh(decoder([s | z])), latent clamped to
// +-0.5 when drawn), algorithm/imitation/bcq.py:196-256 (VAE loss, lmbda-mixed target with the max over the sampled actions,
// one-step done-masked target), :91-116 (the policy's argmax over sampled actions).  Where the rounding order matters it
// follows torch's operation order with __f*_rn, as td3.cu and cql.cu do.
#include <math.h>

#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kRowThreads = 1024;

// torch.clamp: NaN passes through
__device__ __forceinline__ float clampf(float x, float lo, float hi) { return x != x ? x : fminf(fmaxf(x, lo), hi); }

// [s | z] with std = exp(clamp(log_std_raw, -4, 15)), z = mean + std * eps; head = [mean | log_std_raw] [B][2L].  Grid-stride
// over the B * (O + L) elements of x.
__global__ void __launch_bounds__(kThreads) bcq_vae_reparam_kernel(
        const float* __restrict__ head, const float* __restrict__ eps, int64_t B, int L, const float* __restrict__ s, int O,
        float* __restrict__ std_out, float* __restrict__ x) {
    const int W = O + L;
    const int64_t n = B * W;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) {
        const int64_t b = t / W;
        const int c = (int)(t - b * W);
        if (c < O) {
            x[t] = s[b * O + c];
            continue;
        }
        const int j = c - O;
        const float sd = expf(clampf(head[b * 2 * L + L + j], -4.0f, 15.0f));
        std_out[b * L + j] = sd;
        x[t] = __fadd_rn(head[b * 2 * L + j], __fmul_rn(sd, eps[b * L + j]));
    }
}

// One block.  Fixed-order sums of (act - recon)^2 and of the KL terms -log std + (std^2 + mean^2 - 1) / 2, then
// loss = sum_sq / (B A) + (sum_kl / (B L)) / 2, and dy = d loss / d y through recon = max_action * tanh(y) for every element
// (block-stride).
__global__ void __launch_bounds__(kRowThreads) bcq_vae_loss_kernel(
        const float* __restrict__ y, const float* __restrict__ act, const float* __restrict__ head, const float* __restrict__ sd,
        int64_t B, int A, int L, float max_action, float* __restrict__ dy, float* __restrict__ loss) {
    __shared__ float part[2][kRowThreads / 32];
    const int64_t na = B * A, nl = B * L;
    const float inv_n = __fdiv_rn(2.0f, (float)na);
    float sq = 0.0f, kl = 0.0f;
    for (int64_t e = threadIdx.x; e < na; e += kRowThreads) {
        const float t = tanhf(y[e]);
        const float d = __fsub_rn(act[e], __fmul_rn(max_action, t));
        sq = __fadd_rn(sq, __fmul_rn(d, d));
        dy[e] = __fmul_rn(__fmul_rn(__fmul_rn(-d, inv_n), max_action), __fsub_rn(1.0f, __fmul_rn(t, t)));
    }
    for (int64_t e = threadIdx.x; e < nl; e += kRowThreads) {
        const int64_t b = e / L;
        const float m = head[b * 2 * L + (e - b * L)], v = sd[e];
        const float q = __fdiv_rn(__fsub_rn(__fadd_rn(__fmul_rn(v, v), __fmul_rn(m, m)), 1.0f), 2.0f);
        kl = __fadd_rn(kl, __fadd_rn(-logf(v), q));
    }
    sq = tsb::warp_sum(sq);
    kl = tsb::warp_sum(kl);
    if (tsb::lane_id() == 0) {
        part[0][tsb::warp_id()] = sq;
        part[1][tsb::warp_id()] = kl;
    }
    __syncthreads();
    if (tsb::warp_id() == 0) {
        const float a = tsb::warp_sum(part[0][tsb::lane_id()]);
        const float k = tsb::warp_sum(part[1][tsb::lane_id()]);
        if (tsb::lane_id() == 0) *loss = __fadd_rn(__fdiv_rn(a, (float)na), __fdiv_rn(__fdiv_rn(k, (float)nl), 2.0f));
    }
}

// d[mean | log_std_raw] from dz = d loss / d z (the decoder's input gradient over the z columns) and the KL term:
//   dmean = dz + g 2 mean,  dstd = dz eps - 2 g / std + g 2 std,  dlog_std_raw = [-4 <= raw <= 15] dstd std,
// g = (1/2) (1/(B L)) / 2 the gradient reaching each of std^2 and mean^2 (torch's clamp passes the gradient at the bounds).
__global__ void __launch_bounds__(kThreads) bcq_vae_head_bwd_kernel(
        const float* __restrict__ head, const float* __restrict__ sd, const float* __restrict__ eps, const float* __restrict__ dz,
        int64_t B, int L, float* __restrict__ dhead) {
    const int64_t n = B * L;
    const float g_kl = __fdiv_rn(0.5f, (float)n);          // d loss / d (KL element)
    const float g_sq = __fdiv_rn(g_kl, 2.0f);              // through (... ) / 2
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t b = e / L;
        const int j = (int)(e - b * L);
        const float m = head[b * 2 * L + j], raw = head[b * 2 * L + L + j], v = sd[e], d = dz[e];
        dhead[b * 2 * L + j] = __fadd_rn(d, __fmul_rn(g_sq, __fmul_rn(2.0f, m)));
        const float dstd = __fadd_rn(__fadd_rn(__fmul_rn(d, eps[e]), __fdiv_rn(-g_kl, v)), __fmul_rn(g_sq, __fmul_rn(2.0f, v)));
        dhead[b * 2 * L + L + j] = (raw >= -4.0f && raw <= 15.0f) ? __fmul_rn(dstd, v) : 0.0f;
    }
}

// x [B N][O + L] = [s[r / N] | clamp(z[r], -clip, clip)]: repeat_interleave of s fused with the latent clamp.  Grid-stride.
__global__ void __launch_bounds__(kThreads) bcq_decode_input_kernel(
        const float* __restrict__ s, int64_t B, int N, int O, const float* __restrict__ z, int L, float clip,
        float* __restrict__ x) {
    const int W = O + L;
    const int64_t n = B * N * W;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = t / W;
        const int c = (int)(t - r * W);
        x[t] = c < O ? s[(r / N) * O + c] : clampf(z[r * L + (c - O)], -clip, clip);
    }
}

// x [rows][O + A] = [s[r step] | max_action * tanh(y[r step])]: the decoder's action rows beside their states (s: row stride
// lds).  Grid-stride.
__global__ void __launch_bounds__(kThreads) bcq_act_rows_kernel(
        const float* __restrict__ s, int64_t lds, const float* __restrict__ y, int64_t step, int64_t rows, int O, int A,
        float max_action, float* __restrict__ x) {
    const int W = O + A;
    const int64_t n = rows * W;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = t / W;
        const int c = (int)(t - r * W);
        const int64_t src = r * step;
        x[t] = c < O ? s[src * lds + c] : __fmul_rn(max_action, tanhf(y[src * A + (c - O)]));
    }
}

// x [rows][O + A] = [s[r] | clamp(vae_max tanh(y[r]) + phi_m tanh(logits[r / S]), +-max_action)] (phi_m = phi * max_action;
// vae_max scales the VAE's decoded action, max_action is the perturbation's).  Grid-stride.
__global__ void __launch_bounds__(kThreads) bcq_perturb_kernel(
        const float* __restrict__ logits, int64_t S, const float* __restrict__ y, int64_t rows, int A, float vae_max,
        float max_action, float phi_m, const float* __restrict__ s, int64_t lds, int O, float* __restrict__ x) {
    const int W = O + A;
    const int64_t n = rows * W;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = t / W;
        const int c = (int)(t - r * W);
        if (c < O) {
            x[t] = s[r * lds + c];
            continue;
        }
        const int j = c - O;
        const float a = __fmul_rn(vae_max, tanhf(y[r * A + j]));
        const float noise = __fmul_rn(tanhf(logits[(r / S) * A + j]), phi_m);
        x[t] = clampf(__fadd_rn(noise, a), -max_action, max_action);
    }
}

// dlogits [G][A] of the perturbation: per group g of S rows and column j, the fixed-order sum over the group of dact where the
// clamp passed (-max_action <= pre <= max_action, inclusive as torch's clamp backward), times phi_m (1 - tanh(logits)^2).  One
// block per group (grid-stride over groups).
__global__ void __launch_bounds__(kThreads) bcq_perturb_bwd_kernel(
        const float* __restrict__ logits, int64_t S, int64_t G, const float* __restrict__ y, const float* __restrict__ dact, int A,
        float vae_max, float max_action, float phi_m, float* __restrict__ dlogits) {
    __shared__ float part[kThreads / 32];
    for (int64_t g = blockIdx.x; g < G; g += gridDim.x) {
        for (int j = 0; j < A; ++j) {
            const float t = tanhf(logits[g * A + j]);
            const float noise = __fmul_rn(t, phi_m);
            float acc = 0.0f;
            for (int64_t i = threadIdx.x; i < S; i += kThreads) {
                const int64_t e = (g * S + i) * A + j;
                const float pre = __fadd_rn(noise, __fmul_rn(vae_max, tanhf(y[e])));
                if (pre >= -max_action && pre <= max_action) acc = __fadd_rn(acc, dact[e]);
            }
            acc = tsb::warp_sum(acc);
            if (tsb::lane_id() == 0) part[tsb::warp_id()] = acc;
            __syncthreads();
            if (threadIdx.x == 0) {
                float tot = 0.0f;
#pragma unroll
                for (int w = 0; w < kThreads / 32; ++w) tot = __fadd_rn(tot, part[w]);
                dlogits[g * A + j] = __fmul_rn(__fmul_rn(tot, phi_m), __fsub_rn(1.0f, __fmul_rn(t, t)));
            }
            __syncthreads();
        }
    }
}

// out[b] = rew[b] + logical_not(done[b]) * gamma * max_j (lmbda min(q1, q2) + (1 - lmbda) max(q1, q2)) over the N rows of group
// b; NaN propagates through min, max and the group max.  Grid-stride over groups.
__global__ void __launch_bounds__(kThreads) bcq_target_kernel(
        const float* __restrict__ q1, const float* __restrict__ q2, int64_t B, int N, float lmbda, float one_minus_lmbda,
        const float* __restrict__ rew, const float* __restrict__ done, float gamma, float* __restrict__ out) {
    for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b < B; b += (int64_t)gridDim.x * blockDim.x) {
        float best = 0.0f;
        for (int j = 0; j < N; ++j) {
            const float u = q1[b * N + j], w = q2[b * N + j];
            const bool nan = u != u || w != w;
            const float mn = nan ? __fadd_rn(u, w) : fminf(u, w), mx = nan ? __fadd_rn(u, w) : fmaxf(u, w);
            const float v = __fadd_rn(__fmul_rn(lmbda, mn), __fmul_rn(one_minus_lmbda, mx));
            if (j == 0 || v != v || v > best) best = v;
            if (v != v) break;
        }
        const float nd = done[b] != 0.0f ? 0.0f : 1.0f;
        out[b] = __fadd_rn(rew[b], __fmul_rn(__fmul_rn(nd, gamma), best));
    }
}

// Per group g of S rows of q: the first index of the maximum (torch.argmax: a NaN is the maximum, the first NaN wins); its row
// of x (columns col0 .. col0 + A, row stride ldx) goes to act[g], the index to idx[g] (nullable).  Grid-stride over groups.
__global__ void __launch_bounds__(kThreads) bcq_select_kernel(
        const float* __restrict__ q, int64_t G, int64_t S, const float* __restrict__ x, int64_t ldx, int col0, int A,
        float* __restrict__ act, int64_t* __restrict__ idx) {
    for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < G; g += (int64_t)gridDim.x * blockDim.x) {
        int64_t bi = 0;
        float best = q[g * S];
        if (best == best) {
            for (int64_t i = 1; i < S; ++i) {
                const float v = q[g * S + i];
                if (v != v) {
                    bi = i;
                    break;
                }
                if (v > best) {
                    best = v;
                    bi = i;
                }
            }
        }
        const float* row = x + (g * S + bi) * ldx + col0;
        for (int c = 0; c < A; ++c) act[g * A + c] = row[c];
        if (idx) idx[g] = bi;
    }
}

inline unsigned grid_for(int64_t items) {
    int64_t b = (items + kThreads - 1) / kThreads;
    const int64_t cap = (int64_t)tsb::num_sms() * 4;
    return (unsigned)(b > cap ? cap : (b < 1 ? 1 : b));
}

inline unsigned grid_groups(int64_t groups) {
    const int64_t cap = (int64_t)tsb::num_sms() * 8;
    return (unsigned)(groups > cap ? cap : (groups < 1 ? 1 : groups));
}

}  // namespace

extern "C" int ts_bcq_vae_reparam(const float* head, const float* eps, int64_t B, int32_t L, const float* s, int32_t O,
                                  float* std_out, float* x, ts_stream_t stream) {
    TS_REQUIRE(head && eps && s && std_out && x && B >= 0 && L >= 1 && O >= 0, "ts_bcq_vae_reparam: bad argument");
    if (B == 0) return 0;
    bcq_vae_reparam_kernel<<<grid_for(B * (O + L)), kThreads, 0, tsb::as_stream(stream)>>>(head, eps, B, L, s, O, std_out, x);
    return tsb::check_launch("ts_bcq_vae_reparam");
}

extern "C" int ts_bcq_vae_loss(const float* y, const float* act, const float* head, const float* std_in, int64_t B, int32_t A,
                               int32_t L, float max_action, float* dy, float* loss, ts_stream_t stream) {
    TS_REQUIRE(y && act && head && std_in && dy && loss && B >= 1 && A >= 1 && L >= 1, "ts_bcq_vae_loss: bad argument");
    bcq_vae_loss_kernel<<<1, kRowThreads, 0, tsb::as_stream(stream)>>>(y, act, head, std_in, B, A, L, max_action, dy, loss);
    return tsb::check_launch("ts_bcq_vae_loss");
}

extern "C" int ts_bcq_vae_head_bwd(const float* head, const float* std_in, const float* eps, const float* dz, int64_t B, int32_t L,
                                   float* dhead, ts_stream_t stream) {
    TS_REQUIRE(head && std_in && eps && dz && dhead && B >= 1 && L >= 1, "ts_bcq_vae_head_bwd: bad argument");
    bcq_vae_head_bwd_kernel<<<grid_for(B * L), kThreads, 0, tsb::as_stream(stream)>>>(head, std_in, eps, dz, B, L, dhead);
    return tsb::check_launch("ts_bcq_vae_head_bwd");
}

extern "C" int ts_bcq_decode_input(const float* s, int64_t B, int32_t N, int32_t O, const float* z, int32_t L, float clip, float* x,
                                   ts_stream_t stream) {
    TS_REQUIRE(s && z && x && B >= 0 && N >= 1 && O >= 0 && L >= 1, "ts_bcq_decode_input: bad argument");
    if (B == 0) return 0;
    bcq_decode_input_kernel<<<grid_for(B * N * (O + L)), kThreads, 0, tsb::as_stream(stream)>>>(s, B, N, O, z, L, clip, x);
    return tsb::check_launch("ts_bcq_decode_input");
}

extern "C" int ts_bcq_act_rows(const float* s, int64_t lds, const float* y, int64_t step, int64_t rows, int32_t O, int32_t A,
                               float max_action, float* x, ts_stream_t stream) {
    TS_REQUIRE(s && y && x && rows >= 0 && step >= 1 && lds >= O && O >= 0 && A >= 1, "ts_bcq_act_rows: bad argument");
    if (rows == 0) return 0;
    bcq_act_rows_kernel<<<grid_for(rows * (O + A)), kThreads, 0, tsb::as_stream(stream)>>>(s, lds, y, step, rows, O, A, max_action, x);
    return tsb::check_launch("ts_bcq_act_rows");
}

extern "C" int ts_bcq_perturb(const float* logits, int64_t S, const float* y, int64_t rows, int32_t A, float vae_max, float max_action,
                              float phi_m, const float* s, int64_t lds, int32_t O, float* x, ts_stream_t stream) {
    TS_REQUIRE(logits && y && s && x && S >= 1 && rows >= 0 && A >= 1 && O >= 0 && lds >= O, "ts_bcq_perturb: bad argument");
    if (rows == 0) return 0;
    bcq_perturb_kernel<<<grid_for(rows * (O + A)), kThreads, 0, tsb::as_stream(stream)>>>(logits, S, y, rows, A, vae_max, max_action,
                                                                                         phi_m, s, lds, O, x);
    return tsb::check_launch("ts_bcq_perturb");
}

extern "C" int ts_bcq_perturb_bwd(const float* logits, int64_t S, int64_t G, const float* y, const float* dact, int32_t A,
                                  float vae_max, float max_action, float phi_m, float* dlogits, ts_stream_t stream) {
    TS_REQUIRE(logits && y && dact && dlogits && S >= 1 && G >= 0 && A >= 1, "ts_bcq_perturb_bwd: bad argument");
    if (G == 0) return 0;
    bcq_perturb_bwd_kernel<<<grid_groups(G), kThreads, 0, tsb::as_stream(stream)>>>(logits, S, G, y, dact, A, vae_max, max_action,
                                                                                   phi_m, dlogits);
    return tsb::check_launch("ts_bcq_perturb_bwd");
}

extern "C" int ts_bcq_target(const float* q1, const float* q2, int64_t B, int32_t N, float lmbda, float one_minus_lmbda,
                             const float* rew, const float* done, float gamma, float* out, ts_stream_t stream) {
    TS_REQUIRE(q1 && q2 && rew && done && out && B >= 0 && N >= 1, "ts_bcq_target: bad argument");
    if (B == 0) return 0;
    bcq_target_kernel<<<grid_for(B), kThreads, 0, tsb::as_stream(stream)>>>(q1, q2, B, N, lmbda, one_minus_lmbda, rew, done, gamma,
                                                                           out);
    return tsb::check_launch("ts_bcq_target");
}

extern "C" int ts_bcq_select(const float* q, int64_t G, int64_t S, const float* x, int64_t ldx, int32_t col0, int32_t A, float* act,
                             int64_t* idx, ts_stream_t stream) {
    TS_REQUIRE(q && x && act && G >= 0 && S >= 1 && A >= 1 && col0 >= 0 && ldx >= col0 + A, "ts_bcq_select: bad argument");
    if (G == 0) return 0;
    bcq_select_kernel<<<grid_for(G), kThreads, 0, tsb::as_stream(stream)>>>(q, G, S, x, ldx, col0, A, act, idx);
    return tsb::check_launch("ts_bcq_select");
}
