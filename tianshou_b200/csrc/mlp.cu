// Actor-critic MLP kernels for the PPO update, fp32 SIMT baseline path (sm_90a).
//
// Network (examples/mujoco/mujoco_ppo.py:90-120): actor  obs -> 64 -> 64 -(tanh)-> mu[act] with a
// state-independent log-sigma, critic obs -> 64 -> 64 -(tanh)-> 1; torch layouts ([out][in]).
// Reference code replaced:
//   critic forward in 256-row Python chunks        modelfree/a2c.py:123-126
//   logp_old in 256-row Python chunks              modelfree/ppo.py:157-161, reinforce.py:167-192
//   minibatch loss + autograd backward             modelfree/ppo.py:179-211, algorithm_base.py:497
//   clip_grad_norm_ + Adam.step                    algorithm_base.py:498-500, optim.py:89-110
//
// Design: one CTA = one tile of 128 rows; all weights of the net being evaluated are staged in
// shared memory once per CTA (k-major copies for the forward GEMMs, the natural [out][in] copy of
// W2 for the input-gradient GEMM); activations of the tile never leave shared memory between
// forward and backward; each thread owns an 8x4 register tile of every 128x64 layer output.
// Weight gradients are reduced over the 128 rows inside the CTA and then added to the flat
// gradient buffer with one RED per parameter per CTA.  Loss sums ride in the same buffer so that
// a multi-GPU caller needs exactly one allreduce per optimiser step.
#include <math.h>
#include <stdlib.h>

#include "common.cuh"
#include "optim_math.cuh"
#include "ppo_math.cuh"

namespace {

constexpr int H = 64;          // hidden width (both layers)
constexpr int kRows = 128;     // rows per CTA tile
constexpr int kThreads = 256;
constexpr int LDH = H + 4;     // activation tile leading dimension (bank shift of 4 per row)
constexpr int LDW3 = H + 4;    // head weight rows, padded
constexpr int LDO = 32;        // dout tile leading dim: [0,A) = dmu, [16,16+A) = dlogstd terms
constexpr int kMaxAct = 16;
constexpr int kMaxObs = 64;

struct NetOff {  // shared-memory offsets (floats) of one network's staged weights
    int w1t, b1, w2t, w2, b2, w3, b3, ls;
};
struct Layout {
    int KX, LDX, A;
    NetOff actor, critic;
    int X, H1, H2, ACT, DOUT, ROWV, RED;
    int total;  // floats
};

__host__ __device__ inline int roundup4(int x) { return (x + 3) & ~3; }

// mode: 0 = critic forward only, 1 = actor forward only, 2 = train (both, with backward copies)
__host__ __device__ inline Layout make_layout(int obs_dim, int act_dim, int mode) {
    Layout L;
    L.KX = roundup4(obs_dim);
    L.LDX = L.KX + 4;
    L.A = act_dim;
    int o = 0;
    auto net = [&](NetOff& n, int out_dim, bool need) {
        n = NetOff{0, 0, 0, 0, 0, 0, 0, 0};
        if (!need) return;
        n.w1t = o; o += L.KX * H;
        n.b1 = o;  o += H;
        n.w2t = o; o += H * H;
        n.w2 = o;  o += (mode == 2) ? H * H : 0;
        n.b2 = o;  o += H;
        n.w3 = o;  o += out_dim * LDW3;
        n.b3 = o;  o += kMaxAct;
        n.ls = o;  o += kMaxAct;
    };
    net(L.actor, act_dim, mode != 0);
    net(L.critic, 1, mode != 1);
    L.X = o;    o += kRows * L.LDX;
    L.H1 = o;   o += kRows * LDH;
    L.H2 = o;   o += kRows * LDH;
    L.ACT = o;  o += (mode != 0) ? kRows * kMaxAct : 0;
    L.DOUT = o; o += (mode == 2) ? kRows * LDO : 0;
    L.ROWV = o; o += 4 * kRows;   // adv, ret, logp_old, v_s  (train) / scratch
    L.RED = o;  o += 64;
    L.total = o;
    return L;
}

struct NetGlobal {  // offsets into the flat parameter buffer
    int64_t w1, b1, w2, b2, w3, b3, ls;
};

// ---- staging ------------------------------------------------------------------------------
__device__ void stage_net(float* sm, const NetOff& n, const float* __restrict__ params,
                          const NetGlobal& g, int obs_dim, int KX, int out_dim, bool with_w2,
                          bool with_ls) {
    const int tid = threadIdx.x;
    // W1 [H][obs] -> w1t [KX][H] (zero rows for k >= obs_dim)
    for (int e = tid; e < KX * H; e += kThreads) {
        const int k = e / H, c = e - k * H;
        sm[n.w1t + e] = (k < obs_dim) ? __ldg(params + g.w1 + (int64_t)c * obs_dim + k) : 0.0f;
    }
    for (int e = tid; e < H * H; e += kThreads) {
        const int o = e / H, i = e - o * H;          // W2[o][i]
        const float w = __ldg(params + g.w2 + e);
        sm[n.w2t + i * H + o] = w;
        if (with_w2) sm[n.w2 + e] = w;
    }
    for (int e = tid; e < H; e += kThreads) {
        sm[n.b1 + e] = __ldg(params + g.b1 + e);
        sm[n.b2 + e] = __ldg(params + g.b2 + e);
    }
    for (int e = tid; e < out_dim * H; e += kThreads) {
        const int a = e / H, k = e - a * H;
        sm[n.w3 + a * LDW3 + k] = __ldg(params + g.w3 + e);
    }
    for (int e = tid; e < out_dim; e += kThreads) {
        sm[n.b3 + e] = __ldg(params + g.b3 + e);
        if (with_ls) sm[n.ls + e] = __ldg(params + g.ls + e);
    }
}

// Load up to 128 rows of `width` floats (gathered through perm when given) into a padded tile;
// rows >= nrows and columns in [width, ld) are zero.
__device__ void load_rows(float* tile, int ld, int kpad, const float* __restrict__ src, int width,
                          const int32_t* __restrict__ perm, int64_t pos0, int nrows) {
    const int tid = threadIdx.x;
    for (int e = tid; e < kRows * kpad; e += kThreads) {
        const int r = e / kpad, k = e - r * kpad;
        float v = 0.0f;
        if (r < nrows && k < width) {
            const int64_t row = perm ? (int64_t)perm[pos0 + r] : (pos0 + r);
            v = __ldg(src + row * width + k);
        }
        tile[r * ld + k] = v;
    }
}

// ---- 128 x 64 dense layer: OUT = epi(b + IN[128 x K] * Wk[K x 64]) ---------------------------
// Thread (rg = tid>>4, cg = tid&15) owns rows {rg + 16 j, j<8} and columns {4 cg .. 4 cg + 3}.
// EPI 0: act(.) -> OUT;  EPI 1: acc * act'(OUT) -> OUT (in-place derivative form, bias unused).
// relu: activation is max(x, 0) instead of tanh (the reference's Net default, common.py MLP); its derivative in
// terms of the stored output h is (h > 0), exactly torch's (z > 0).
template <int EPI>
__device__ __forceinline__ void dense_128x64(const float* __restrict__ IN, int ldin, int K,
                                             const float* __restrict__ Wk,
                                             const float* __restrict__ bias, float* OUT, int ldout, bool relu) {
    const int tid = threadIdx.x;
    const int rg = tid >> 4, cg = tid & 15;
    float acc[8][4];
    float4 bv = make_float4(0.f, 0.f, 0.f, 0.f);
    if (EPI == 0) bv = *reinterpret_cast<const float4*>(bias + 4 * cg);
#pragma unroll
    for (int j = 0; j < 8; ++j) { acc[j][0] = bv.x; acc[j][1] = bv.y; acc[j][2] = bv.z; acc[j][3] = bv.w; }
    for (int k0 = 0; k0 < K; k0 += 4) {
        const float4 w0 = *reinterpret_cast<const float4*>(Wk + (k0 + 0) * H + 4 * cg);
        const float4 w1 = *reinterpret_cast<const float4*>(Wk + (k0 + 1) * H + 4 * cg);
        const float4 w2 = *reinterpret_cast<const float4*>(Wk + (k0 + 2) * H + 4 * cg);
        const float4 w3 = *reinterpret_cast<const float4*>(Wk + (k0 + 3) * H + 4 * cg);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float4 x = *reinterpret_cast<const float4*>(IN + (rg + 16 * j) * ldin + k0);
            acc[j][0] = fmaf(x.x, w0.x, acc[j][0]); acc[j][1] = fmaf(x.x, w0.y, acc[j][1]);
            acc[j][2] = fmaf(x.x, w0.z, acc[j][2]); acc[j][3] = fmaf(x.x, w0.w, acc[j][3]);
            acc[j][0] = fmaf(x.y, w1.x, acc[j][0]); acc[j][1] = fmaf(x.y, w1.y, acc[j][1]);
            acc[j][2] = fmaf(x.y, w1.z, acc[j][2]); acc[j][3] = fmaf(x.y, w1.w, acc[j][3]);
            acc[j][0] = fmaf(x.z, w2.x, acc[j][0]); acc[j][1] = fmaf(x.z, w2.y, acc[j][1]);
            acc[j][2] = fmaf(x.z, w2.z, acc[j][2]); acc[j][3] = fmaf(x.z, w2.w, acc[j][3]);
            acc[j][0] = fmaf(x.w, w3.x, acc[j][0]); acc[j][1] = fmaf(x.w, w3.y, acc[j][1]);
            acc[j][2] = fmaf(x.w, w3.z, acc[j][2]); acc[j][3] = fmaf(x.w, w3.w, acc[j][3]);
        }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        float* o = OUT + (rg + 16 * j) * ldout + 4 * cg;
        float4 r;
        if (EPI == 0) {
            r = relu ? make_float4(fmaxf(acc[j][0], 0.f), fmaxf(acc[j][1], 0.f), fmaxf(acc[j][2], 0.f), fmaxf(acc[j][3], 0.f))
                     : make_float4(tanhf(acc[j][0]), tanhf(acc[j][1]), tanhf(acc[j][2]), tanhf(acc[j][3]));
        } else {
            const float4 h = *reinterpret_cast<const float4*>(o);
            r = relu ? make_float4(h.x > 0.f ? acc[j][0] : 0.f, h.y > 0.f ? acc[j][1] : 0.f,
                                   h.z > 0.f ? acc[j][2] : 0.f, h.w > 0.f ? acc[j][3] : 0.f)
                     : make_float4(acc[j][0] * (1.0f - h.x * h.x), acc[j][1] * (1.0f - h.y * h.y),
                                   acc[j][2] * (1.0f - h.z * h.z), acc[j][3] * (1.0f - h.w * h.w));
        }
        *reinterpret_cast<float4*>(o) = r;
    }
}

// trunk forward: X -> H1 -> H2 (ends with a barrier)
__device__ void trunk_forward(float* sm, const Layout& L, const NetOff& n, bool relu) {
    dense_128x64<0>(sm + L.X, L.LDX, L.KX, sm + n.w1t, sm + n.b1, sm + L.H1, LDH, relu);
    __syncthreads();
    dense_128x64<0>(sm + L.H1, LDH, H, sm + n.w2t, sm + n.b2, sm + L.H2, LDH, relu);
    __syncthreads();
}

// head: out[r][a] = b3[a] + H2[r][:] . W3[a][:]
__device__ __forceinline__ float head_dot(const float* sm, const Layout& L, const NetOff& n, int r, int a) {
    const float* h = sm + L.H2 + r * LDH;
    const float* w = sm + n.w3 + a * LDW3;
    float acc = 0.0f;
#pragma unroll
    for (int k = 0; k < H; k += 4) {
        const float4 hv = *reinterpret_cast<const float4*>(h + k);
        const float4 wv = *reinterpret_cast<const float4*>(w + k);
        acc = fmaf(hv.x, wv.x, acc); acc = fmaf(hv.y, wv.y, acc);
        acc = fmaf(hv.z, wv.z, acc); acc = fmaf(hv.w, wv.w, acc);
    }
    return acc + sm[n.b3 + a];
}

__device__ __forceinline__ NetGlobal actor_global(const ts_actor_critic_desc& d) {
    return NetGlobal{d.a_w1, d.a_b1, d.a_w2, d.a_b2, d.a_w3, d.a_b3, d.a_logstd};
}
__device__ __forceinline__ NetGlobal critic_global(const ts_actor_critic_desc& d) {
    return NetGlobal{d.c_w1, d.c_b1, d.c_w2, d.c_b2, d.c_w3, d.c_b3, 0};
}

// ---- kernels --------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads, 1) critic_forward_kernel(
    const float* __restrict__ params, const ts_actor_critic_desc d, const float* __restrict__ obs0,
    float* __restrict__ out0, const float* __restrict__ obs1, float* __restrict__ out1, int64_t n) {
    extern __shared__ __align__(16) float sm[];
    const Layout L = make_layout(d.obs_dim, d.act_dim, 0);
    stage_net(sm, L.critic, params, critic_global(d), d.obs_dim, L.KX, 1, false, false);
    const int64_t tiles_per = (n + kRows - 1) / kRows;
    const int64_t tiles = tiles_per * (obs1 ? 2 : 1);
    for (int64_t t = blockIdx.x; t < tiles; t += gridDim.x) {
        const bool second = t >= tiles_per;
        const int64_t row0 = (second ? t - tiles_per : t) * kRows;
        const int nrows = (int)tsb::imin((int64_t)kRows, n - row0);
        __syncthreads();
        load_rows(sm + L.X, L.LDX, L.KX, second ? obs1 : obs0, d.obs_dim, nullptr, row0, nrows);
        __syncthreads();
        trunk_forward(sm, L, L.critic, (d.flags & TS_AC_RELU) != 0);
        if (threadIdx.x < nrows)
            (second ? out1 : out0)[row0 + threadIdx.x] = head_dot(sm, L, L.critic, threadIdx.x, 0);
    }
}

__global__ void __launch_bounds__(kThreads, 1) actor_logp_kernel(
    const float* __restrict__ params, const ts_actor_critic_desc d, const float* __restrict__ obs,
    const float* __restrict__ act, int64_t n, float* __restrict__ logp_out, float* __restrict__ mu_out) {
    extern __shared__ __align__(16) float sm[];
    const Layout L = make_layout(d.obs_dim, d.act_dim, 1);
    const int A = d.act_dim;
    const bool categorical = (d.flags & TS_AC_CATEGORICAL) != 0, relu = (d.flags & TS_AC_RELU) != 0;
    const int act_w = categorical ? 1 : A;     // discrete actions are ONE index per row (stored as float)
    stage_net(sm, L.actor, params, actor_global(d), d.obs_dim, L.KX, A, false, !categorical);
    const int64_t tiles = (n + kRows - 1) / kRows;
    for (int64_t t = blockIdx.x; t < tiles; t += gridDim.x) {
        const int64_t row0 = t * kRows;
        const int nrows = (int)tsb::imin((int64_t)kRows, n - row0);
        __syncthreads();
        load_rows(sm + L.X, L.LDX, L.KX, obs, d.obs_dim, nullptr, row0, nrows);
        load_rows(sm + L.ACT, kMaxAct, act_w, act, act_w, nullptr, row0, nrows);
        __syncthreads();
        trunk_forward(sm, L, L.actor, relu);
        // mu -> DOUT-less: reuse X tile region? keep it simple: each (r,a) pair writes mu to H1
        for (int o = threadIdx.x; o < kRows * A; o += kThreads) {
            const int r = o / A, a = o - r * A;
            sm[L.H1 + r * LDH + a] = head_dot(sm, L, L.actor, r, a);
        }
        __syncthreads();
        if (threadIdx.x < nrows && categorical) {
            const int r = threadIdx.x;
            float z[kMaxAct];
            for (int a = 0; a < A; ++a) z[a] = sm[L.H1 + r * LDH + a];
            ppo::CatT<kMaxAct> c;
            float lp, ent;
            ppo::cat_forward(z, A, (int)sm[L.ACT + r * kMaxAct], c, lp, ent);
            if (mu_out) for (int a = 0; a < A; ++a) mu_out[(row0 + r) * A + a] = c.p[a];   // the actor's output: probabilities
            logp_out[row0 + r] = lp;
        } else if (threadIdx.x < nrows) {
            const int r = threadIdx.x;
            float lp = 0.0f;
            for (int a = 0; a < A; ++a) {
                const float sigma = expf(sm[L.actor.ls + a]);
                const float mu = sm[L.H1 + r * LDH + a];
                lp += ppo::normal_logp_term(sm[L.ACT + r * kMaxAct + a], mu, sigma);
                if (mu_out) mu_out[(row0 + r) * A + a] = mu;
            }
            logp_out[row0 + r] = lp;
        }
    }
}

// column sums / outer products over the 128 rows of the tile, added to the flat gradient -----
// gW3[a][k] += sum_r DOUT[r][a] * H2[r][k];  gb3[a] += sum_r DOUT[r][a]
__device__ void head_backward(const float* sm, const Layout& L, int out_dim, float* __restrict__ grad,
                              int64_t g_w3, int64_t g_b3) {
    for (int o = threadIdx.x; o < out_dim * H; o += kThreads) {
        const int a = o / H, k = o - a * H;
        float acc = 0.0f, accb = 0.0f;
#pragma unroll 4
        for (int r = 0; r < kRows; ++r) {
            const float dv = sm[L.DOUT + r * LDO + a];
            acc = fmaf(dv, sm[L.H2 + r * LDH + k], acc);
            accb += dv;
        }
        atomicAdd(grad + g_w3 + o, acc);
        if (k == 0) atomicAdd(grad + g_b3 + a, accb);
    }
}
// H2 <- (DOUT * W3) * (1 - H2^2)     (dz2, in place)
__device__ void head_input_grad(float* sm, const Layout& L, const NetOff& n, int out_dim, bool relu) {
    const int tid = threadIdx.x, rg = tid >> 4, cg = tid & 15;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int r = rg + 16 * j;
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int a = 0; a < out_dim; ++a) {
            const float dv = sm[L.DOUT + r * LDO + a];
            const float4 w = *reinterpret_cast<const float4*>(sm + n.w3 + a * LDW3 + 4 * cg);
            acc.x = fmaf(dv, w.x, acc.x); acc.y = fmaf(dv, w.y, acc.y);
            acc.z = fmaf(dv, w.z, acc.z); acc.w = fmaf(dv, w.w, acc.w);
        }
        float* hp = sm + L.H2 + r * LDH + 4 * cg;
        const float4 h = *reinterpret_cast<const float4*>(hp);
        *reinterpret_cast<float4*>(hp) =
            relu ? make_float4(h.x > 0.f ? acc.x : 0.f, h.y > 0.f ? acc.y : 0.f, h.z > 0.f ? acc.z : 0.f, h.w > 0.f ? acc.w : 0.f)
                 : make_float4(acc.x * (1.f - h.x * h.x), acc.y * (1.f - h.y * h.y),
                               acc.z * (1.f - h.z * h.z), acc.w * (1.f - h.w * h.w));
    }
}
// gW[o][i] += sum_r DZ[r][o] * IN[r][i]  (64 x 64), gb[o] += sum_r DZ[r][o]
__device__ void weight_grad_64x64(const float* __restrict__ DZ, const float* __restrict__ IN,
                                  float* __restrict__ grad, int64_t g_w, int64_t g_b) {
    const int tid = threadIdx.x, og = tid >> 4, ig = tid & 15;
    float acc[4][4];
    float accb[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) acc[a][b] = 0.0f;
#pragma unroll 2
    for (int r = 0; r < kRows; ++r) {
        const float4 dz = *reinterpret_cast<const float4*>(DZ + r * LDH + 4 * og);
        const float4 x = *reinterpret_cast<const float4*>(IN + r * LDH + 4 * ig);
        const float dzv[4] = {dz.x, dz.y, dz.z, dz.w};
        const float xv[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
        for (int a = 0; a < 4; ++a) {
            accb[a] += dzv[a];
#pragma unroll
            for (int b = 0; b < 4; ++b) acc[a][b] = fmaf(dzv[a], xv[b], acc[a][b]);
        }
    }
#pragma unroll
    for (int a = 0; a < 4; ++a) {
#pragma unroll
        for (int b = 0; b < 4; ++b) atomicAdd(grad + g_w + (4 * og + a) * H + 4 * ig + b, acc[a][b]);
        if (ig == 0) atomicAdd(grad + g_b + 4 * og + a, accb[a]);
    }
}
// gW1[o][i] += sum_r DZ[r][o] * X[r][i]  (64 x obs), gb1[o] += sum_r DZ[r][o]
__device__ void weight_grad_first(const float* __restrict__ DZ, const float* __restrict__ X, int ldx,
                                  int obs_dim, float* __restrict__ grad, int64_t g_w, int64_t g_b) {
    const int tid = threadIdx.x, o = tid >> 2, iq = tid & 3;
    float acc[kMaxObs / 4];
    float accb = 0.0f;
#pragma unroll
    for (int j = 0; j < kMaxObs / 4; ++j) acc[j] = 0.0f;
    const int nj = (obs_dim - iq + 3) / 4;  // i = iq + 4 j < obs_dim
    for (int r = 0; r < kRows; ++r) {
        const float dz = DZ[r * LDH + o];
        accb += dz;
#pragma unroll
        for (int j = 0; j < kMaxObs / 4; ++j)
            if (j < nj) acc[j] = fmaf(dz, X[r * ldx + iq + 4 * j], acc[j]);
    }
#pragma unroll
    for (int j = 0; j < kMaxObs / 4; ++j)
        if (j < nj) atomicAdd(grad + g_w + (int64_t)o * obs_dim + iq + 4 * j, acc[j]);
    if (iq == 0) atomicAdd(grad + g_b + o, accb);
}

// backward through one trunk given DOUT (head gradient) and H1/H2/X of the tile
__device__ void trunk_backward(float* sm, const Layout& L, const NetOff& n, const NetGlobal& g,
                               int out_dim, int obs_dim, float* __restrict__ grad, bool relu) {
    head_backward(sm, L, out_dim, grad, g.w3, g.b3);
    __syncthreads();
    head_input_grad(sm, L, n, out_dim, relu);                        // H2 := dz2
    __syncthreads();
    weight_grad_64x64(sm + L.H2, sm + L.H1, grad, g.w2, g.b2);       // reads H1, dz2
    __syncthreads();
    dense_128x64<1>(sm + L.H2, LDH, H, sm + n.w2, nullptr, sm + L.H1, LDH, relu);  // H1 := dz1
    __syncthreads();
    weight_grad_first(sm + L.H1, sm + L.X, L.LDX, obs_dim, grad, g.w1, g.b1);
    __syncthreads();
}

__device__ __forceinline__ float block_sum_128(float v, float* red) {
    // sum over threads 0..127 (warps 0..3); result valid in thread 0
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
    if ((threadIdx.x & 31) == 0 && threadIdx.x < 128) red[threadIdx.x >> 5] = v;
    __syncthreads();
    float s = 0.0f;
    if (threadIdx.x == 0) s = red[0] + red[1] + red[2] + red[3];
    __syncthreads();
    return s;
}

__global__ void __launch_bounds__(kThreads, 1) ppo_grad_kernel(
    const float* __restrict__ params, const ts_actor_critic_desc d, const ts_ppo_hparams hp,
    const float* __restrict__ obs, const float* __restrict__ act, const float* __restrict__ adv,
    const float* __restrict__ ret, const float* __restrict__ logp_old, const float* __restrict__ v_s,
    const int32_t* __restrict__ perm, int64_t lo, int64_t hi, int64_t global_rows,
    const float* __restrict__ adv_moments, float* __restrict__ partials) {
    extern __shared__ __align__(16) float sm[];
    const Layout L = make_layout(d.obs_dim, d.act_dim, 2);
    const int A = d.act_dim;
    const int tid = threadIdx.x;
    // this CTA's private partial-gradient row (folded later by clip_adam_kernel / grad_reduce_kernel)
    float* __restrict__ grad = partials + (size_t)blockIdx.x * (size_t)(d.n_params + TS_PPO_GRAD_EXTRA);
    for (int64_t i = tid; i < d.n_params + TS_PPO_GRAD_EXTRA; i += kThreads) grad[i] = 0.0f;
    const NetGlobal ga = actor_global(d), gc = critic_global(d);
    const bool categorical = (d.flags & TS_AC_CATEGORICAL) != 0, relu = (d.flags & TS_AC_RELU) != 0;
    const int act_w = categorical ? 1 : A;
    // A shared trunk (DiscreteActor / DiscreteCritic on one preprocess net) is expressed by ALIASED offsets
    // (c_w1 == a_w1, ...): both backward passes add into the same gradient slots of this CTA's row.
    stage_net(sm, L.actor, params, ga, d.obs_dim, L.KX, A, true, !categorical);
    stage_net(sm, L.critic, params, gc, d.obs_dim, L.KX, 1, true, false);
    const ppo::Scalars sc = ppo::make_scalars(hp, global_rows, adv_moments);
    float* rowv = sm + L.ROWV;  // [0]=adv [1]=ret [2]=logp_old [3]=v_s, each kRows
    const int64_t B = hi - lo;
    const int64_t tiles = (B + kRows - 1) / kRows;
    for (int64_t t = blockIdx.x; t < tiles; t += gridDim.x) {
        const int64_t pos0 = lo + t * kRows;
        const int nrows = (int)tsb::imin((int64_t)kRows, hi - pos0);
        __syncthreads();
        load_rows(sm + L.X, L.LDX, L.KX, obs, d.obs_dim, perm, pos0, nrows);
        load_rows(sm + L.ACT, kMaxAct, act_w, act, act_w, perm, pos0, nrows);
        if (tid < kRows) {
            float a_ = 0.f, r_ = 0.f, l_ = 0.f, v_ = 0.f;
            if (tid < nrows) {
                const int64_t row = perm ? (int64_t)perm[pos0 + tid] : pos0 + tid;
                a_ = __ldg(adv + row); r_ = __ldg(ret + row); l_ = __ldg(logp_old + row); v_ = __ldg(v_s + row);
            }
            rowv[tid] = a_; rowv[kRows + tid] = r_; rowv[2 * kRows + tid] = l_; rowv[3 * kRows + tid] = v_;
        }
        __syncthreads();

        // ================= critic: forward, value loss, backward ===========================
        trunk_forward(sm, L, L.critic, relu);
        float vf_row = 0.0f;
        if (tid < kRows) {
            float dv = 0.0f;
            if (tid < nrows)
                ppo::critic_row(sc, head_dot(sm, L, L.critic, tid, 0), rowv[kRows + tid], rowv[3 * kRows + tid], vf_row, dv);
            sm[L.DOUT + tid * LDO] = dv;
        }
        __syncthreads();
        trunk_backward(sm, L, L.critic, gc, 1, d.obs_dim, grad, relu);

        // ================= actor: forward, clipped surrogate, backward =======================
        trunk_forward(sm, L, L.actor, relu);
        for (int o = tid; o < kRows * A; o += kThreads) {   // mu / logits into DOUT[r][a] (overwritten below)
            const int r = o / A, a = o - r * A;
            sm[L.DOUT + r * LDO + a] = head_dot(sm, L, L.actor, r, a);
        }
        __syncthreads();
        float clip_row = 0.0f, ent_row = 0.0f;
        if (tid < kRows && categorical) {
            const int r = tid;
            float z[kMaxAct], dz[kMaxAct];
            for (int a = 0; a < A; ++a) z[a] = sm[L.DOUT + r * LDO + a];
            const int action = (int)sm[L.ACT + r * kMaxAct];
            ppo::CatT<kMaxAct> c;
            float lp, ent;
            ppo::cat_forward(z, A, action, c, lp, ent);
            for (int a = 0; a < A; ++a) dz[a] = 0.0f;
            if (r < nrows) {
                float gl;
                ppo::actor_row(sc, lp, rowv[2 * kRows + r], rowv[r], clip_row, gl);
                ent_row = ent;
                ppo::cat_backward(c, A, action, gl, -sc.ent_coef * sc.inv_b, dz);
            }
            for (int a = 0; a < A; ++a) sm[L.DOUT + r * LDO + a] = dz[a];
        } else if (tid < kRows) {
            const int r = tid;
            float gl = 0.0f;     // d loss / d logp for this row
            float lp = 0.0f;
            float sig[kMaxAct], mu[kMaxAct];
#pragma unroll
            for (int a = 0; a < kMaxAct; ++a) {
                if (a < A) {
                    sig[a] = expf(sm[L.actor.ls + a]);
                    mu[a] = sm[L.DOUT + r * LDO + a];
                    lp += ppo::normal_logp_term(sm[L.ACT + r * kMaxAct + a], mu[a], sig[a]);
                }
            }
            if (r < nrows) ppo::actor_row(sc, lp, rowv[2 * kRows + r], rowv[r], clip_row, gl);
#pragma unroll
            for (int a = 0; a < kMaxAct; ++a) {
                if (a < A)
                    ppo::normal_backward(sm[L.ACT + r * kMaxAct + a], mu[a], sig[a], gl, sm[L.DOUT + r * LDO + a],
                                         sm[L.DOUT + r * LDO + 16 + a]);
            }
        }
        __syncthreads();
        // logstd gradient: column sums of DOUT[:, 16..16+A) plus the entropy term
        if (tid < A && !categorical) {
            float s = 0.0f;
            for (int r = 0; r < kRows; ++r) s += sm[L.DOUT + r * LDO + 16 + tid];
            s += -sc.ent_coef * sc.inv_b * (float)nrows;   // d(-ent_coef * mean(entropy))/d logstd
            atomicAdd(grad + d.a_logstd + tid, s);
        }
        trunk_backward(sm, L, L.actor, ga, A, d.obs_dim, grad, relu);

        // ================= loss sums ==========================================================
        const float s_clip = block_sum_128(tid < kRows ? clip_row : 0.0f, sm + L.RED);
        const float s_vf = block_sum_128(tid < kRows ? vf_row : 0.0f, sm + L.RED);
        const float s_ent = block_sum_128(tid < kRows ? ent_row : 0.0f, sm + L.RED);      // categorical: per-row entropies
        if (tid == 0) {
            float ent = 0.0f;   // Normal entropy summed over dims
            if (!categorical) for (int a = 0; a < A; ++a) ent += ppo::normal_entropy_term(expf(sm[L.actor.ls + a]));
            float* ex = grad + d.n_params;
            atomicAdd(ex + 0, s_clip);
            atomicAdd(ex + 1, s_vf);
            atomicAdd(ex + 2, categorical ? s_ent : ent * (float)nrows);
            atomicAdd(ex + 3, (float)nrows);
        }
    }
}

// ---- clip_grad_norm_ + Adam + stats + zero_grad : one CTA ------------------------------------
// Grid barrier / reduction state of clip_adam_kernel (self-resetting; launches are stream-ordered).
// One state block per launch SLOT (the caller's stream hashed into kAdamSlots): two models updating on different streams do
// not share barrier state, and every launch starts from a block the host zeroed on that stream (a trapped / aborted launch
// cannot poison the next one).  The launch is cooperative: every CTA of the (<= #SMs) grid is resident, so the spin is safe.
struct AdamCtl { unsigned int arrive, depart; double ss; };
constexpr int kAdamSlots = 64;
__device__ AdamCtl g_adam_ctl[kAdamSlots];

// gradient fold + clip_grad_norm_ + Adam in one launch.  CTA = 256 parameters x 4 partial groups
// (1024 threads), ~44 co-resident CTAs: (0) thread (e, q) folds the partial rows p = q (mod 4) of
// its parameter (coalesced across e, L2 resident), the 4 groups are combined through shared memory
// in a fixed order; (1) block sum of squares -> one f64 atomic per CTA; (2) grid barrier; (3) norm,
// clip coefficient, Adam update of the CTA's 256 parameters.
constexpr int kAdamElems = 256, kAdamGroups = 4;
__global__ void __launch_bounds__(kAdamElems * kAdamGroups) clip_adam_kernel(
    float* __restrict__ params, float* __restrict__ grad, const float* __restrict__ partials, int n_partials,
    float* __restrict__ exp_avg, float* __restrict__ exp_avg_sq, int64_t* __restrict__ step_count,
    int64_t n_params, const ts_ppo_hparams hp, float* __restrict__ stats_row, int ctl_slot) {
    AdamCtl& ctl = g_adam_ctl[ctl_slot];
    __shared__ double s_red[8];
    __shared__ float s_part[kAdamGroups][kAdamElems];
    __shared__ float s_coef, s_norm;
    __shared__ optim::AdamBias s_bias;
    const int tid = threadIdx.x, e = tid & (kAdamElems - 1), q = tid >> 8;
    const int64_t step = *step_count + 1;
    const int64_t width = n_params + TS_PPO_GRAD_EXTRA;
    const int64_t i = (int64_t)blockIdx.x * kAdamElems + e;
    float g = 0.0f;
    if (partials) {
        float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        if (i < width) {
            int p = q;
            for (; p + 7 * kAdamGroups < n_partials; p += 8 * kAdamGroups) {
#pragma unroll
                for (int u = 0; u < 8; ++u) acc[u] += __ldcg(partials + (int64_t)(p + u * kAdamGroups) * width + i);
            }
            for (; p < n_partials; p += kAdamGroups) acc[0] += __ldcg(partials + (int64_t)p * width + i);
        }
        s_part[q][e] = ((acc[0] + acc[1]) + (acc[2] + acc[3])) + ((acc[4] + acc[5]) + (acc[6] + acc[7]));
        __syncthreads();
        if (q == 0) {
            g = (s_part[0][e] + s_part[1][e]) + (s_part[2][e] + s_part[3][e]);
            if (i >= n_params && i < width) grad[i] = g;   // loss sums, read by CTA 0 after the barrier
        }
    } else if (q == 0 && i < width) {
        g = __ldcg(grad + i);
    }
    double ss = (q == 0 && i < n_params) ? (double)g * (double)g : 0.0;
    if (tid < kAdamElems) {   // warps 0..7 hold the q == 0 threads
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) ss += tsb::shfl_xor_f64(ss, off);
        if ((tid & 31) == 0) s_red[tid >> 5] = ss;
    }
    __syncthreads();
    if (tid == 0) {
        double t = 0.0;
        for (int w = 0; w < kAdamElems / 32; ++w) t += s_red[w];
        atomicAdd(&ctl.ss, t);
        __threadfence();
        atomicAdd(&ctl.arrive, 1u);
        while (*((volatile unsigned int*)&ctl.arrive) < gridDim.x) {}
        __threadfence();
        const float total_norm = (float)sqrt(*((volatile double*)&ctl.ss));
        s_coef = hp.max_grad_norm > 0.0 ? optim::clip_coef((float)hp.max_grad_norm, total_norm) : 1.0f;
        s_norm = total_norm;
        if (hp.optimizer != TS_OPT_RMSPROP) s_bias = optim::adam_bias(hp.lr, hp.beta1, hp.beta2, step);   // RMSprop has no bias correction
    }
    __syncthreads();
    const float coef = s_coef, step_size = s_bias.step_size, bc2_sqrt = s_bias.bc2_sqrt;
    const float w1 = (float)(1.0 - hp.beta1), w2 = (float)(1.0 - hp.beta2);
    const float beta2 = (float)hp.beta2, adam_eps = (float)hp.adam_eps, wd = (float)hp.weight_decay;
    if (hp.optimizer == TS_OPT_RMSPROP) {
        if (q == 0 && i < n_params) {               // beta2 holds alpha
            float p = params[i], v = exp_avg_sq[i];
            optim::rmsprop_elem(g * coef, p, v, (float)hp.lr, beta2, w2, adam_eps, wd);
            exp_avg_sq[i] = v; params[i] = p;
        }
    } else if (q == 0 && i < n_params) {
        float p = params[i], m = exp_avg[i], v = exp_avg_sq[i];
        optim::adam_elem(g * coef, p, m, v, step_size, bc2_sqrt, beta2, w1, w2, adam_eps, wd);
        exp_avg[i] = m; exp_avg_sq[i] = v; params[i] = p;
    }
    if (tid == 0) {
        if (blockIdx.x == 0) {
            const float e0 = __ldcg(grad + n_params), e1 = __ldcg(grad + n_params + 1);
            const float e2 = __ldcg(grad + n_params + 2), e3 = __ldcg(grad + n_params + 3);
            if (stats_row) {
                ppo::loss_row(e0, e1, e2, e3 > 0.0f ? e3 : 1.0f, hp, stats_row);
                stats_row[4] = s_norm; stats_row[5] = e3; stats_row[6] = 0.0f; stats_row[7] = 0.0f;
            }
            *step_count = step;
        }
        (void)ctl.depart;      // the block is zeroed by the host (cudaMemsetAsync on the launch stream) before every launch
    }
}

__global__ void grad_reduce_kernel(const float* __restrict__ partials, int n_partials, int64_t width,
                                   float* __restrict__ grad) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= width) return;
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    int p = 0;
    for (; p + 8 <= n_partials; p += 8) {
#pragma unroll
        for (int u = 0; u < 8; ++u) acc[u] += __ldcg(partials + (int64_t)(p + u) * width + i);
    }
    for (; p < n_partials; ++p) acc[0] += __ldcg(partials + (int64_t)p * width + i);
    grad[i] = ((acc[0] + acc[1]) + (acc[2] + acc[3])) + ((acc[4] + acc[5]) + (acc[6] + acc[7]));
}

// (sum, sum of squares) in f64 of adv over the positions [lo, hi) (through perm when given), in a fixed summation order that
// depends on blockDim.x alone; the result is valid in thread 0
__device__ __forceinline__ void adv_block_sums(const float* __restrict__ adv, const int32_t* __restrict__ perm, int64_t lo, int64_t hi,
                                               double& x, double& y) {
    __shared__ double s1[32], s2[32];
    double a = 0.0, b = 0.0;
    for (int64_t p = lo + threadIdx.x; p < hi; p += blockDim.x) {
        const double v = adv[perm ? (int64_t)perm[p] : p];
        a += v; b += v * v;
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) { a += tsb::shfl_xor_f64(a, off); b += tsb::shfl_xor_f64(b, off); }
    if ((threadIdx.x & 31) == 0) { s1[threadIdx.x >> 5] = a; s2[threadIdx.x >> 5] = b; }
    __syncthreads();
    x = 0.0; y = 0.0;
    if (threadIdx.x == 0)
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) { x += s1[w]; y += s2[w]; }
}

// (mean, unbiased std) of n values from their (sum, sum of squares), as torch's adv.mean() / adv.std().  One row: std 0,
// where torch's adv.std() of a single element is NaN (see DESIGN.md section 4).
__device__ __forceinline__ void moments_from_sums(double x, double y, int64_t n, float* __restrict__ out) {
    const double mean = x / (double)n;
    double var = (y - x * mean) / (double)(n > 1 ? n - 1 : 1);
    if (var < 0.0) var = 0.0;
    out[0] = (float)mean; out[1] = (float)sqrt(var);
}

// mean / unbiased std of the advantages of EVERY minibatch of one pass (one CTA per minibatch, fixed
// summation order): out[2 m] = mean, out[2 m + 1] = std                       (ppo.py:181-183)
__global__ void __launch_bounds__(1024) epoch_adv_moments_kernel(const float* __restrict__ adv, const int32_t* __restrict__ perm,
                                                                 int64_t lo0, int64_t mb_size, int64_t end, int n_mb,
                                                                 float* __restrict__ out) {
    const int m = blockIdx.x;
    const int64_t lo = lo0 + (int64_t)m * mb_size, hi = m == n_mb - 1 ? end : lo + mb_size;
    double x, y;
    adv_block_sums(adv, perm, lo, hi, x, y);
    if (threadIdx.x == 0) moments_from_sums(x, y, hi - lo, out + 2 * m);
}

// multi-GPU variant: per-minibatch (sum, sum of squares) in f64 -> all-reduce on the host side -> finalize
__global__ void __launch_bounds__(1024) epoch_adv_sums_kernel(const float* __restrict__ adv, const int32_t* __restrict__ perm,
                                                              int64_t lo0, int64_t mb_size, int64_t end, int n_mb,
                                                              double* __restrict__ sums) {
    const int m = blockIdx.x;
    const int64_t lo = lo0 + (int64_t)m * mb_size, hi = m == n_mb - 1 ? end : lo + mb_size;
    double x, y;
    adv_block_sums(adv, perm, lo, hi, x, y);
    if (threadIdx.x == 0) { sums[2 * m] = x; sums[2 * m + 1] = y; }
}
__global__ void epoch_adv_finalize_kernel(const double* __restrict__ sums, int64_t lo0, int64_t mb_size, int64_t end, int n_mb,
                                          int world, float* __restrict__ out) {
    const int m = blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= n_mb) return;
    const int64_t lo = lo0 + (int64_t)m * mb_size, hi = m == n_mb - 1 ? end : lo + mb_size;
    moments_from_sums(sums[2 * m], sums[2 * m + 1], (hi - lo) * world, out + 2 * m);
}

// ---- keyed bijection of [0, n): balanced Feistel on an even number of bits + cycle walking ----
__device__ __forceinline__ uint32_t mix32(uint32_t x) {
    x ^= x >> 16; x *= 0x7feb352dU; x ^= x >> 15; x *= 0x846ca68bU; x ^= x >> 16;
    return x;
}
__global__ void permutation_kernel(uint64_t seed, int first_epoch, int n_epochs, int64_t n, int half_bits,
                                   int32_t* __restrict__ out) {
    const int64_t total = n * n_epochs;
    const uint32_t mask = (1u << half_bits) - 1u;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total;
         t += (int64_t)gridDim.x * blockDim.x) {
        const int ep = (int)(t / n);
        const int64_t i = t - (int64_t)ep * n;
        uint64_t k = seed + 0x9E3779B97F4A7C15ull * (uint64_t)(first_epoch + ep + 1);
        k ^= k >> 30; k *= 0xBF58476D1CE4E5B9ull; k ^= k >> 27; k *= 0x94D049BB133111EBull; k ^= k >> 31;
        const uint32_t k0 = (uint32_t)k, k1 = (uint32_t)(k >> 32);
        uint64_t x = (uint64_t)i;
        do {
            uint32_t l = (uint32_t)(x >> half_bits) & mask, r = (uint32_t)x & mask;
#pragma unroll
            for (int round = 0; round < 6; ++round) {
                const uint32_t f = mix32(r ^ (round & 1 ? k1 : k0) ^ (0x9E3779B9u * (uint32_t)(round + 1))) & mask;
                const uint32_t nl = r;
                r = l ^ f;
                l = nl;
            }
            x = ((uint64_t)l << half_bits) | r;
        } while ((int64_t)x >= n);
        out[t] = (int32_t)x;
    }
}

size_t smem_bytes(const ts_actor_critic_desc& d, int mode) {
    return (size_t)make_layout(d.obs_dim, d.act_dim, mode).total * sizeof(float);
}

int check_desc(const ts_actor_critic_desc* d, const char* fn) {
    TS_REQUIRE(d != nullptr, "%s: null desc", fn);
    TS_REQUIRE(d->hidden == H, "%s: hidden width %d unsupported (only %d)", fn, d->hidden, H);
    TS_REQUIRE(d->obs_dim >= 1 && d->obs_dim <= kMaxObs, "%s: obs_dim %d out of [1,%d]", fn, d->obs_dim, kMaxObs);
    TS_REQUIRE(d->act_dim >= 1 && d->act_dim <= kMaxAct, "%s: act_dim %d out of [1,%d]", fn, d->act_dim, kMaxAct);
    TS_REQUIRE((d->flags & ~(TS_AC_RELU | TS_AC_CATEGORICAL)) == 0, "%s: unknown desc flags 0x%x", fn, d->flags);
    TS_REQUIRE((d->flags & TS_AC_CATEGORICAL) || d->a_logstd >= 0, "%s: Gaussian head needs a_logstd", fn);
    return 0;
}

template <typename K>
int set_smem(K kernel, size_t bytes, const char* fn) {
    static thread_local size_t configured[tsb::kMaxDevices] = {};  // per kernel instantiation and device
    const int dev = tsb::device_ordinal();
    if (bytes > configured[dev]) {
        // the tile layout grows with obs_dim and act_dim: a shape past the per-block opt-in limit (227 KB on H100, e.g. the
        // training layout at obs 64 / act 16) is refused with its size instead of an opaque cudaErrorInvalidValue
        int optin = 0;
        TS_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
        TS_REQUIRE(bytes <= (size_t)optin, "%s: this network shape needs %zu bytes of shared memory per block, the device allows %d",
                   fn, bytes, optin);
        TS_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
        configured[dev] = bytes;
    }
    return 0;
}

}  // namespace

namespace tsb {  // tensor-core path (mlp_tc.cu)
bool tc_supported(const ts_actor_critic_desc& d);
int launch_ppo_grad_tc(const float* params, const ts_actor_critic_desc& d, const ts_ppo_hparams& hp, const float* obs,
                       const float* act, const float* adv, const float* ret, const float* logp_old, const float* v_s,
                       const int32_t* perm, int64_t lo, int64_t hi, int64_t global_rows, const float* adv_moments,
                       float* grad, cudaStream_t st);
int launch_forward_tc(int mode, const float* params, const ts_actor_critic_desc& d, const float* in0, float* out0,
                      const float* in1, float* out1, int64_t n, cudaStream_t st);
int launch_ppo_epoch_tc(float* params, const ts_actor_critic_desc& d, const ts_ppo_hparams& hp, const float* obs,
                        const float* act, const float* adv, const float* ret, const float* logp_old, const float* v_s,
                        const int32_t* perm, int64_t lo0, int64_t mb_size, int64_t end, int n_mb, const float* adv_moments,
                        float* partials, float* grad_scratch, float* exp_avg, float* exp_avg_sq, int64_t* step_count,
                        float* stats, void* weight_image, const PeerArgs& px, cudaStream_t st);
int64_t weight_image_bytes(const ts_actor_critic_desc& d);
static bool simt_forced() {
    static const bool f = [] { const char* e = getenv("TS_B200_FORCE_SIMT"); return e && e[0] == '1'; }();
    return f;
}
}  // namespace tsb

extern "C" int ts_critic_forward(const float* params, const ts_actor_critic_desc* desc,
                                 const float* obs0, float* v_out0, const float* obs1,
                                 float* v_out1, int64_t n, ts_stream_t stream) {
    if (check_desc(desc, "ts_critic_forward")) return 2;
    if (n == 0) return 0;
    TS_REQUIRE(params && obs0 && v_out0 && (!obs1 || v_out1), "ts_critic_forward: null pointer");
    if (tsb::tc_supported(*desc) && !tsb::simt_forced())
        return tsb::launch_forward_tc(0, params, *desc, obs0, v_out0, obs1, v_out1, n, tsb::as_stream(stream));
    const size_t smem = smem_bytes(*desc, 0);
    if (set_smem(critic_forward_kernel, smem, "ts_critic_forward")) return 1;
    const int64_t tiles = ((n + kRows - 1) / kRows) * (obs1 ? 2 : 1);
    const unsigned grid = (unsigned)tsb::imin((int64_t)tiles, tsb::num_sms());
    critic_forward_kernel<<<grid, kThreads, smem, tsb::as_stream(stream)>>>(params, *desc, obs0, v_out0, obs1, v_out1, n);
    return tsb::check_launch("ts_critic_forward");
}

extern "C" int ts_actor_logp(const float* params, const ts_actor_critic_desc* desc, const float* obs,
                             const float* act, int64_t n, float* logp_out, float* mu_out,
                             ts_stream_t stream) {
    if (check_desc(desc, "ts_actor_logp")) return 2;
    if (n == 0) return 0;
    TS_REQUIRE(params && obs && act && logp_out, "ts_actor_logp: null pointer");
    if (tsb::tc_supported(*desc) && !tsb::simt_forced())
        return tsb::launch_forward_tc(1, params, *desc, obs, logp_out, act, mu_out, n, tsb::as_stream(stream));
    const size_t smem = smem_bytes(*desc, 1);
    if (set_smem(actor_logp_kernel, smem, "ts_actor_logp")) return 1;
    const int64_t tiles = (n + kRows - 1) / kRows;
    const unsigned grid = (unsigned)tsb::imin((int64_t)tiles, tsb::num_sms());
    actor_logp_kernel<<<grid, kThreads, smem, tsb::as_stream(stream)>>>(params, *desc, obs, act, n, logp_out, mu_out);
    return tsb::check_launch("ts_actor_logp");
}

extern "C" int ts_ppo_grad(const float* params, const ts_actor_critic_desc* desc,
                           const ts_ppo_hparams* hp, const float* obs, const float* act,
                           const float* adv, const float* ret, const float* logp_old,
                           const float* v_s, const int32_t* perm, int64_t lo, int64_t hi,
                           int64_t global_rows, const float* adv_moments, float* partials,
                           int32_t* n_partials_out, ts_stream_t stream) {
    if (check_desc(desc, "ts_ppo_grad")) return 2;
    TS_REQUIRE(hp != nullptr, "ts_ppo_grad: null hparams");
    TS_REQUIRE(hi >= lo && global_rows > 0, "ts_ppo_grad: bad row range");
    if (n_partials_out) *n_partials_out = 0;
    if (hi == lo) return 0;
    TS_REQUIRE(params && obs && act && adv && ret && logp_old && v_s && partials && n_partials_out, "ts_ppo_grad: null pointer");
    {
        const int64_t tiles_ = (hi - lo + kRows - 1) / kRows;
        *n_partials_out = (int32_t)tsb::imin(tiles_, tsb::num_sms());
    }
    TS_REQUIRE(!hp->advantage_normalization || adv_moments, "ts_ppo_grad: advantage_normalization needs adv_moments");
    if (tsb::tc_supported(*desc) && !tsb::simt_forced())   // tensor-core path (mlp_tc.cu); SIMT covers obs_dim > 32
        return tsb::launch_ppo_grad_tc(params, *desc, *hp, obs, act, adv, ret, logp_old, v_s, perm, lo, hi,
                                       global_rows, adv_moments, partials, tsb::as_stream(stream));
    const size_t smem = smem_bytes(*desc, 2);
    if (set_smem(ppo_grad_kernel, smem, "ts_ppo_grad")) return 1;
    const int64_t tiles = (hi - lo + kRows - 1) / kRows;
    const unsigned grid = (unsigned)tsb::imin((int64_t)tiles, tsb::num_sms());
    ppo_grad_kernel<<<grid, kThreads, smem, tsb::as_stream(stream)>>>(params, *desc, *hp, obs, act, adv, ret, logp_old, v_s, perm, lo, hi, global_rows, adv_moments, partials);
    return tsb::check_launch("ts_ppo_grad");
}

extern "C" int ts_minibatch_adv_sums(const float* adv, const int32_t* perm, int64_t lo, int64_t hi,
                                     double* sums, ts_stream_t stream) {
    TS_REQUIRE(adv && sums, "ts_minibatch_adv_sums: null pointer");
    // one minibatch of the epoch kernel: the same fixed summation order as ts_epoch_adv_sums and the fused path's
    // epoch_adv_moments_kernel, so all three give bit-identical moments.  An empty range writes (0, 0).
    epoch_adv_sums_kernel<<<1, 1024, 0, tsb::as_stream(stream)>>>(adv, perm, lo, hi - lo, hi, 1, sums);
    return tsb::check_launch("ts_minibatch_adv_sums");
}

extern "C" int ts_adv_moments_finalize(const double* sums, int64_t global_rows, float* out,
                                       ts_stream_t stream) {
    TS_REQUIRE(sums && out && global_rows > 0, "ts_adv_moments_finalize: bad arguments");
    // one minibatch [0, global_rows) of one rank
    epoch_adv_finalize_kernel<<<1, 128, 0, tsb::as_stream(stream)>>>(sums, 0, global_rows, global_rows, 1, 1, out);
    return tsb::check_launch("ts_adv_moments_finalize");
}

extern "C" int32_t ts_ppo_partial_rows(void) { return tsb::num_sms(); }

extern "C" int64_t ts_ppo_weight_image_bytes(const ts_actor_critic_desc* desc) {
    return desc ? tsb::weight_image_bytes(*desc) : 0;
}

extern "C" int ts_grad_reduce(const float* partials, int32_t n_partials, const ts_actor_critic_desc* desc,
                              float* grad, ts_stream_t stream) {
    TS_REQUIRE(partials && desc && grad && n_partials >= 0, "ts_grad_reduce: bad arguments");
    const int64_t width = desc->n_params + TS_PPO_GRAD_EXTRA;
    grad_reduce_kernel<<<(unsigned)((width + 255) / 256), 256, 0, tsb::as_stream(stream)>>>(partials, n_partials, width, grad);
    return tsb::check_launch("ts_grad_reduce");
}

extern "C" int ts_clip_adam_step(float* params, float* grad, const float* partials, int32_t n_partials,
                                 float* exp_avg, float* exp_avg_sq, int64_t* step_count,
                                 const ts_actor_critic_desc* desc, const ts_ppo_hparams* hp, float* stats_row,
                                 ts_stream_t stream) {
    TS_REQUIRE(params && grad && exp_avg && exp_avg_sq && step_count && desc && hp, "ts_clip_adam_step: null pointer");
    const unsigned adam_ctas = (unsigned)((desc->n_params + TS_PPO_GRAD_EXTRA + kAdamElems - 1) / kAdamElems);
    TS_REQUIRE(adam_ctas <= (unsigned)tsb::num_sms(), "ts_clip_adam_step: parameter vector too large for the single-wave grid barrier");
    cudaStream_t st = tsb::as_stream(stream);
    const int slot = (int)((reinterpret_cast<uintptr_t>(st) >> 4) % (uintptr_t)kAdamSlots);
    void* ctl_ptr = nullptr;
    TS_CUDA(cudaGetSymbolAddress(&ctl_ptr, g_adam_ctl));
    TS_CUDA(cudaMemsetAsync(static_cast<AdamCtl*>(ctl_ptr) + slot, 0, sizeof(AdamCtl), st));
    int64_t n_params = desc->n_params;
    ts_ppo_hparams hpv = *hp;
    int slot_arg = slot;
    void* args[] = {&params, &grad, &partials, &n_partials, &exp_avg, &exp_avg_sq, &step_count, &n_params, &hpv, &stats_row, &slot_arg};
    TS_CUDA(cudaLaunchCooperativeKernel((const void*)clip_adam_kernel, dim3(adam_ctas), dim3(kAdamElems * kAdamGroups), args, 0, st));
    return tsb::check_launch("ts_clip_adam_step");
}

extern "C" int ts_make_permutation(uint64_t seed, int32_t first_epoch, int32_t n_epochs, int64_t n,
                                   int32_t* out, ts_stream_t stream) {
    if (n == 0 || n_epochs == 0) return 0;
    TS_REQUIRE(out && n > 0 && n < (1ll << 31) && n_epochs > 0, "ts_make_permutation: bad arguments");
    int bits = 1;
    while ((1ll << bits) < n) ++bits;
    const int half = (bits + 1) / 2 < 1 ? 1 : (bits + 1) / 2;
    const int64_t total = n * n_epochs;
    const unsigned grid = (unsigned)tsb::imin((int64_t)(total + 255) / 256, (int64_t)tsb::num_sms() * 8);
    permutation_kernel<<<grid, 256, 0, tsb::as_stream(stream)>>>(seed, first_epoch, n_epochs, n, half, out);
    return tsb::check_launch("ts_make_permutation");
}

extern "C" int ts_ppo_update(float* params, float* grad, float* partials, float* exp_avg, float* exp_avg_sq,
                             int64_t* step_count, const ts_actor_critic_desc* desc,
                             const ts_ppo_hparams* hp, const float* obs, const float* obs_next,
                             const float* act, const double* rew, const uint8_t* terminated,
                             const uint8_t* truncated, const uint8_t* extra_end, float* v_s,
                             float* returns, float* adv, const float* logp_old, float* v_next_tmp,
                             int64_t N, const int32_t* perm, int32_t repeat, const int64_t* bounds,
                             int32_t n_minibatch, int32_t recompute_adv, double gamma, double lam,
                             double* rms_state, double rms_eps, void* gae_ws, void* adv_tmp,
                             void* weight_image, float* stats, void* row_feed, ts_stream_t stream) {
    if (check_desc(desc, "ts_ppo_update")) return 2;
    TS_REQUIRE(hp && bounds && stats && partials && grad && repeat >= 0 && n_minibatch >= 0, "ts_ppo_update: bad arguments");
    TS_REQUIRE(!hp->advantage_normalization || adv_tmp, "ts_ppo_update: adv_tmp required");
    static const bool no_fuse = [] { const char* e = getenv("TS_B200_NO_FUSED_STEP"); return e && e[0] == '1'; }();
    const bool fused = tsb::tc_supported(*desc) && !tsb::simt_forced() && !no_fuse;
    double* adv_sums = static_cast<double*>(adv_tmp);
    float* adv_mom = adv_tmp ? reinterpret_cast<float*>(adv_sums + 2) : nullptr;
    float* epoch_mom = adv_tmp ? reinterpret_cast<float*>(static_cast<uint8_t*>(adv_tmp) + 32) : nullptr;
    // Batch.split minibatches are regular: [m * size, (m + 1) * size) with the remainder merged into the last one
    bool regular = n_minibatch > 0;
    const int64_t lo0 = n_minibatch > 0 ? bounds[0] : 0, mb_size = n_minibatch > 0 ? bounds[1] - bounds[0] : 0;
    for (int m = 0; m < n_minibatch && regular; ++m) {
        regular = bounds[2 * m] == lo0 + (int64_t)m * mb_size && bounds[2 * m + 1] > bounds[2 * m] &&
                  (m == n_minibatch - 1 || bounds[2 * m + 1] == lo0 + (int64_t)(m + 1) * mb_size);
    }
    for (int r = 0; r < repeat; ++r) {
        if (recompute_adv && r > 0) {    // ppo.py:174-178 -> a2c.py:115-153
            TS_REQUIRE(obs_next && rew && v_next_tmp && gae_ws, "ts_ppo_update: recompute needs obs_next/rew/scratch");
            if (int e = ts_critic_forward(params, desc, obs, v_s, obs_next, v_next_tmp, N, stream)) return e;
            if (int e = ts_gae(v_s, v_next_tmp, TS_F32, rew, terminated, truncated, extra_end, 1, N, gamma,
                               lam, rms_state, rms_eps, nullptr, adv, returns, TS_F32, gae_ws, stream)) return e;
        }
        const int32_t* pr = perm ? perm + (int64_t)r * N : nullptr;
        float* rows = stats + (int64_t)r * n_minibatch * TS_PPO_STATS_STRIDE;
        if (row_feed) {      // row r of `perm` arrives from a host permutation job: the recompute above did not need it
            if (int e = ts_host_perm_feed_wait_row(row_feed, r, stream)) return e;
        }
        if (fused && regular) {   // ONE persistent launch for all optimiser steps of this pass
            const int64_t end = bounds[2 * n_minibatch - 1];
            if (hp->advantage_normalization) {
                epoch_adv_moments_kernel<<<n_minibatch, 1024, 0, tsb::as_stream(stream)>>>(adv, pr, lo0, mb_size, end, n_minibatch, epoch_mom);
                if (int e = tsb::check_launch("ts_ppo_update(adv moments)")) return e;
            }
            if (int e = tsb::launch_ppo_epoch_tc(params, *desc, *hp, obs, act, adv, returns, logp_old, v_s, pr, lo0, mb_size, end,
                                                 n_minibatch, hp->advantage_normalization ? epoch_mom : nullptr, partials, grad,
                                                 exp_avg, exp_avg_sq, step_count, rows, weight_image, tsb::PeerArgs{}, tsb::as_stream(stream))) return e;
            continue;
        }
        for (int m = 0; m < n_minibatch; ++m) {
            const int64_t lo = bounds[2 * m], hi = bounds[2 * m + 1];
            if (hp->advantage_normalization) {
                if (int e = ts_minibatch_adv_sums(adv, pr, lo, hi, adv_sums, stream)) return e;
                if (int e = ts_adv_moments_finalize(adv_sums, hi - lo, adv_mom, stream)) return e;
            }
            float* row = rows + (int64_t)m * TS_PPO_STATS_STRIDE;
            if (fused) {   // irregular bounds: one launch per optimiser step
                if (int e = tsb::launch_ppo_epoch_tc(params, *desc, *hp, obs, act, adv, returns, logp_old, v_s, pr, lo, hi - lo, hi,
                                                     1, adv_mom, partials, grad, exp_avg, exp_avg_sq, step_count, row,
                                                     weight_image, tsb::PeerArgs{}, tsb::as_stream(stream))) return e;
                continue;
            }
            int32_t n_part = 0;
            if (int e = ts_ppo_grad(params, desc, hp, obs, act, adv, returns, logp_old, v_s, pr, lo, hi,
                                    hi - lo, adv_mom, partials, &n_part, stream)) return e;
            if (int e = ts_clip_adam_step(params, grad, partials, n_part, exp_avg, exp_avg_sq, step_count, desc, hp, row, stream)) return e;
        }
    }
    return 0;
}

extern "C" int ts_epoch_adv_sums(const float* adv, const int32_t* perm, int64_t lo0, int64_t mb_size, int64_t end,
                                 int32_t n_minibatch, double* sums, ts_stream_t stream) {
    TS_REQUIRE(adv && sums && n_minibatch > 0 && mb_size > 0, "ts_epoch_adv_sums: bad arguments");
    epoch_adv_sums_kernel<<<n_minibatch, 1024, 0, tsb::as_stream(stream)>>>(adv, perm, lo0, mb_size, end, n_minibatch, sums);
    return tsb::check_launch("ts_epoch_adv_sums");
}

extern "C" int ts_epoch_adv_finalize(const double* sums, int64_t lo0, int64_t mb_size, int64_t end, int32_t n_minibatch,
                                     int32_t world, float* out, ts_stream_t stream) {
    TS_REQUIRE(sums && out && n_minibatch > 0 && world >= 1, "ts_epoch_adv_finalize: bad arguments");
    epoch_adv_finalize_kernel<<<(n_minibatch + 127) / 128, 128, 0, tsb::as_stream(stream)>>>(sums, lo0, mb_size, end, n_minibatch, world, out);
    return tsb::check_launch("ts_epoch_adv_finalize");
}

extern "C" int ts_ppo_epoch_multi(float* params, float* grad, float* partials, float* exp_avg, float* exp_avg_sq,
                                  int64_t* step_count, const ts_actor_critic_desc* desc, const ts_ppo_hparams* hp,
                                  const float* obs, const float* act, const float* adv, const float* returns,
                                  const float* logp_old, const float* v_s, const int32_t* perm, int64_t lo0,
                                  int64_t mb_size, int64_t end, int32_t n_minibatch, const float* adv_moments,
                                  void* weight_image, float* stats, int32_t rank, int32_t world,
                                  void* const* peer_buffers, ts_stream_t stream) {
    if (check_desc(desc, "ts_ppo_epoch_multi")) return 2;
    TS_REQUIRE(hp && params && grad && partials && stats && n_minibatch > 0 && mb_size > 0 && end > lo0 + (int64_t)(n_minibatch - 1) * mb_size,
               "ts_ppo_epoch_multi: bad arguments");
    TS_REQUIRE(tsb::tc_supported(*desc) && !tsb::simt_forced(), "ts_ppo_epoch_multi: network shape not covered by the tensor-core kernels");
    TS_REQUIRE(world >= 1 && world <= tsb::kMaxPeers && rank >= 0 && rank < world, "ts_ppo_epoch_multi: bad rank / world");
    TS_REQUIRE(!hp->advantage_normalization || adv_moments, "ts_ppo_epoch_multi: advantage normalisation needs the global per-minibatch moments");
    tsb::PeerArgs px;
    px.rank = rank; px.world = world;
    if (world > 1) {
        TS_REQUIRE(peer_buffers, "ts_ppo_epoch_multi: peer_buffers required for world > 1");
        for (int r = 0; r < world; ++r) {
            TS_REQUIRE(peer_buffers[r], "ts_ppo_epoch_multi: null peer buffer");
            px.recv[r] = reinterpret_cast<unsigned long long*>(static_cast<uint8_t*>(peer_buffers[r]) + tsb::kPeerHeaderBytes);
        }
        px.hdr = static_cast<unsigned int*>(peer_buffers[rank]);
    }
    return tsb::launch_ppo_epoch_tc(params, *desc, *hp, obs, act, adv, returns, logp_old, v_s, perm, lo0, mb_size, end, n_minibatch,
                                    adv_moments, partials, grad, exp_avg, exp_avg_sq, step_count, stats, weight_image, px,
                                    tsb::as_stream(stream));
}
