// Actor-critic MLP kernels on the Hopper tensor cores (wgmma), sm_90a.
//
// Same contract as the SIMT kernels in mlp.cu (ts_ppo_grad / ts_critic_forward / ts_actor_logp);
// reference code replaced: modelfree/ppo.py:157-161,179-211, modelfree/a2c.py:123-126,
// algorithm_base.py:497.
//
// Numerics: every GEMM is an fp32-faithful product built from bf16 tensor-core MMAs with fp32
// accumulation: each operand element x is stored as three bf16 pieces b0 + b1 + b2 = x (24
// significant bits) and the six partial products of weight >= 2^-16 are accumulated
// (wg::gemm_bf16x3).  A single-pass bf16/tf32 MMA would be 6x / 3x cheaper but is ~1e-3 off
// the reference's fp32 results, which breaks the 1e-5 parity bar on v_s / returns / advantages.
//
// Layout: one CTA = one tile of 128 transitions, 512 threads = four warpgroups.  Every operand
// matrix (activations X, H1, H2, gradients, weights) lives in shared memory in the blocked
// no-swizzle layout of wgmma.cuh (8-row x 16-byte core matrices), ONE copy per matrix: the same
// bytes are consumed K-major by the forward / input-gradient GEMMs and MN-major (reduction over
// the 128 rows) by the weight-gradient GEMMs.  Activations never leave the SM between forward and backward:
//   X -(W1)-> D1 -tanh-> H1 -(W2)-> D2 -tanh-> H2 -(W3)-> D3 -> loss -> dOut
//   dW3 = H2^T dOut ; dZ2 = (dOut W3) (1-H2^2) [overwrites H2] ; dW2 = dZ2^T H1 ; db2 = dZ2^T 1 ;
//   dH1 = dZ2 W2 ; dZ1 = dH1 (1-H1^2) [overwrites H1] ; dW1 = dZ1^T X ; db1 = dZ1^T 1
// Bias gradients come out of the tensor core too (B operand = a 128 x 8 block of ones).
// A 128 x 64 layer product is split over the warpgroups (warpgroup g: rows 64 (g & 1) .., columns
// 32 (g >> 1) ..); its register accumulator feeds the thread's epilogue (tanh, loss, bf16x3 split)
// directly, and h1 / h2 stay in the same registers for the backward pass.
#include <cuda_bf16.h>
#include <math.h>

#include <type_traits>

#include "common.cuh"
#include "optim_math.cuh"
#include "ppo_math.cuh"
#include "wgmma.cuh"

namespace {

constexpr int H = 64;
constexpr int kRows = 128;
constexpr int kThreads = 512;        // four warpgroups
constexpr int kCols = 16;            // accumulator elements of a 128 x 64 layer held by one thread (64 x 32 per warpgroup)
constexpr int kMaxAct = 16;
constexpr int NO = 16;            // padded head width (N of the head GEMM, columns of dOut)

// Optional phase timeline (DIAGNOSTICS build only, -DTS_B200_DIAGNOSTICS -> libts_b200_diag.so): when enabled, one CTA /
// thread 0 stores %globaltimer at each phase boundary; read back with ts_tc_timeline().  Compiled out of the product library.
#ifdef TS_B200_DIAGNOSTICS
__device__ unsigned long long g_tc_timeline[32];
__device__ int g_tc_timeline_on = 0;
__device__ int g_tc_timeline_gate = 1;      // written and read by CTA 0 / thread 0 only: which step is recorded
__device__ __forceinline__ void tstamp(int slot) {
    if (g_tc_timeline_on && (int)blockIdx.x == g_tc_timeline_on - 1 && threadIdx.x == 0 && g_tc_timeline_gate) {
        unsigned long long t;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
        g_tc_timeline[slot] = t;
    }
}
#else
__device__ __forceinline__ void tstamp(int) {}
#endif


// ---- bf16x3 operand matrices in shared memory --------------------------------------------------
struct Mat {
    uint32_t base;   // shared address of piece 0
    uint32_t part;   // bytes between pieces
    uint32_t RS;     // bytes between 8-row groups (= cols/8 * 128)
};
__host__ __device__ constexpr uint32_t mat_bytes(int rows, int cols) { return (uint32_t)rows * cols * 2u; }
// 8 consecutive columns (one 16-byte chunk) of row r
__device__ __forceinline__ void store_chunk8(uint8_t* sm0, const Mat& m, uint32_t r, uint32_t c0, const float* v) {
    uint32_t w0[4], w1[4], w2[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) wg::split3_pair(v[2 * j], v[2 * j + 1], w0[j], w1[j], w2[j]);
    uint8_t* p = sm0 + (m.base + wg::moff(r, c0, m.RS));
    *reinterpret_cast<uint4*>(p) = make_uint4(w0[0], w0[1], w0[2], w0[3]);
    *reinterpret_cast<uint4*>(p + m.part) = make_uint4(w1[0], w1[1], w1[2], w1[3]);
    *reinterpret_cast<uint4*>(p + 2 * m.part) = make_uint4(w2[0], w2[1], w2[2], w2[3]);
}

// Warpgroup index of the calling thread.  Broadcast from lane 0 so that the compiler knows it is warp-uniform: the tile
// origins and wgmma descriptors derived from it then live in uniform registers instead of being computed per thread
// (threadIdx.x counts as divergent), which is what keeps the 128-register kernels free of spills.
__device__ __forceinline__ int wg_index() { return __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 7), 0); }
// Layer tiles: warpgroup g computes rows [64 (g & 1), + 64) x columns [32 (g >> 1), + 32) of a 128 x 64 product;
// element e of the thread's accumulator is (lay_row0() + wg::frag_row(e), lay_col0() + wg::frag_col(e)).
__device__ __forceinline__ int lay_row0() { return 64 * (wg_index() & 1); }
__device__ __forceinline__ int lay_col0() { return 32 * (wg_index() >> 1); }

// the thread's 16 layer elements -> bf16x3 operand M (two consecutive columns per 32-bit store)
__device__ __forceinline__ void store_frag(uint8_t* sm0, const Mat& m, const float (&v)[kCols]) {
#pragma unroll
    for (int e = 0; e < kCols; e += 2) {
        uint32_t w0, w1, w2;
        wg::split3_pair(v[e], v[e + 1], w0, w1, w2);
        uint8_t* p = sm0 + (m.base + wg::moff((uint32_t)(lay_row0() + wg::frag_row(e)), (uint32_t)(lay_col0() + wg::frag_col(e)), m.RS));
        *reinterpret_cast<uint32_t*>(p) = w0;
        *reinterpret_cast<uint32_t*>(p + m.part) = w1;
        *reinterpret_cast<uint32_t*>(p + 2 * m.part) = w2;
    }
}
// inverse of store_frag, bit-exact: split3_pair truncates, so every piece is exact, b0 + b1 is x with its last 8 significant
// bits cleared (representable), and (b0 + b1) + b2 == x
__device__ __forceinline__ void load_frag(const uint8_t* sm0, const Mat& m, float (&v)[kCols]) {
#pragma unroll
    for (int e = 0; e < kCols; e += 2) {
        const uint8_t* p = sm0 + (m.base + wg::moff((uint32_t)(lay_row0() + wg::frag_row(e)), (uint32_t)(lay_col0() + wg::frag_col(e)), m.RS));
        const uint32_t w0 = *reinterpret_cast<const uint32_t*>(p);
        const uint32_t w1 = *reinterpret_cast<const uint32_t*>(p + m.part);
        const uint32_t w2 = *reinterpret_cast<const uint32_t*>(p + 2 * m.part);
        v[e] = (__uint_as_float(w0 << 16) + __uint_as_float(w1 << 16)) + __uint_as_float(w2 << 16);
        v[e + 1] = (__uint_as_float(w0 & 0xffff0000u) + __uint_as_float(w1 & 0xffff0000u)) + __uint_as_float(w2 & 0xffff0000u);
    }
}

// tanh(x) = 1 - 2 / (exp(2x) + 1) from two MUFU ops; absolute error ~1e-7 (the hidden activations
// feed 64-term dot products, so absolute -- not relative -- accuracy near 0 is what matters)
__device__ __forceinline__ float tanh_mufu(float x) {
    float e, r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x * 2.8853900817779268f));
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(e + 1.0f));
    return fmaf(-2.0f, r, 1.0f);
}

// D[64 x N] (the calling warpgroup's tile) = A * B with fp32-faithful bf16x3 MMAs, K = 16 * KSTEPS.  TA / TB = 1: the
// operand is used MN-major.  a_mn0 / b_mn0: first M / N index of the tile within A / B.  Runs to completion.
template <int N, int KSTEPS, int TA, int TB, bool FULL = true>
__device__ __forceinline__ void wg_gemm(float (&d)[N / 2], const Mat& A, uint32_t a_mn0, const Mat& B, uint32_t b_mn0) {
    const uint32_t a_lbo = TA ? A.RS : 128u, a_sbo = TA ? 128u : A.RS, a_step = TA ? 2u * A.RS : 256u;
    const uint32_t b_lbo = TB ? B.RS : 128u, b_sbo = TB ? 128u : B.RS, b_step = TB ? 2u * B.RS : 256u;
    wg::fence();
    wg::gemm_bf16x3<N, KSTEPS, TA, TB, FULL>(d, A.base + (a_mn0 >> 3) * a_sbo, A.part, a_lbo, a_sbo, a_step,
                                             B.base + (b_mn0 >> 3) * b_sbo, B.part, b_lbo, b_sbo, b_step, false);
    wg::commit();
    wg::wait<0>();
}
// weight-gradient GEMMs: three-product scheme unless TS_B200_WGRAD_FULL is defined at build time
#ifdef TS_B200_WGRAD_FULL
constexpr bool kWgradFull = true;
#else
constexpr bool kWgradFull = false;
#endif
// all threads: shared-memory operand writes become visible to the tensor core and to every thread
__device__ __forceinline__ void publish() {
    wg::fence_async_smem();
    __syncthreads();
}
struct Smem {   // byte offsets from the dynamic shared memory base (all multiples of 128)
    int KXP;
    Mat X, H1, H2, DO, W1, W2, W3;
    uint32_t w3f, b1, b2, b3, ls, dof, d3, rowv, red, act;
    uint32_t wblk, wblk_bytes;   // the "weight block" W1 | W2 | W3 | w3f | b1 | b2 | b3 | ls: one contiguous range, the unit
                                 // of the pre-split weight image in global memory (one bulk copy per network)
    uint32_t total;
};
// The kernels are instantiated per padded obs width KXP (16 or 32), so that inside them every offset below is an immediate.
__host__ __device__ constexpr int kxp_of(int obs_dim) { return (obs_dim + 15) & ~15; }
__host__ __device__ constexpr Smem make_smem(int kxp, uint32_t sbase) {
    Smem s{};
    s.KXP = kxp;
    uint32_t o = 0;
    auto mat = [&](Mat& m, int rows, int cols) {
        m.base = sbase + o; m.part = mat_bytes(rows, cols); m.RS = (uint32_t)(cols / 8) * 128u; o += 3u * m.part;
    };
    // X and H1 carry one extra 8-column chunk of ones (piece 0 = 1.0, pieces 1, 2 = 0): as the B operand of the
    // weight-gradient GEMMs it yields the bias gradient as 8 more accumulator columns instead of a GEMM of its own
    mat(s.X, kRows, s.KXP + 8);
    mat(s.H1, kRows, H + 8);
    mat(s.H2, kRows, H);
    mat(s.DO, kRows, NO);
    s.wblk = o;
    mat(s.W1, H, s.KXP);
    mat(s.W2, H, H);
    mat(s.W3, NO, H);
    s.w3f = o;  o += kMaxAct * H * 4;      // natural fp32 W3 [a][k] for the SIMT K=act GEMM
    s.b1 = o;   o += H * 4;
    s.b2 = o;   o += H * 4;
    s.b3 = o;   o += kMaxAct * 4;
    s.ls = o;   o += kMaxAct * 4;
    s.wblk_bytes = o - s.wblk;             // multiple of 128
    s.dof = o;  o += kRows * kMaxAct * 4;  // dOut in fp32 [a][r] (rows on consecutive banks)
    s.d3 = o;   o += kRows * NO * 4;       // head GEMM output (without bias) in fp32 [a][r]
    s.act = o;  o += kRows * kMaxAct * 4;  // actions of the tile
    s.rowv = o; o += 4 * kRows * 4;        // adv, ret, logp_old, v_s
    s.red = o;  o += 256 * 4;              // [0,12) per-warp sums, [64,80) 1/var, [80,96) log sigma + log sqrt(2 pi),
                                           // [128,256) per-warp column sums of (dmu, dlogstd)
    s.total = o;
    return s;
}

struct NetG { int64_t w1, b1, w2, b2, w3, b3, ls; };

// Stage a [rows x cols] fp32 matrix (row pointer by functor, cols padded with zeros up to ncols_pad)
// into a bf16x3 operand: one thread = one (row, 8-column chunk) -> 8 loads in flight, 3 STS.128, no
// integer division (chunks per row is a power of two).
template <class RowPtrF>
__device__ __forceinline__ void stage_chunks(uint8_t* sm0, const Mat& M, int rows, int cols, int cols_pad,
                                             RowPtrF&& rowptr) {
    const int nch = cols_pad >> 3;                 // 2, 4 or 8
    const int sh = nch == 8 ? 3 : (nch == 4 ? 2 : 1);
    for (int task = threadIdx.x; task < rows * nch; task += kThreads) {
        const int r = task >> sh, ch = task & (nch - 1);
        const float* src = rowptr(r);              // nullptr -> zero row
        float v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int k = 8 * ch + j;
            v[j] = (src != nullptr && k < cols) ? __ldg(src + k) : 0.0f;
        }
        store_chunk8(sm0, M, r, 8 * ch, v);
    }
}

// Split form of stage_chunks for matrices with at most one task per thread: issue the 8 loads of the
// thread's chunk now (chunk_load), convert + store later (chunk_store), so that the loads of several
// matrices are in flight together.
// COHERENT: read through L2 (ld.global.cg) -- required for the parameters, which other CTAs rewrite
// between the steps of the persistent epoch kernel (the read-only / L1 path could return stale lines).
template <bool COHERENT = false, class RowPtrF>
__device__ __forceinline__ void chunk_load(int rows, int cols, int cols_pad, RowPtrF&& rowptr, float (&v)[8]) {
    const int nch = cols_pad >> 3;
    const int sh = nch == 8 ? 3 : (nch == 4 ? 2 : 1);
    const int task = threadIdx.x;
    const int r = task >> sh, ch = task & (nch - 1);
    const float* src = task < rows * nch ? rowptr(r) : (const float*)nullptr;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int k = 8 * ch + j;
        v[j] = (src != nullptr && k < cols) ? (COHERENT ? __ldcg(src + k) : __ldg(src + k)) : 0.0f;
    }
}
__device__ __forceinline__ void chunk_store(uint8_t* sm0, const Mat& M, int rows, int cols_pad, const float (&v)[8]) {
    const int nch = cols_pad >> 3;
    const int sh = nch == 8 ? 3 : (nch == 4 ? 2 : 1);
    const int task = threadIdx.x;
    if (task < rows * nch) store_chunk8(sm0, M, task >> sh, 8 * (task & (nch - 1)), v);
}

// stage one network's weights: bf16x3 blocked copies for the tensor core + fp32 side copies
__device__ void stage_weights(uint8_t* sm, uint8_t* sm0, const Smem& S, const float* params, const NetG& g,
                              int obs_dim, int out_dim) {
    const int tid = threadIdx.x;
    float* w3f = reinterpret_cast<float*>(sm + S.w3f);
    {   // <= one chunk per thread and matrix (H = 64, KXP <= 32, 512 threads): all loads first
        float v1[8], v2[8], v3[8], vf[2];
        chunk_load<true>(H, obs_dim, S.KXP, [&](int o) { return params + g.w1 + (int64_t)o * obs_dim; }, v1);
        chunk_load<true>(H, H, H, [&](int o) { return params + g.w2 + (int64_t)o * H; }, v2);
        chunk_load<true>(NO, H, H, [&](int a) { return a < out_dim ? params + g.w3 + (int64_t)a * H : (const float*)nullptr; }, v3);
#pragma unroll
        for (int u = 0; u < 2; ++u) {
            const int e = tid + u * kThreads;
            vf[u] = (e >> 6) < out_dim ? __ldcg(params + g.w3 + e) : 0.0f;
        }
        chunk_store(sm0, S.W1, H, S.KXP, v1);
        chunk_store(sm0, S.W2, H, H, v2);
        chunk_store(sm0, S.W3, NO, H, v3);
        w3f[tid] = vf[0]; w3f[tid + kThreads] = vf[1];
    }
    float* b1 = reinterpret_cast<float*>(sm + S.b1);
    float* b2 = reinterpret_cast<float*>(sm + S.b2);
    float* b3 = reinterpret_cast<float*>(sm + S.b3);
    float* ls = reinterpret_cast<float*>(sm + S.ls);
    for (int e = tid; e < H; e += kThreads) { b1[e] = __ldcg(params + g.b1 + e); b2[e] = __ldcg(params + g.b2 + e); }
    if (tid < kMaxAct) {
        b3[tid] = tid < out_dim ? __ldcg(params + g.b3 + tid) : 0.0f;
        const float l = (tid < out_dim && g.ls >= 0) ? __ldcg(params + g.ls + tid) : 0.0f;
        ls[tid] = l;
        // per-dimension constants of the diagonal Gaussian, once per CTA instead of once per row
        float* gs = reinterpret_cast<float*>(sm + S.red) + 64;
        const float sigma = expf(l);
        gs[tid] = 1.0f / (sigma * sigma);
        gs[16 + tid] = logf(sigma) + 0.9189385332046727f;
    }
}

// ---- pre-split weight image --------------------------------------------------------------------------
// Global-memory copy of both networks' weight blocks in exactly the shared-memory layout (bf16x3 blocked
// operands + fp32 side copies; block 0 = critic, block 1 = actor), so that staging a network is ONE
// cp.async.bulk instead of ~13 k scattered loads + splits per CTA and step.  Built by
// weight_image_build_kernel; the Adam phase of the epoch kernel updates the entries of the parameters it
// rewrites.  Padding (columns >= obs_dim, head rows >= out_dim) is zero and never touched.
__device__ __forceinline__ void img_put(uint8_t* blk, uint32_t rel, uint32_t part, uint32_t RS, uint32_t r, uint32_t c, float x) {
    uint32_t w0, w1, w2;
    wg::split3_pair(x, 0.0f, w0, w1, w2);
    uint8_t* p = blk + rel + wg::moff(r, c, RS);
    *reinterpret_cast<uint16_t*>(p) = (uint16_t)w0;
    *reinterpret_cast<uint16_t*>(p + part) = (uint16_t)w1;
    *reinterpret_cast<uint16_t*>(p + 2 * part) = (uint16_t)w2;
}
__device__ __forceinline__ bool img_scatter_net(const Smem& S, uint32_t sbase, const NetG& g, int obs_dim, int out_dim,
                                                int64_t i, float x, uint8_t* blk) {
    const uint32_t w0 = sbase + S.wblk;       // Mat bases are shared addresses; the image uses block-relative offsets
    int64_t o;
    if ((o = i - g.w1) >= 0 && o < (int64_t)H * obs_dim) {
        const uint32_t r = (uint32_t)o / (uint32_t)obs_dim, c = (uint32_t)o - r * (uint32_t)obs_dim;
        img_put(blk, S.W1.base - w0, S.W1.part, S.W1.RS, r, c, x);
        return true;
    }
    if ((o = i - g.w2) >= 0 && o < H * H) { img_put(blk, S.W2.base - w0, S.W2.part, S.W2.RS, (uint32_t)o >> 6, (uint32_t)o & 63u, x); return true; }
    if ((o = i - g.w3) >= 0 && o < (int64_t)out_dim * H) {
        img_put(blk, S.W3.base - w0, S.W3.part, S.W3.RS, (uint32_t)o >> 6, (uint32_t)o & 63u, x);
        reinterpret_cast<float*>(blk + (S.w3f - S.wblk))[o] = x;
        return true;
    }
    if ((o = i - g.b1) >= 0 && o < H) { reinterpret_cast<float*>(blk + (S.b1 - S.wblk))[o] = x; return true; }
    if ((o = i - g.b2) >= 0 && o < H) { reinterpret_cast<float*>(blk + (S.b2 - S.wblk))[o] = x; return true; }
    if ((o = i - g.b3) >= 0 && o < out_dim) { reinterpret_cast<float*>(blk + (S.b3 - S.wblk))[o] = x; return true; }
    if (g.ls >= 0 && (o = i - g.ls) >= 0 && o < out_dim) { reinterpret_cast<float*>(blk + (S.ls - S.wblk))[o] = x; return true; }
    return false;
}
__device__ __forceinline__ void img_scatter(const ts_actor_critic_desc& d, const Smem& S, uint32_t sbase, int64_t i, float x,
                                            uint8_t* wimg) {
    const NetG gc{d.c_w1, d.c_b1, d.c_w2, d.c_b2, d.c_w3, d.c_b3, -1};
    if (img_scatter_net(S, sbase, gc, d.obs_dim, 1, i, x, wimg)) return;
    const NetG ga{d.a_w1, d.a_b1, d.a_w2, d.a_b2, d.a_w3, d.a_b3, d.a_logstd};
    img_scatter_net(S, sbase, ga, d.obs_dim, d.act_dim, i, x, wimg + S.wblk_bytes);
}
template <int KXP>
__global__ void weight_image_build_kernel(const float* __restrict__ params, const ts_actor_critic_desc d, uint8_t* __restrict__ wimg) {
    const Smem S = make_smem(KXP, 0u);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < d.n_params; i += (int64_t)gridDim.x * blockDim.x)
        img_scatter(d, S, 0u, i, params[i], wimg);
}

// acc := h = tanh(acc + bias) -> bf16x3 operand OUT (the backward pass reads h back from there: load_frag)
__device__ __forceinline__ void epi_tanh(uint8_t* sm0, const Mat& OUT, float (&acc)[kCols], const float* __restrict__ bias) {
#pragma unroll
    for (int e = 0; e < kCols; ++e) acc[e] = tanh_mufu(acc[e] + bias[lay_col0() + wg::frag_col(e)]);
    store_frag(sm0, OUT, acc);
}
// dZ2 = (dOut W3) * (1 - H2^2) for the thread's layer elements (K = out_dim is tiny: SIMT)
__device__ __forceinline__ void head_input_grad(uint8_t* sm, uint8_t* sm0, const Smem& S, int out_dim, float (&acc)[kCols]) {
    const int r0 = lay_row0() + wg::frag_row(0);        // rows r0 (elements 4 i, 4 i + 1) and r0 + 8 (4 i + 2, 4 i + 3)
    const float* dof = reinterpret_cast<const float*>(sm + S.dof);
    const float* w3f = reinterpret_cast<const float*>(sm + S.w3f) + lay_col0();
#pragma unroll
    for (int e = 0; e < kCols; ++e) acc[e] = 0.0f;
    for (int a = 0; a < out_dim; ++a) {
        const float d0 = dof[a * kRows + r0], d1 = dof[a * kRows + r0 + 8];
#pragma unroll
        for (int i = 0; i < kCols / 4; ++i) {
            const float2 w = *reinterpret_cast<const float2*>(w3f + a * H + wg::frag_col(4 * i));
            acc[4 * i] = fmaf(d0, w.x, acc[4 * i]); acc[4 * i + 1] = fmaf(d0, w.y, acc[4 * i + 1]);
            acc[4 * i + 2] = fmaf(d1, w.x, acc[4 * i + 2]); acc[4 * i + 3] = fmaf(d1, w.y, acc[4 * i + 3]);
        }
    }
    float h[kCols];
    load_frag(sm0, S.H2, h);
#pragma unroll
    for (int e = 0; e < kCols; ++e) acc[e] = acc[e] * fmaf(-h[e], h[e], 1.0f);
}
// write one row of dOut: fp32 side copy + bf16x3 operand (columns >= out_dim are zero)
__device__ __forceinline__ void write_dout_row(uint8_t* sm, uint8_t* sm0, const Smem& S, uint32_t r, const float* dv) {
    float* dof = reinterpret_cast<float*>(sm + S.dof) + r;
#pragma unroll
    for (int a = 0; a < kMaxAct; ++a) dof[a * kRows] = dv[a];
    store_chunk8(sm0, S.DO, r, 0, dv);
    store_chunk8(sm0, S.DO, r, 8, dv + 8);
}

// The partial row is private to the CTA: the first tile of a CTA stores, later tiles read-modify-write.
__device__ __forceinline__ void out_acc(float* p, float v, bool first) { *p = first ? v : *p + v; }

// Weight-gradient accumulators (M = 64: row o of the accumulator = output feature o) -> the CTA's partial gradient row.
// A thread owns scattered elements of an accumulator, so they are transposed through shared memory (the H2 operand is
// dead by then; padded leading dimensions keep the reads bank-conflict free) and written out with consecutive threads
// on consecutive addresses.
constexpr int kLdW2 = H + 1, kLdW1 = 33, kScrW2 = 0, kScrW1 = kScrW2 + H * kLdW2, kScrW3 = kScrW1 + H * kLdW1,
              kScrB1 = kScrW3 + NO * kLdW2, kScrB2 = kScrB1 + H, kScrEnd = kScrB2 + H;
static_assert(kScrEnd * 4 <= 3 * kRows * H * 2, "gradient scratch must fit in the H2 operand");
__device__ __forceinline__ float* grad_scratch(uint8_t* sm0, const Smem& S) { return reinterpret_cast<float*>(sm0 + S.H2.base); }

// [dW1 | db1] = dZ1^T [X | 1] (one warpgroup, N = KXP + 8 columns) -> scratch
template <int N>
__device__ __forceinline__ void wgrad_w1(uint8_t* sm0, const Smem& S) {
    float d[N / 2];
    wg_gemm<N, kRows / 16, 1, 1, kWgradFull>(d, S.H1, 0u, S.X, 0u);
    float* scr = grad_scratch(sm0, S);
#pragma unroll
    for (int e = 0; e < N / 2; ++e) {
        const int o = wg::frag_row(e), c = wg::frag_col(e);
        if (c < S.KXP) scr[kScrW1 + o * kLdW1 + c] = d[e];
        else if (c == S.KXP) scr[kScrB1 + o] = d[e];          // the ones column
    }
}

// PART 0: dW2, db2, dW3 (in scratch after the dW2 / dH1 stage: written out while the dW1 MMA runs); PART 1: dW1, db1.
template <int PART>
__device__ __forceinline__ void grad_out(uint8_t* sm0, const Smem& S, const NetG& g, int obs_dim, int out_dim,
                                         float* __restrict__ grad, bool first) {
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const float* scr = grad_scratch(sm0, S);
    if (PART == 0) {
#pragma unroll
        for (int u = 0; u < H * H / kThreads; ++u) {
            const int e = tid + u * kThreads;
            out_acc(grad + g.w2 + e, scr[kScrW2 + (e >> 6) * kLdW2 + (e & (H - 1))], first);
        }
        if (warp < out_dim) {
            out_acc(grad + g.w3 + warp * H + lane, scr[kScrW3 + warp * kLdW2 + lane], first);
            out_acc(grad + g.w3 + warp * H + 32 + lane, scr[kScrW3 + warp * kLdW2 + 32 + lane], first);
        }
        if (tid < H) out_acc(grad + g.b2 + tid, scr[kScrB2 + tid], first);
    } else {
        if (lane < obs_dim) {
#pragma unroll
            for (int r = warp; r < H; r += kThreads / 32)
                out_acc(grad + g.w1 + (int64_t)r * obs_dim + lane, scr[kScrW1 + r * kLdW1 + lane], first);
        }
        if (tid < H) out_acc(grad + g.b1 + tid, scr[kScrB1 + tid], first);
    }
}

// Sum 32 per-lane values over the warp with 31 shuffles; lane j returns the total of v[j].
__device__ __forceinline__ float warp_transpose_sum32(float (&v)[32]) {
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int n = 16; n >= 1; n >>= 1) {
        const bool upper = (lane & n) != 0;
#pragma unroll
        for (int i = 0; i < n; ++i) {
            const float send = upper ? v[i] : v[i + n];
            const float keep = upper ? v[i + n] : v[i];
            v[i] = keep + __shfl_xor_sync(0xffffffffu, send, n);
        }
    }
    return v[0];
}

// forward of one trunk: X -> H1 -> H2 -> head D3 (fp32 [a][r] in shared memory, without bias)
__device__ __forceinline__ void trunk_forward(uint8_t* sm, uint8_t* sm0, const Smem& S) {
    float acc[kCols];
    publish();
    if (S.KXP == 16) wg_gemm<2 * kCols, 1, 0, 0>(acc, S.X, lay_row0(), S.W1, lay_col0());
    else wg_gemm<2 * kCols, 2, 0, 0>(acc, S.X, lay_row0(), S.W1, lay_col0());
    epi_tanh(sm0, S.H1, acc, reinterpret_cast<const float*>(sm + S.b1));
    publish();
    wg_gemm<2 * kCols, H / 16, 0, 0>(acc, S.H1, lay_row0(), S.W2, lay_col0());
    epi_tanh(sm0, S.H2, acc, reinterpret_cast<const float*>(sm + S.b2));
    publish();
    float d3[4];                                          // head: warpgroup g -> rows 64 (g & 1) .., columns 8 (g >> 1) ..
    const int c0 = 8 * (wg_index() >> 1);
    wg_gemm<8, H / 16, 0, 0>(d3, S.H2, lay_row0(), S.W3, c0);
    float* out = reinterpret_cast<float*>(sm + S.d3);
#pragma unroll
    for (int e = 0; e < 4; ++e) out[(c0 + wg::frag_col(e)) * kRows + lay_row0() + wg::frag_row(e)] = d3[e];
    __syncthreads();
}

// backward of one trunk given dOut (S.DO / dof); writes all weight and bias gradients of the net.
// `weights_dead()` is called (all threads) once nothing reads the network's weight block any more.
template <class F>
__device__ __forceinline__ void trunk_backward(uint8_t* sm, uint8_t* sm0, const Smem& S, const NetG& g, int obs_dim, int out_dim,
                                               float* __restrict__ grad, bool first, F&& weights_dead) {
    const int wgi = wg_index();
    float* scr = grad_scratch(sm0, S);
    publish();                                                 // dOut (fp32 and operand) complete
    float dz2[kCols];
    head_input_grad(sm, sm0, S, out_dim, dz2);
    float dw3[NO / 2];
    if (wgi == 3) wg_gemm<NO, kRows / 16, 1, 1, kWgradFull>(dw3, S.H2, 0u, S.DO, 0u);        // dW3^T = H2^T dOut
    tstamp(16);
    __syncthreads();                                           // H2 is no longer read
    store_frag(sm0, S.H2, dz2);                                // H2 := dZ2
    tstamp(17);
    publish();
    float dw2[12], dh1[kCols];
    if (wgi < 3) wg_gemm<24, kRows / 16, 1, 1, kWgradFull>(dw2, S.H2, 0u, S.H1, 24u * wgi);  // [dW2 | db2] = dZ2^T [H1 | 1]
    wg_gemm<2 * kCols, H / 16, 0, 1>(dh1, S.H2, lay_row0(), S.W2, lay_col0());              // dH1 = dZ2 W2
    __syncthreads();                                           // H2 (now scratch), H1 and the weight block are no longer read
    tstamp(18);
    weights_dead();
    if (wgi < 3) {
#pragma unroll
        for (int e = 0; e < 12; ++e) {
            const int o = wg::frag_row(e), c = 24 * wgi + wg::frag_col(e);
            if (c < H) scr[kScrW2 + o * kLdW2 + c] = dw2[e];
            else if (c == H) scr[kScrB2 + o] = dw2[e];        // the ones column
        }
    } else {
#pragma unroll
        for (int e = 0; e < NO / 2; ++e) scr[kScrW3 + wg::frag_col(e) * kLdW2 + wg::frag_row(e)] = dw3[e];   // dW3^T [k][a] -> [a][k]
    }
    {
        float h1[kCols];
        load_frag(sm0, S.H1, h1);
#pragma unroll
        for (int e = 0; e < kCols; ++e) dh1[e] *= fmaf(-h1[e], h1[e], 1.0f);
    }
    store_frag(sm0, S.H1, dh1);                                // H1 := dZ1
    tstamp(19);
    publish();
    if (wgi == 0) {
        if (S.KXP == 16) wgrad_w1<24>(sm0, S);
        else wgrad_w1<40>(sm0, S);
    }
    grad_out<0>(sm0, S, g, obs_dim, out_dim, grad, first);    // dW2 / db2 / dW3 leave while warpgroup 0 runs the dW1 MMAs
    __syncthreads();
    tstamp(20);
    grad_out<1>(sm0, S, g, obs_dim, out_dim, grad, first);
}

// State of the in-kernel grid barriers of the fused epoch kernel (self-resetting; launches are
// stream-ordered and every CTA of the grid is resident: cooperative launch, 1 CTA / SM).
// They live in the 128-byte control block in front of the caller's weight image (one per model instance, so
// two models updating on different streams never share barrier state); without an image: this global block.
struct EpochCtl {
    unsigned int arrive, depart;
    double ss[2];
};
constexpr size_t kCtlBytes = 128;
__device__ EpochCtl g_ep_ctl = {0u, 0u, {0.0, 0.0}};

struct AdamArgs {     // optimiser half of the fused single-GPU path
    float* params_w;
    float* grad_scratch;   // n_params + TS_PPO_GRAD_EXTRA folded values (loss sums are read back from here)
    float* exp_avg;
    float* exp_avg_sq;
    int64_t* step_count;
    float* stats;          // one row of TS_PPO_STATS_STRIDE floats per minibatch (nullable)
};

struct GridBarrier {   // monotonic counter: the k-th use waits for k * gridDim.x arrivals
    unsigned int target;
    unsigned int* ctr;
    // Split phase.  arrive(): release at gpu scope (cumulative over the bar.sync) -- a release waits for the
    // calling thread's OUTSTANDING LOADS too, so prefetches that should fly across the barrier are issued
    // between arrive() and wait().
    __device__ __forceinline__ void arrive() {
        __syncthreads();
        if (threadIdx.x == 0) {
            target += gridDim.x;
            asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(ctr) : "memory");
        }
    }
    __device__ __forceinline__ void wait() {
        if (threadIdx.x == 0) {
            unsigned int seen;
            do {
                asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(seen) : "l"(ctr) : "memory");
            } while (seen < target);
        }
        __syncthreads();
    }
    __device__ __forceinline__ void sync() { arrive(); wait(); }
};

// Cross-GPU sum of one gradient element (fused all-reduce of the epoch kernel): the peers' (value, seq) packets of this
// step are polled CONCURRENTLY -- one load per missing peer and round, all in flight together -- so the wait is one NVLink
// latency, not world - 1 dependent ones; the sum runs in rank order (bit-identical on every rank).  Kept out of line: its
// register arrays must not weigh on the single-GPU path.
__device__ __noinline__ float peer_gather_sum(const unsigned long long* src0, int world, int rank, float g, unsigned int seq,
                                              size_t peer_stride) {
    float vals[tsb::kMaxPeers];
    unsigned int missing = ((1u << world) - 1u) & ~(1u << rank);
    unsigned long long t_start = 0ull;
    unsigned int spins = 0u;
    while (missing) {
        unsigned long long got[tsb::kMaxPeers];
#pragma unroll
        for (int r = 0; r < tsb::kMaxPeers; ++r) {
            if (missing & (1u << r))
                asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(got[r]) : "l"(src0 + (size_t)r * peer_stride) : "memory");
        }
#pragma unroll
        for (int r = 0; r < tsb::kMaxPeers; ++r) {
            if ((missing & (1u << r)) && (unsigned int)(got[r] >> 32) == seq) {
                vals[r] = __uint_as_float((unsigned int)got[r]);
                missing &= ~(1u << r);
            }
        }
        if (missing && (++spins & 0xffffu) == 0u) {      // a peer that never shows up must not hang the GPU
            unsigned long long now;
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
            if (t_start == 0ull) t_start = now;
            else if (now - t_start > 20000000000ull) __trap();
        }
    }
    float sum = 0.0f;
#pragma unroll
    for (int r = 0; r < tsb::kMaxPeers; ++r) {
        if (r < world) sum += (r == rank) ? g : vals[r];
    }
    return sum;
}

// one thread's share of a tile's gathers: an (8-column chunk) of X, and for row r = tid % 128, group q = tid / 128, the
// actions q + 4 u and row value q (adv, ret, logp_old, v_s) -- spread over all 512 threads, so that the prefetch that is
// held in registers across the grid barrier stays small
struct TileIn { float xv[8]; float av[kMaxAct / 4]; float rv; };

// The minibatches of one launch are [lo0 + m * mb_size, lo0 + (m + 1) * mb_size) for m < n_mb - 1 and
// [lo0 + (n_mb - 1) * mb_size, end) for the last one (Batch.split with merge_last, batch.py:1196-1215).
//
// EPOCH = false: n_mb = 1; write this CTA's partial gradient row and stop (multi-GPU: fold + all-reduce
// + ts_clip_adam_step follow).
// EPOCH = true: persistent over the n_mb optimiser steps of one pass over the rollout.  Per step: tile
// forward/backward -> grid barrier -> every CTA folds its slice of the gradient over the partial rows ->
// barrier (global sum of squares) -> clip + Adam on the slice -> barrier (parameters visible).  The gathers
// of the NEXT minibatch's tile are issued before the first barrier and land while the CTA waits.
template <bool EPOCH, int KXP>
__global__ void __launch_bounds__(kThreads, 1) ppo_tc_kernel(
    const float* params, const ts_actor_critic_desc d, const ts_ppo_hparams hp,
    const float* __restrict__ obs, const float* __restrict__ act, const float* __restrict__ adv,
    const float* __restrict__ ret, const float* __restrict__ logp_old, const float* __restrict__ v_s,
    const int32_t* __restrict__ perm, int64_t lo0, int64_t mb_size, int64_t end, int n_mb, int64_t global_rows,
    const float* __restrict__ adv_moments, float* __restrict__ partials, const AdamArgs opt, uint8_t* wimg /* nullable */,
    const __grid_constant__ tsb::PeerArgs px) {
    extern __shared__ __align__(1024) uint8_t sm[];
    __shared__ __align__(8) uint64_t s_wbar;
    __shared__ float s_coef, s_norm, s_step_size, s_bc2_sqrt;
    __shared__ int32_t s_row[kRows];
    __shared__ float s_part[4][128];      // actor loss epilogue: log-prob partials of the 4 action groups; optimiser half: fold partials
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int P = (int)gridDim.x;
    const int64_t width = d.n_params + TS_PPO_GRAD_EXTRA;
    // this CTA's private partial-gradient row: no cross-CTA atomics
    float* __restrict__ grad = partials + (size_t)blockIdx.x * (size_t)width;
    auto mb_lo = [&](int m) { return lo0 + (int64_t)m * mb_size; };
    auto mb_hi = [&](int m) { return m == n_mb - 1 ? end : lo0 + (int64_t)(m + 1) * mb_size; };
    auto mb_tiles = [&](int m) { return (mb_hi(m) - mb_lo(m) + kRows - 1) / kRows; };
    auto prefetch_rows = [&](int m, int64_t t) {   // dataset row of every tile row, ahead of its use
        if (tid < kRows) {
            const int64_t pos = mb_lo(m) + t * kRows + tid;
            s_row[tid] = pos < mb_hi(m) ? (perm ? __ldg(perm + pos) : (int32_t)pos) : 0;
        }
    };
    if ((int64_t)blockIdx.x < mb_tiles(0)) prefetch_rows(0, blockIdx.x);
    const uint32_t sbase = wg::smem_u32(sm);
    uint8_t* sm0 = sm - sbase;     // so that (sm0 + shared_address) is the generic pointer
    const Smem S = make_smem(KXP, sbase);
    const int A = d.act_dim;
    const NetG ga{d.a_w1, d.a_b1, d.a_w2, d.a_b2, d.a_w3, d.a_b3, d.a_logstd};
    const NetG gc{d.c_w1, d.c_b1, d.c_w2, d.c_b2, d.c_w3, d.c_b3, -1};
    const int64_t step0 = EPOCH ? *opt.step_count : 0;
    const unsigned int seq0 = (EPOCH && px.world > 1) ? *((volatile unsigned int*)px.hdr) : 0u;

    if (tid == 0) { wg::mbar_init(&s_wbar, 1); wg::fence_mbar_init(); }
    for (int e = tid; e < 2 * 3 * kRows; e += kThreads) {   // the ones chunks of X and H1 (bf16 1.0 = 0x3F80 in piece 0)
        const int r = e % kRows, pc = (e / kRows) % 3;
        const Mat& M = e < 3 * kRows ? S.X : S.H1;
        const uint32_t c = e < 3 * kRows ? (uint32_t)S.KXP : (uint32_t)H;
        const uint32_t w = pc == 0 ? 0x3F803F80u : 0u;
        *reinterpret_cast<uint4*>(sm0 + (M.base + pc * M.part + wg::moff((uint32_t)r, c, M.RS))) = make_uint4(w, w, w, w);
    }
    __syncthreads();
    EpochCtl* ctl = wimg != nullptr ? reinterpret_cast<EpochCtl*>(wimg - kCtlBytes) : &g_ep_ctl;
    GridBarrier gbar{0u, &ctl->arrive};
    // Weight staging.  With a weight image: one bulk copy (TMA engine) per network, issued as early as the
    // block is dead, completion on s_wbar.  Without: gather + split in the CTA (stage_weights).
    uint32_t wphase = 0u;
    bool critic_issued = false;
    auto issue_weights = [&](int net) {   // every earlier access to the weight block is ordered before this call
        if (wimg != nullptr && tid == 0) {
            wg::fence_proxy_async_all();
            wg::mbar_expect_tx(&s_wbar, S.wblk_bytes);
            wg::bulk_g2s(sbase + S.wblk, wimg + (size_t)net * S.wblk_bytes, S.wblk_bytes, &s_wbar);
        }
    };
    auto wait_weights = [&](const NetG& g, int out_dim) {
        if (wimg == nullptr) { stage_weights(sm, sm0, S, params, g, d.obs_dim, out_dim); return; }
        wg::mbar_wait(&s_wbar, wphase);
        wphase ^= 1u;
        if (g.ls >= 0 && tid < kMaxAct) {     // per-dimension constants of the diagonal Gaussian
            float* gs = reinterpret_cast<float*>(sm + S.red) + 64;
            const float sigma = expf(reinterpret_cast<const float*>(sm + S.ls)[tid]);
            gs[tid] = 1.0f / (sigma * sigma);
            gs[16 + tid] = logf(sigma) + 0.9189385332046727f;
        }
    };
    float* rowv = reinterpret_cast<float*>(sm + S.rowv);
    float* red = reinterpret_cast<float*>(sm + S.red);
    float* actt = reinterpret_cast<float*>(sm + S.act);

    // every gather of a tile in flight together (rows from s_row) ...
    auto load_inputs = [&](int nrows, TileIn& in) {
        chunk_load(kRows, d.obs_dim, S.KXP, [&](int r) {
            return r < nrows ? obs + (int64_t)s_row[r] * d.obs_dim : (const float*)nullptr;
        }, in.xv);
        const int r = tid & (kRows - 1), q = tid >> 7;
        const int64_t row = r < nrows ? (int64_t)s_row[r] : -1;
#pragma unroll
        for (int u = 0; u < kMaxAct / 4; ++u) {
            const int a = q + 4 * u;
            in.av[u] = (row >= 0 && a < A) ? __ldg(act + row * A + a) : 0.0f;
        }
        const float* rsrc = q == 0 ? adv : (q == 1 ? ret : (q == 2 ? logp_old : v_s));
        in.rv = row >= 0 ? __ldg(rsrc + row) : 0.0f;
    };
    // ... and their conversion into the tile's operands
    auto store_inputs = [&](const TileIn& in) {
        chunk_store(sm0, S.X, kRows, S.KXP, in.xv);
        const int r = tid & (kRows - 1), q = tid >> 7;
#pragma unroll
        for (int u = 0; u < kMaxAct / 4; ++u) actt[(q + 4 * u) * kRows + r] = in.av[u];      // [a][r]: rows on consecutive banks
        rowv[q * kRows + r] = in.rv;
    };

    double beta1_pow = 1.0, beta2_pow = 1.0;
    const bool rmsprop = hp.optimizer == TS_OPT_RMSPROP;       // block-uniform: RMSprop has no bias correction
    if (EPOCH && tid == 256 && !rmsprop) { beta1_pow = pow(hp.beta1, (double)step0); beta2_pow = pow(hp.beta2, (double)step0); }
    bool staged = false;        // the tile's inputs were already stored by the previous step's prefetch
    tstamp(0);
    for (int m = 0; m < n_mb; ++m) {
        const int64_t lo = mb_lo(m), hi = mb_hi(m);
        const int64_t tiles = (hi - lo + kRows - 1) / kRows;
        // the loss is the mean over the GLOBAL minibatch: every rank contributes hi - lo rows of its own shard
        // in shared memory rather than in 13 registers held across the tile: the loss epilogues read it from there (the first
        // read is behind trunk_forward's barriers; the previous minibatch's last read is behind the optimiser half's barriers)
        __shared__ ppo::Scalars s_sc;
        if (tid == 0) s_sc = ppo::make_scalars(hp, EPOCH ? (hi - lo) * px.world : global_rows, adv_moments ? adv_moments + 2 * m : nullptr);
        const ppo::Scalars& sc = s_sc;
#ifdef TS_B200_DIAGNOSTICS
        if (tid == 0 && g_tc_timeline_on && (int)blockIdx.x == g_tc_timeline_on - 1) g_tc_timeline_gate = (n_mb == 1 || m == n_mb - 2);   // a step WITH barrier 3
#endif
        tstamp(22);
        if (EPOCH && tid == 256 && !rmsprop) {    // Adam bias corrections of this step, off the critical path
            beta1_pow *= hp.beta1; beta2_pow *= hp.beta2;          // beta^(step0 + m + 1)
            s_step_size = (float)(hp.lr / (1.0 - beta1_pow));
            s_bc2_sqrt = (float)sqrt(1.0 - beta2_pow);
        }
        bool next_rows_ready = false;   // s_row holds the rows of this CTA's first tile of minibatch m + 1
        for (int64_t t = blockIdx.x; t < tiles; t += P) {
            const bool first = (t == (int64_t)blockIdx.x);     // first tile of this CTA: gradients are stored, not added
            const int nrows = (int)tsb::imin((int64_t)kRows, hi - (lo + t * kRows));
            if (!staged) {
                TileIn in;
                load_inputs(nrows, in);
                store_inputs(in);
            }
            staged = false;

            // dataset rows of this CTA's NEXT tile: the (DRAM-latency) load of the permutation entry is issued here and
            // committed to s_row after the critic pass -- s_row itself was consumed by load_inputs above / one step ago
            int32_t next_row = 0;
            int next_kind = 0;                                   // 1: next tile of this minibatch, 2: first tile of the next one
            if (t + P < tiles) next_kind = 1;
            else if (m + 1 < n_mb && (int64_t)blockIdx.x < mb_tiles(m + 1)) next_kind = 2;
            if (next_kind != 0 && tid < kRows) {
                const int mm = next_kind == 1 ? m : m + 1;
                const int64_t pos = mb_lo(mm) + (next_kind == 1 ? t + P : (int64_t)blockIdx.x) * kRows + tid;
                next_row = pos < mb_hi(mm) ? (perm ? __ldg(perm + pos) : (int32_t)pos) : 0;
            }

            // ================= critic ================================================================
            tstamp(1);
            if (!critic_issued) issue_weights(0);
            critic_issued = false;
            wait_weights(gc, 1);
            tstamp(2);
            trunk_forward(sm, sm0, S);
            tstamp(3);
            float vf_row = 0.0f;
            if (tid < kRows) {
                float dv[kMaxAct];
#pragma unroll
                for (int a = 0; a < kMaxAct; ++a) dv[a] = 0.0f;
                if (tid < nrows) {
                    const float value = reinterpret_cast<const float*>(sm + S.d3)[tid] + reinterpret_cast<const float*>(sm + S.b3)[0];
                    ppo::critic_row(sc, value, rowv[kRows + tid], rowv[3 * kRows + tid], vf_row, dv[0]);
                }
                write_dout_row(sm, sm0, S, tid, dv);
                const float sdv = tsb::warp_sum(dv[0]);
                if (lane == 0) red[warp] = sdv;                    // db3 (critic), one slot per warp
            }
            tstamp(4);
            trunk_backward(sm, sm0, S, gc, d.obs_dim, 1, grad, first, [&] { issue_weights(1); });
            tstamp(5);
            __syncthreads();
            if (tid == 0) out_acc(grad + gc.b3, (red[0] + red[1]) + (red[2] + red[3]), first);
            // row ids of this CTA's next tile (loaded at the top of the tile; s_row was consumed by load_inputs long ago)
            if (next_kind != 0 && tid < kRows) s_row[tid] = next_row;
            if (next_kind == 2) next_rows_ready = true;

            // ================= actor =================================================================
            wait_weights(ga, A);
            tstamp(6);
            trunk_forward(sm, sm0, S);
            tstamp(7);
            // Actor loss epilogue on all 16 warps: thread (row r = 32 q + lane, group cq) owns the actions a = cq + 4 u -- the
            // four groups' log-prob partials meet in shared memory, every thread then evaluates the row's surrogate and writes
            // dOut / column sums of ITS actions only (the 128-thread version was a 2 us dependent chain on one warp per scheduler).
            float clip_row = 0.0f;
            {
                const int q = warp & 3, cq = warp >> 2;
                const int r = 32 * q + lane;
                const float* b3 = reinterpret_cast<const float*>(sm + S.b3);
                const float* inv_var = red + 64;      // 1 / sigma^2
                const float* logc = red + 80;         // log sigma + log sqrt(2 pi)
                float diff[4], d2v[4];
                float lpp = 0.0f;
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const int a = cq + 4 * u;
                    diff[u] = 0.0f; d2v[u] = 0.0f;
                    if (a < A) {     // warp-uniform
                        const float mu = reinterpret_cast<const float*>(sm + S.d3)[a * kRows + r] + b3[a];
                        diff[u] = actt[a * kRows + r] - mu;
                        d2v[u] = diff[u] * diff[u] * inv_var[a];
                        lpp += fmaf(-0.5f, d2v[u], -logc[a]);      // log N(x; mu, sigma)
                    }
                }
                s_part[cq][r] = lpp;
                __syncthreads();
                const float lp = (s_part[0][r] + s_part[1][r]) + (s_part[2][r] + s_part[3][r]);
                float gl = 0.0f, obj = 0.0f;
                if (r < nrows) ppo::actor_row(sc, lp, rowv[2 * kRows + r], rowv[r], obj, gl);
                if (cq == 0) clip_row = obj;          // one group carries the row's objective into the loss sum
                float* dof = reinterpret_cast<float*>(sm + S.dof);
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const int a = cq + 4 * u;
                    if (a < A) {     // warp-uniform
                        const float g_mu = gl * diff[u] * inv_var[a];          // d loss / d mu_a
                        const float g_ls = gl * (d2v[u] - 1.0f);               // d loss / d logstd_a
                        dof[a * kRows + r] = g_mu;
                        uint32_t w0, w1, w2;
                        wg::split3_pair(g_mu, 0.0f, w0, w1, w2);
                        uint8_t* pdo = sm0 + (S.DO.base + wg::moff((uint32_t)r, (uint32_t)a, S.DO.RS));   // columns >= A stay zero (critic pass)
                        *reinterpret_cast<uint16_t*>(pdo) = (uint16_t)w0;
                        *reinterpret_cast<uint16_t*>(pdo + S.DO.part) = (uint16_t)w1;
                        *reinterpret_cast<uint16_t*>(pdo + 2 * S.DO.part) = (uint16_t)w2;
                        // column sums over the 32 rows of this warp: red[128 + 32 q + a] <- db3[a], red[128 + 32 q + 16 + a] <- dlogstd[a]
                        const float s_mu = tsb::warp_sum(g_mu), s_ls = tsb::warp_sum(g_ls);
                        if (lane == 0) { red[128 + 32 * q + a] = s_mu; red[128 + 32 * q + 16 + a] = s_ls; }
                    }
                }
            }
            tstamp(8);
            trunk_backward(sm, sm0, S, ga, d.obs_dim, A, grad, first, [] {});
            tstamp(9);

            // ================= loss sums + small gradients ===========================================
            const float s_clip = tsb::warp_sum(tid < kRows ? clip_row : 0.0f);
            const float s_vf = tsb::warp_sum(tid < kRows ? vf_row : 0.0f);
            if (lane == 0 && tid < kRows) { red[4 + warp] = s_clip; red[8 + warp] = s_vf; }
            __syncthreads();
            if (tid < A) {
                const float* cw = red + 128 + tid;
                out_acc(grad + ga.b3 + tid, (cw[0] + cw[32]) + (cw[64] + cw[96]), first);
                out_acc(grad + ga.ls + tid, (cw[16] + cw[48]) + (cw[80] + cw[112]) - sc.ent_coef * sc.inv_b * (float)nrows, first);
            }
            if (tid == 0) {
                float ent = 0.0f;     // entropy of the diagonal Gaussian: sum_a (0.5 + log sqrt(2 pi) + log sigma_a)
                for (int a = 0; a < A; ++a) ent += 0.5f + red[80 + a];
                float* ex = grad + d.n_params;
                out_acc(ex + 0, (red[4] + red[5]) + (red[6] + red[7]), first);
                out_acc(ex + 1, (red[8] + red[9]) + (red[10] + red[11]), first);
                out_acc(ex + 2, ent * (float)nrows, first);
                out_acc(ex + 3, (float)nrows, first);
            }
            __syncthreads();
        }
        if (!EPOCH) break;

        // ---- optimiser half of the step --------------------------------------------------------------
        __shared__ double s_red[4];
        const int Pm = (int)tsb::imin((int64_t)P, tiles);           // partial rows written for this minibatch
        const int64_t slice = (width + P - 1) / P;
        const int64_t i0 = (int64_t)blockIdx.x * slice;
        const int64_t i1 = tsb::imin(i0 + slice, width);
        const int e = tid & 127, q = tid >> 7;
        const int64_t step = step0 + m + 1;
        double* ss_cur = &ctl->ss[m & 1];
        tstamp(10);
        // gathers of this CTA's tile of the next minibatch: in flight across the barrier
        TileIn pin;
        const bool pre = (m + 1 < n_mb) && (int64_t)blockIdx.x < mb_tiles(m + 1);
        if (pre && !next_rows_ready) prefetch_rows(m + 1, blockIdx.x);
        gbar.arrive();
        if (pre) {
            const int nrows_next = (int)tsb::imin((int64_t)kRows, mb_hi(m + 1) - (mb_lo(m + 1) + (int64_t)blockIdx.x * kRows));
            load_inputs(nrows_next, pin);
        }
        gbar.wait();                                                // every partial row is complete
        tstamp(11);
        if (pre) { store_inputs(pin); staged = true; }
        tstamp(23);
        // fold: thread (e, q) sums rows q, q + 4, ... of element i0 + e [+ 128, ...]; 32 loads in flight
        double ss = 0.0;
        for (int64_t c = i0; c < i1; c += 128) {
            const int64_t i = c + e;
            float acc[4] = {0.f, 0.f, 0.f, 0.f};
            if (i < i1) {
                for (int p0 = q; p0 < Pm; p0 += 128) {
                    float v[32];
#pragma unroll
                    for (int u = 0; u < 32; ++u) {
                        const int p = p0 + 4 * u;
                        v[u] = p < Pm ? __ldcg(partials + (int64_t)p * width + i) : 0.0f;
                    }
#pragma unroll
                    for (int u = 0; u < 32; u += 4) { acc[0] += v[u]; acc[1] += v[u + 1]; acc[2] += v[u + 2]; acc[3] += v[u + 3]; }
                }
            }
            s_part[q][e] = (acc[0] + acc[1]) + (acc[2] + acc[3]);
            __syncthreads();
            tstamp(24);
            if (q == 0 && i < i1) {
                float g = (s_part[0][e] + s_part[1][e]) + (s_part[2][e] + s_part[3][e]);
                if (px.world > 1) {
                    // ---- cross-GPU sum of this element over NVLink peer memory (fused all-reduce) -----------
                    // push (value, seq) into every peer's receive slot of this rank, then gather the peers'
                    // packets from the local buffer and add in rank order (bit-identical on every rank)
                    const unsigned int seq = seq0 + (unsigned int)m + 1u;
                    const size_t slot = (size_t)(seq & 1u) * (size_t)width + (size_t)i;
                    const unsigned long long pkt = ((unsigned long long)seq << 32) | (unsigned long long)__float_as_uint(g);
                    for (int r = 0; r < px.world; ++r) {
                        if (r == px.rank) continue;
                        unsigned long long* dst = px.recv[r] + (size_t)px.rank * 2u * (size_t)width + slot;
                        asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(dst), "l"(pkt) : "memory");
                    }
                    g = peer_gather_sum(px.recv[px.rank] + slot, px.world, px.rank, g, seq, 2u * (size_t)width);
                }
                opt.grad_scratch[i] = g;
                if (i < d.n_params) ss += (double)g * (double)g;
            }
            __syncthreads();
        }
        if (tid < 128) {
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) ss += tsb::shfl_xor_f64(ss, off);
            if (lane == 0) s_red[warp] = ss;
        }
        __syncthreads();
        tstamp(12);
        if (tid == 0) atomicAdd(ss_cur, (s_red[0] + s_red[1]) + (s_red[2] + s_red[3]));
        // the optimiser state of this thread's elements: loads in flight across the barrier
        const bool one_pass = slice <= kThreads;      // (always, unless the network is far larger than the grid)
        const int64_t i_own = i0 + tid;
        const bool own = one_pass && i_own < i1 && i_own < d.n_params;
        float pv_own = 0.f, m_own = 0.f, v_own = 0.f;
        gbar.arrive();
        if (own) { pv_own = opt.params_w[i_own]; m_own = opt.exp_avg[i_own]; v_own = opt.exp_avg_sq[i_own]; }
        gbar.wait();                                                // global sum of squares is complete
        tstamp(13);
        if (tid == 0) {
            const float total_norm = (float)sqrt(*((volatile double*)ss_cur));
            s_coef = hp.max_grad_norm > 0.0 ? optim::clip_coef((float)hp.max_grad_norm, total_norm) : 1.0f;
            s_norm = total_norm;
            if (blockIdx.x == 0) ctl->ss[(m + 1) & 1] = 0.0;       // next step's accumulator (idle until barrier 3)
        }
        __syncthreads();
        tstamp(25);
        const float coef = s_coef, step_size = s_step_size, bc2_sqrt = s_bc2_sqrt;
        const float w1 = (float)(1.0 - hp.beta1), w2 = (float)(1.0 - hp.beta2);
        const float beta2 = (float)hp.beta2, adam_eps = (float)hp.adam_eps, wd = (float)hp.weight_decay;
        const float lr = (float)hp.lr;     // RMSprop: beta2 holds alpha, w2 = 1 - alpha
        auto adam_elem = [&](int64_t i, float g, float pv, float mm, float v) {
            if (rmsprop) {
                optim::rmsprop_elem(g * coef, pv, v, lr, beta2, w2, adam_eps, wd);
                opt.exp_avg_sq[i] = v; opt.params_w[i] = pv;
                if (wimg != nullptr) img_scatter(d, S, sbase, i, pv, wimg);
                return;
            }
            optim::adam_elem<true>(g * coef, pv, mm, v, step_size, bc2_sqrt, beta2, w1, w2, adam_eps, wd);
            opt.exp_avg[i] = mm; opt.exp_avg_sq[i] = v; opt.params_w[i] = pv;
            if (wimg != nullptr) img_scatter(d, S, sbase, i, pv, wimg);
        };
        if (one_pass) {
            if (own) adam_elem(i_own, opt.grad_scratch[i_own], pv_own, m_own, v_own);
        } else {
            for (int64_t i = i0 + tid; i < i1 && i < d.n_params; i += kThreads)
                adam_elem(i, opt.grad_scratch[i], opt.params_w[i], opt.exp_avg[i], opt.exp_avg_sq[i]);
        }
        tstamp(26);
        if (wimg != nullptr) wg::fence_proxy_async_all();      // image stores (generic proxy) before the peers' bulk copies
        tstamp(14);
        const bool more = m + 1 < n_mb;
        if (more) gbar.arrive();                                    // barrier 3 (updated parameters visible to every CTA) ...
        if (tid == 32 && blockIdx.x == 0) {                         // ... the loss table row is written under it, off tid 0's poll
            // the folded loss sums were written by the owner of the last slice before barrier 2; nothing rewrites them before the
            // next step's fold, i.e. after every CTA passed the NEXT barrier 1
            const float* ex = opt.grad_scratch + d.n_params;
            const float e0 = __ldcg(ex), e1 = __ldcg(ex + 1), e2 = __ldcg(ex + 2), e3 = __ldcg(ex + 3);
            if (opt.stats) {
                float* sr = opt.stats + (int64_t)m * TS_PPO_STATS_STRIDE;
                ppo::loss_row(e0, e1, e2, e3 > 0.0f ? e3 : 1.0f, hp, sr);
                sr[4] = s_norm; sr[5] = e3; sr[6] = 0.0f; sr[7] = 0.0f;
            }
        }
        if (more) {
            gbar.wait();
            if (pre) { issue_weights(0); critic_issued = true; }
        }
        tstamp(15);
    }
    if (EPOCH && tid == 0) {
        if (blockIdx.x == 0) {
            *opt.step_count = step0 + n_mb;
            if (px.world > 1) *px.hdr = seq0 + (unsigned int)n_mb;
        }
        __threadfence();
        if (atomicAdd(&ctl->depart, 1u) == gridDim.x - 1) {
            ctl->arrive = 0u; ctl->depart = 0u; ctl->ss[0] = 0.0; ctl->ss[1] = 0.0;
            __threadfence();
        }
    }
}


// ---- forward-only kernels (value pass / log-prob pass), persistent over 128-row tiles -----------
// Per tile: X (bf16x3) -> layer 1 -> tanh -> H1 (bf16x3) -> layer 2 -> tanh in registers -> head as SIMT dot products
// over the thread's columns.  The next tile's rows are loaded from global memory while this tile's MMAs run.
struct SmemF {
    int KXP;
    Mat X, H1, W1, W2;
    uint32_t w3f, b1, b2, b3, ls, part;
    uint32_t total;
};
__host__ __device__ constexpr SmemF make_smem_f(int kxp, uint32_t sbase) {
    SmemF s{};
    s.KXP = kxp;
    uint32_t o = 0;
    auto mat = [&](Mat& m, int rows, int cols) {
        m.base = sbase + o; m.part = mat_bytes(rows, cols); m.RS = (uint32_t)(cols / 8) * 128u; o += 3u * m.part;
    };
    mat(s.X, kRows, s.KXP);
    mat(s.H1, kRows, H);
    mat(s.W1, H, s.KXP);
    mat(s.W2, H, H);
    s.w3f = o;  o += kMaxAct * H * 4;
    s.b1 = o;   o += H * 4;
    s.b2 = o;   o += H * 4;
    s.b3 = o;   o += kMaxAct * 4;
    s.ls = o;   o += kMaxAct * 4;
    s.part = o; o += 2 * kRows * kMaxAct * 4;   // head partial sums of the two column halves [half][a][row]
    s.total = o;
    return s;
}

// MODE 0: out0[r] = critic(in0[r]) and (if in1) out1[r] = critic(in1[r])      (a2c.py:123-126)
// MODE 1: out0[r] = log N(in1[r] | mu(in0[r]), exp(logstd)), out1 = mu (nullable)   (ppo.py:157-161)
template <int MODE, int KXP>
__global__ void __launch_bounds__(kThreads, 1) forward_tc_kernel(
    const float* __restrict__ params, const ts_actor_critic_desc d, const float* __restrict__ in0,
    float* __restrict__ out0, const float* __restrict__ in1, float* __restrict__ out1, int64_t n) {
    extern __shared__ __align__(1024) uint8_t sm[];
    const int tid = threadIdx.x, lane = tid & 31;
    const uint32_t sbase = wg::smem_u32(sm);
    uint8_t* sm0 = sm - sbase;
    const SmemF S = make_smem_f(KXP, sbase);
    const int out_dim = MODE == 0 ? 1 : d.act_dim;
    const NetG g = MODE == 0 ? NetG{d.c_w1, d.c_b1, d.c_w2, d.c_b2, d.c_w3, d.c_b3, -1}
                             : NetG{d.a_w1, d.a_b1, d.a_w2, d.a_b2, d.a_w3, d.a_b3, d.a_logstd};
    // weights: W1, W2 as tensor-core B operands (shared memory); head weights / biases as fp32
    stage_chunks(sm0, S.W1, H, d.obs_dim, S.KXP, [&](int o) { return params + g.w1 + (int64_t)o * d.obs_dim; });
    stage_chunks(sm0, S.W2, H, H, H, [&](int o) { return params + g.w2 + (int64_t)o * H; });
    float* w3f = reinterpret_cast<float*>(sm + S.w3f);
    float* b1 = reinterpret_cast<float*>(sm + S.b1);
    float* b2 = reinterpret_cast<float*>(sm + S.b2);
    float* b3 = reinterpret_cast<float*>(sm + S.b3);
    float* ls = reinterpret_cast<float*>(sm + S.ls);
    float* part = reinterpret_cast<float*>(sm + S.part);
    for (int e = tid; e < kMaxAct * H; e += kThreads) w3f[e] = (e >> 6) < out_dim ? __ldg(params + g.w3 + e) : 0.0f;
    for (int e = tid; e < H; e += kThreads) { b1[e] = __ldg(params + g.b1 + e); b2[e] = __ldg(params + g.b2 + e); }
    if (tid < kMaxAct) {
        b3[tid] = tid < out_dim ? __ldg(params + g.b3 + tid) : 0.0f;
        // sigma_a = exp(logstd_a), once per CTA; the log-prob keeps torch's expression order (normal_logp_term)
        ls[tid] = (MODE == 1 && tid < out_dim) ? expf(__ldg(params + g.ls + tid)) : 1.0f;
    }

    const int64_t tiles_per = (n + kRows - 1) / kRows;
    const int64_t tiles = tiles_per * ((MODE == 0 && in1) ? 2 : 1);
    const int64_t my_n = tiles > (int64_t)blockIdx.x ? (tiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;   // tiles of this CTA
    auto tile_of = [&](int64_t k) { return (int64_t)blockIdx.x + k * gridDim.x; };
    auto tile_src = [&](int64_t t, const float*& src, int64_t& row0, int& nrows, bool& second) {
        second = t >= tiles_per;
        row0 = (second ? t - tiles_per : t) * kRows;
        nrows = (int)tsb::imin((int64_t)kRows, n - row0);
        src = (MODE == 0 && second) ? in1 : in0;
    };
    auto x_load = [&](int64_t k, float (&xv)[8]) {     // one (row, 8-column chunk) per thread
        const float* src; int64_t row0; int nrows; bool second;
        tile_src(tile_of(k), src, row0, nrows, second);
        chunk_load(kRows, d.obs_dim, S.KXP, [&](int r) {
            return r < nrows ? src + (row0 + r) * d.obs_dim : (const float*)nullptr;
        }, xv);
    };
    const int half = tid >> 8;                 // column half of the thread's layer elements
    const int r0 = lay_row0() + wg::frag_row(0);    // its rows: r0 and r0 + 8

    float xv[8];
    if (my_n > 0) x_load(0, xv);
    for (int64_t k = 0; k < my_n; ++k) {
        const float* src; int64_t row0; int nrows; bool second;
        tile_src(tile_of(k), src, row0, nrows, second);
        __syncthreads();                       // the previous tile's operand and `part` reads are complete
        chunk_store(sm0, S.X, kRows, S.KXP, xv);
        if (k + 1 < my_n) x_load(k + 1, xv);   // global loads fly under this tile's MMAs
        publish();
        float acc[kCols], h[kCols];
        if (S.KXP == 16) wg_gemm<2 * kCols, 1, 0, 0>(acc, S.X, lay_row0(), S.W1, lay_col0());
        else wg_gemm<2 * kCols, 2, 0, 0>(acc, S.X, lay_row0(), S.W1, lay_col0());
        epi_tanh(sm0, S.H1, acc, b1);
        publish();
        wg_gemm<2 * kCols, H / 16, 0, 0>(acc, S.H1, lay_row0(), S.W2, lay_col0());
#pragma unroll
        for (int e = 0; e < kCols; ++e) h[e] = tanh_mufu(acc[e] + b2[lay_col0() + wg::frag_col(e)]);
        // head = h2 . W3^T: the thread's 8 columns, then the quad (same rows, the 32 columns of the half)
        for (int a = 0; a < out_dim; ++a) {
            float p0 = 0.0f, p1 = 0.0f;
#pragma unroll
            for (int i = 0; i < kCols / 4; ++i) {
                const float2 w = *reinterpret_cast<const float2*>(w3f + a * H + lay_col0() + wg::frag_col(4 * i));
                p0 = fmaf(h[4 * i], w.x, p0); p0 = fmaf(h[4 * i + 1], w.y, p0);
                p1 = fmaf(h[4 * i + 2], w.x, p1); p1 = fmaf(h[4 * i + 3], w.y, p1);
            }
            p0 += __shfl_xor_sync(0xffffffffu, p0, 1); p0 += __shfl_xor_sync(0xffffffffu, p0, 2);
            p1 += __shfl_xor_sync(0xffffffffu, p1, 1); p1 += __shfl_xor_sync(0xffffffffu, p1, 2);
            if ((lane & 3) == 0) {
                part[(half * kMaxAct + a) * kRows + r0] = p0;
                part[(half * kMaxAct + a) * kRows + r0 + 8] = p1;
            }
        }
        __syncthreads();
        if (tid < nrows) {
            const int r = tid;
            if (MODE == 0) {
                (second ? out1 : out0)[row0 + r] = (part[r] + part[kMaxAct * kRows + r]) + b3[0];
            } else {
                float lp = 0.0f;
                for (int a = 0; a < out_dim; ++a) {
                    const float mu = (part[a * kRows + r] + part[(kMaxAct + a) * kRows + r]) + b3[a];
                    lp += ppo::normal_logp_term(__ldg(in1 + (row0 + r) * out_dim + a), mu, ls[a]);
                    if (out1) out1[(row0 + r) * out_dim + a] = mu;
                }
                out0[row0 + r] = lp;
            }
        }
    }
}

}  // namespace

#ifdef TS_B200_DIAGNOSTICS
extern "C" int ts_tc_timeline(int32_t enable, uint64_t* out32 /* host, nullable */) {
    int on = enable;
    TS_CUDA(cudaMemcpyToSymbol(g_tc_timeline_on, &on, sizeof(int)));
    if (out32) TS_CUDA(cudaMemcpyFromSymbol(out32, g_tc_timeline, 32 * sizeof(unsigned long long)));
    return 0;
}
#endif

namespace tsb {
bool tc_supported(const ts_actor_critic_desc& d) {
    // tanh trunks, Gaussian head, separate actor / critic parameters (a shared trunk = aliased offsets would break
    // the store-not-add gradient write-out); everything else runs the fp32 SIMT kernels
    return d.hidden == H && d.obs_dim >= 1 && d.obs_dim <= 32 && d.act_dim >= 1 && d.act_dim <= kMaxAct && d.flags == 0 &&
           d.a_w1 != d.c_w1 && d.a_logstd >= 0;
}

// the dynamic shared memory opt-in is a per-device attribute of each kernel instantiation
template <auto Kernel>
static int opt_in_smem(size_t smem) {
    static bool configured[kMaxDevices] = {};
    const int dev = device_ordinal();
    if (!configured[dev]) {
        TS_CUDA(cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        configured[dev] = true;
    }
    return 0;
}

// f(std::integral_constant<int, KXP>) for the instantiation that serves obs_dim (tc_supported: obs_dim <= 32)
template <class F>
static int with_kxp(int obs_dim, F&& f) {
    return kxp_of(obs_dim) == 16 ? f(std::integral_constant<int, 16>{}) : f(std::integral_constant<int, 32>{});
}

int launch_ppo_grad_tc(const float* params, const ts_actor_critic_desc& d, const ts_ppo_hparams& hp, const float* obs,
                       const float* act, const float* adv, const float* ret, const float* logp_old, const float* v_s,
                       const int32_t* perm, int64_t lo, int64_t hi, int64_t global_rows, const float* adv_moments,
                       float* grad, cudaStream_t st) {
    return with_kxp(d.obs_dim, [&](auto kxp) {
        constexpr int KXP = decltype(kxp)::value;
        constexpr size_t smem = make_smem(KXP, 0).total;
        if (int e = opt_in_smem<ppo_tc_kernel<false, KXP>>(smem)) return e;
        const int64_t tiles = (hi - lo + kRows - 1) / kRows;
        const unsigned grid = (unsigned)imin(tiles, num_sms());
        ppo_tc_kernel<false, KXP><<<grid, kThreads, smem, st>>>(params, d, hp, obs, act, adv, ret, logp_old, v_s, perm, lo, hi - lo,
                                                                hi, 1, global_rows, adv_moments, grad, AdamArgs{}, (uint8_t*)nullptr,
                                                                PeerArgs{});
        return check_launch("ts_ppo_grad(tc)");
    });
}

// n_mb consecutive optimiser steps (minibatch fwd/bwd + gradient fold + clip + Adam + stats each) in ONE
// cooperative launch: every CTA is resident (grid <= #SMs, 1 CTA / SM), so the in-kernel grid barriers are safe.
int launch_ppo_epoch_tc(float* params, const ts_actor_critic_desc& d, const ts_ppo_hparams& hp, const float* obs,
                        const float* act, const float* adv, const float* ret, const float* logp_old, const float* v_s,
                        const int32_t* perm, int64_t lo0, int64_t mb_size, int64_t end, int n_mb, const float* adv_moments,
                        float* partials, float* grad_scratch, float* exp_avg, float* exp_avg_sq, int64_t* step_count,
                        float* stats, void* weight_image, const PeerArgs& px, cudaStream_t st) {
    return with_kxp(d.obs_dim, [&](auto kxp) {
        constexpr int KXP = decltype(kxp)::value;
        constexpr Smem S = make_smem(KXP, 0);
        if (int e = opt_in_smem<ppo_tc_kernel<true, KXP>>(S.total)) return e;
        const int64_t last = end - (lo0 + (int64_t)(n_mb - 1) * mb_size);
        const int64_t widest = n_mb > 1 ? (mb_size > last ? mb_size : last) : last;
        const unsigned grid = (unsigned)imin((widest + kRows - 1) / kRows, num_sms());
        const AdamArgs opt{params, grad_scratch, exp_avg, exp_avg_sq, step_count, stats};
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(grid); cfg.blockDim = dim3(kThreads); cfg.dynamicSmemBytes = S.total; cfg.stream = st;
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeCooperative;
        attr[0].val.cooperative = 1;
        cfg.attrs = attr; cfg.numAttrs = 1;
        const int64_t zero = 0;
        // scratch layout: [128-byte control block (grid-barrier state, zero between launches)][critic block][actor block]
        uint8_t* wimg = weight_image ? static_cast<uint8_t*>(weight_image) + kCtlBytes : nullptr;
        if (wimg) {   // (re)build the pre-split image from the current parameters: the host may have changed them
            TS_CUDA(cudaMemsetAsync(wimg, 0, 2 * (size_t)S.wblk_bytes, st));
            weight_image_build_kernel<KXP><<<(unsigned)((d.n_params + 255) / 256), 256, 0, st>>>(params, d, wimg);
            if (int e = check_launch("ts_ppo_update(weight image)")) return e;
        }
        TS_CUDA(cudaLaunchKernelEx(&cfg, ppo_tc_kernel<true, KXP>, (const float*)params, d, hp, obs, act, adv, ret, logp_old, v_s,
                                   perm, lo0, mb_size, end, n_mb, zero, adv_moments, partials, opt, wimg, px));
        return check_launch("ts_ppo_epoch(tc)");
    });
}

int64_t weight_image_bytes(const ts_actor_critic_desc& d) {
    return tc_supported(d) ? (int64_t)kCtlBytes + 2 * (int64_t)make_smem(kxp_of(d.obs_dim), 0).wblk_bytes : 0;
}

int launch_forward_tc(int mode, const float* params, const ts_actor_critic_desc& d, const float* in0, float* out0,
                      const float* in1, float* out1, int64_t n, cudaStream_t st) {
    return with_kxp(d.obs_dim, [&](auto kxp) {
        constexpr int KXP = decltype(kxp)::value;
        constexpr size_t smem = make_smem_f(KXP, 0).total;
        const int64_t tiles = ((n + kRows - 1) / kRows) * ((mode == 0 && in1) ? 2 : 1);
        const unsigned grid = (unsigned)imin(tiles, num_sms());
        if (mode == 0) {
            if (int e = opt_in_smem<forward_tc_kernel<0, KXP>>(smem)) return e;
            forward_tc_kernel<0, KXP><<<grid, kThreads, smem, st>>>(params, d, in0, out0, in1, out1, n);
        } else {
            if (int e = opt_in_smem<forward_tc_kernel<1, KXP>>(smem)) return e;
            forward_tc_kernel<1, KXP><<<grid, kThreads, smem, st>>>(params, d, in0, out0, in1, out1, n);
        }
        return check_launch(mode == 0 ? "ts_critic_forward(tc)" : "ts_actor_logp(tc)");
    });
}
}  // namespace tsb
