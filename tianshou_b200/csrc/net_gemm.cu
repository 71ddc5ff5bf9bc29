// Generic fp32-faithful GEMM on the Hopper tensor cores (wgmma, sm_90a) for the layered networks of the off-policy
// algorithms (SAC / DDPG critics MLP[256,256] on obs 376, DQN NatureCNN as implicit GEMM over im2col rows):
//                       C[M,N] (+)= epilogue( A[M,K] * B[N,K]^T )
//
// Reference code replaced: every nn.Linear / nn.Conv2d forward and its autograd backward inside
// SAC._update_with_batch (modelfree/sac.py:304-336), _minimize_critic_squared_loss (modelfree/ddpg.py:267-285),
// DQN._update_with_batch (modelfree/dqn.py:382-404), DQNet (env/atari/atari_network.py:60-122).
//
// Operands are plain fp32 arrays in global memory; each may be given K-major (k contiguous: a[mn*ld + k]) or
// MN-major (mn contiguous: a[k*ld + mn]), which covers forward (X W^T), input gradient (dY W) and weight
// gradient (dY^T X) without materialising a transpose.  A CTA computes a 128 x 128 tile: the 256 threads stage
// 128 x 64 operand chunks into shared memory as bf16x3 pieces (x = b0 + b1 + b2, 24 significant bits) in the
// blocked no-swizzle layout of wgmma.cuh, two stages deep, and each of the two warpgroups issues the six
// partial-product wgmma.mma_async per K = 16 step for its 64 rows into an fp32 register accumulator (64 x 128);
// staging of chunk i + 1 overlaps the MMAs of chunk i.  Epilogue: registers -> bias -> activation -> optional
// ReLU-derivative mask -> fp32 stores (or split-K partial).
#include "common.cuh"
#include "wgmma.cuh"

namespace {

constexpr int BM = 128, BN = 128, BK = 64, kThreads = 256;
constexpr uint32_t kPartBytes = BM * BK * 2;                 // one bf16 piece of a 128 x 64 (or 64 x 128) tile
constexpr uint32_t kOperandBytes = 3 * kPartBytes;           // 48 KB
constexpr uint32_t kStageBytes = 2 * kOperandBytes;          // A + B
constexpr uint32_t kSmemBytes = 2 * kStageBytes;             // two stages: 192 KB

struct Operand {
    const float* p;
    int64_t ld;
    int mn_major;      // 0: p[mn * ld + k] (k contiguous), 1: p[k * ld + mn] (mn contiguous)
    int mn_extent;
};

struct GemmParams {
    Operand a, b;
    float* c;            // [M][ldc] row-major, or split-K workspace [splits][M][N] when splits > 1
    int64_t ldc;
    int M, N, K;
    const float* bias;   // [N], nullable
    int act;             // TS_ACT_*
    const float* mask;   // nullable: activation derivative of the PRODUCER layer from its OUTPUT y = mask[m * ld_mask + n]:
    int64_t ld_mask;     //   mask_kind TS_ACT_RELU: x * (y > 0) ;  TS_ACT_TANH: x * (1 - y^2)
    int mask_kind;
    int accumulate;      // C += result
    int splits;          // split-K factor (grid.z); partials are reduced by splitk_reduce_kernel
    int k_per_split;     // multiple of BK
};

__device__ __forceinline__ uint32_t moff(uint32_t r, uint32_t c, uint32_t RS) {
    return (r >> 3) * RS + (c >> 3) * 128u + (r & 7u) * 16u + (c & 7u) * 2u;
}
__device__ __forceinline__ void split3_pair(float x0, float x1, uint32_t& w0, uint32_t& w1, uint32_t& w2) {
    const uint32_t u0 = __float_as_uint(x0), u1 = __float_as_uint(x1);
    w0 = __byte_perm(u0, u1, 0x7632);
    const float r0 = x0 - __uint_as_float(u0 & 0xffff0000u), r1 = x1 - __uint_as_float(u1 & 0xffff0000u);
    const uint32_t v0 = __float_as_uint(r0), v1 = __float_as_uint(r1);
    w1 = __byte_perm(v0, v1, 0x7632);
    const float s0 = r0 - __uint_as_float(v0 & 0xffff0000u), s1 = r1 - __uint_as_float(v1 & 0xffff0000u);
    w2 = __byte_perm(__float_as_uint(s0), __float_as_uint(s1), 0x7632);
}

// Stage one 128 (mn) x 64 (k) chunk of an operand.  Shared-memory matrix = [rows = non-contiguous dim][cols =
// contiguous dim]: K-major -> [128 mn][64 k] (RS = 1024), MN-major -> [64 k][128 mn] (RS = 2048); one task = 8
// contiguous floats -> one 16-byte chunk per piece.  1024 tasks / 256 threads.
// The global loads of BOTH operands of a chunk are issued before any of them is consumed (one round trip per chunk, not two).
struct Staged { float v[4][8]; };
__device__ __forceinline__ void load_operand(Staged& s, const Operand& op, int mn0, int k0, int k_end) {
    const bool vec_ok = ((op.ld & 3) == 0) && ((reinterpret_cast<uintptr_t>(op.p) & 15u) == 0);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
        const int task = (int)threadIdx.x + u * kThreads;
        int mn, k;
        if (!op.mn_major) { mn = mn0 + (task >> 3); k = k0 + (task & 7) * 8; }
        else              { k = k0 + (task >> 4); mn = mn0 + (task & 15) * 8; }
        float* v = s.v[u];
        // contiguous run of 8 along the fast dimension; `lim` = first invalid index of that dimension
        const int fast = op.mn_major ? mn : k, lim = op.mn_major ? op.mn_extent : k_end;
        const bool row_ok = op.mn_major ? (k < k_end) : (mn < op.mn_extent);
        const float* src = op.p + (int64_t)(op.mn_major ? k : mn) * op.ld + fast;
        if (row_ok && fast + 8 <= lim && vec_ok && ((fast & 3) == 0)) {
            const float4 x0 = __ldg(reinterpret_cast<const float4*>(src));
            const float4 x1 = __ldg(reinterpret_cast<const float4*>(src) + 1);
            v[0] = x0.x; v[1] = x0.y; v[2] = x0.z; v[3] = x0.w; v[4] = x1.x; v[5] = x1.y; v[6] = x1.z; v[7] = x1.w;
        } else {
#pragma unroll
            for (int j = 0; j < 8; ++j) v[j] = (row_ok && fast + j < lim) ? __ldg(src + j) : 0.0f;
        }
    }
}
__device__ __forceinline__ void store_operand(uint8_t* sm0, uint32_t base, const Staged& s, int mn_major) {
#pragma unroll
    for (int u = 0; u < 4; ++u) {
        const int task = (int)threadIdx.x + u * kThreads;
        const int r = mn_major ? (task >> 4) : (task >> 3), c0 = mn_major ? (task & 15) * 8 : (task & 7) * 8;
        uint32_t w0[4], w1[4], w2[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) split3_pair(s.v[u][2 * j], s.v[u][2 * j + 1], w0[j], w1[j], w2[j]);
        const uint32_t RS = mn_major ? 2048u : 1024u;
        uint8_t* p = sm0 + (base + moff((uint32_t)r, (uint32_t)c0, RS));
        *reinterpret_cast<uint4*>(p) = make_uint4(w0[0], w0[1], w0[2], w0[3]);
        *reinterpret_cast<uint4*>(p + kPartBytes) = make_uint4(w1[0], w1[1], w1[2], w1[3]);
        *reinterpret_cast<uint4*>(p + 2 * kPartBytes) = make_uint4(w2[0], w2[1], w2[2], w2[3]);
    }
}

__device__ __forceinline__ float apply_act_grad(float x, float y, int kind) {
    return kind == TS_ACT_TANH ? x * fmaf(-y, y, 1.0f) : (y > 0.0f ? x : 0.0f);
}
__device__ __forceinline__ float apply_act(float x, int act) {
    if (act == TS_ACT_RELU) return fmaxf(x, 0.0f);
    if (act == TS_ACT_TANH) return tanhf(x);
    return x;
}

// TA / TB: operand A / B given MN-major (the wgmma transpose flags are immediates)
template <int TA, int TB>
__global__ void __launch_bounds__(kThreads, 1) net_gemm_kernel(const GemmParams P) {
    extern __shared__ __align__(1024) uint8_t sm[];
    const int tid = threadIdx.x, wgi = tid >> 7;
    const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
    const int kb = blockIdx.z * P.k_per_split;
    const int ke = P.splits > 1 ? (int)tsb::imin((int64_t)P.K, (int64_t)kb + P.k_per_split) : P.K;
    const uint32_t sbase = wg::smem_u32(sm);
    uint8_t* sm0 = sm - sbase;
    // descriptor strides (see wgmma.cuh); warpgroup wgi reads rows [64 wgi, 64 wgi + 64) of A = 8 core matrices along MN
    constexpr uint32_t a_lbo = TA ? 2048u : 128u, a_sbo = TA ? 128u : 1024u, a_step = TA ? 4096u : 256u;
    constexpr uint32_t b_lbo = TB ? 2048u : 128u, b_sbo = TB ? 128u : 1024u, b_step = TB ? 4096u : 256u;
    const uint32_t a_rows = 8u * a_sbo * (uint32_t)wgi;
    float acc[BN / 2];
#pragma unroll
    for (int j = 0; j < BN / 2; ++j) acc[j] = 0.0f;
    const int chunks = (ke - kb + BK - 1) / BK;
    for (int i = 0; i < chunks; ++i) {
        const int st = i & 1;
        const int k0 = kb + i * BK;
        Staged sa, sb;
        load_operand(sa, P.a, m0, k0, ke);
        load_operand(sb, P.b, n0, k0, ke);
        if (i >= 2) {            // both warpgroups' MMAs of chunk i - 2 are done with this stage
            wg::wait<1>();
            __syncthreads();
        }
        const uint32_t a_base = sbase + st * kStageBytes, b_base = a_base + kOperandBytes;
        store_operand(sm0, a_base, sa, TA);
        store_operand(sm0, b_base, sb, TB);
        wg::fence_async_smem();
        __syncthreads();
        // a tail chunk shorter than BK is zero-padded by load_operand: all BK / 16 steps run
        wg::fence();
        wg::gemm_bf16x3<BN, BK / 16, TA, TB>(acc, a_base + a_rows, kPartBytes, a_lbo, a_sbo, a_step, b_base, kPartBytes, b_lbo, b_sbo,
                                              b_step, i > 0);
        wg::commit();
    }
    wg::wait<0>();

    // ---- epilogue: the thread's accumulator elements, two consecutive columns per store ------------------------
    float* cbase = P.c + (P.splits > 1 ? (int64_t)blockIdx.z * P.M * P.N : 0);
    const int64_t ldc = P.splits > 1 ? P.N : P.ldc;
    const bool plain = P.splits > 1;         // partials: raw accumulator, epilogue ops happen in the reduce kernel
#pragma unroll
    for (int e = 0; e < BN / 2; e += 2) {
        const int m = m0 + 64 * wgi + wg::frag_row(e), n = n0 + wg::frag_col(e);
        if (m >= P.M || n >= P.N) continue;
        float* dst = cbase + (int64_t)m * ldc + n;
        float v[2] = {acc[e], acc[e + 1]};
        const bool pair = n + 1 < P.N;
        if (!plain) {
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                if (j == 1 && !pair) break;
                float x = v[j];
                if (P.bias) x += __ldg(P.bias + n + j);
                x = apply_act(x, P.act);
                if (P.mask) x = apply_act_grad(x, __ldg(P.mask + (int64_t)m * P.ld_mask + n + j), P.mask_kind);
                if (P.accumulate) x += dst[j];
                v[j] = x;
            }
        }
        if (pair && (reinterpret_cast<uintptr_t>(dst) & 7u) == 0) *reinterpret_cast<float2*>(dst) = make_float2(v[0], v[1]);
        else {
            dst[0] = v[0];
            if (pair) dst[1] = v[1];
        }
    }
}

// C (+)= epilogue( sum_z partial[z] ), fixed summation order (deterministic)
__global__ void splitk_reduce_kernel(const float* __restrict__ part, int splits, float* __restrict__ c, int64_t ldc, int M, int N,
                                     const float* __restrict__ bias, int act, const float* __restrict__ mask, int64_t ld_mask,
                                     int mask_kind, int accumulate) {
    const int64_t total = (int64_t)M * N;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
        const int m = (int)(e / N), n = (int)(e - (int64_t)m * N);
        float x = 0.0f;
        for (int z = 0; z < splits; ++z) x += part[(int64_t)z * total + e];
        if (bias) x += __ldg(bias + n);
        x = apply_act(x, act);
        if (mask) x = apply_act_grad(x, __ldg(mask + (int64_t)m * ld_mask + n), mask_kind);
        float* dst = c + (int64_t)m * ldc + n;
        if (accumulate) x += *dst;
        *dst = x;
    }
}

// out[n] (+)= sum_m x[m * ld + n]   (bias gradients): block = 32 columns x 8 row lanes, fixed order
__global__ void colsum_kernel(const float* __restrict__ x, int64_t ld, int M, int N, float* __restrict__ out, int accumulate) {
    __shared__ float s[8][33];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int n = blockIdx.x * 32 + lane;
    float acc = 0.0f;
    if (n < N) {
        for (int m = w; m < M; m += 8) acc += __ldg(x + (int64_t)m * ld + n);
    }
    s[w][lane] = acc;
    __syncthreads();
    if (w == 0 && n < N) {
        float t = 0.0f;
#pragma unroll
        for (int k = 0; k < 8; ++k) t += s[k][lane];
        out[n] = accumulate ? out[n] + t : t;
    }
}

}  // namespace

namespace tsb {

size_t net_gemm_workspace_floats(int M, int N, int K, int* splits_out) {
    // split-K whenever the output tiles alone leave most SMs idle: weight gradients over im2col rows (K = tens of thousands),
    // and every layer of a batch-256 MLP (4 output tiles, 4 .. 7 chunks: a lone CTA per tile would walk them one round trip
    // after the other while the other SMs idle)
    const int tiles = ((M + BM - 1) / BM) * ((N + BN - 1) / BN);
    const int chunks = (K + BK - 1) / BK;
    int splits = 1;
    if (chunks >= 2 && tiles < 64) {
        splits = (int)imin((int64_t)((num_sms() + tiles - 1) / tiles), (int64_t)chunks);
        if (splits < 1) splits = 1;
    }
    if (splits_out) *splits_out = splits;
    return splits > 1 ? (size_t)splits * M * N : 0;
}

int net_gemm(const float* a, int64_t lda, int a_mn, const float* b, int64_t ldb, int b_mn, float* c, int64_t ldc, int M, int N,
             int K, const float* bias, int act, const float* mask, int64_t ld_mask, int mask_kind, int accumulate, float* workspace,
             size_t workspace_floats, cudaStream_t st) {
    static bool configured[kMaxDevices] = {};
    const int dev = device_ordinal();
    if (!configured[dev]) {
        TS_CUDA(cudaFuncSetAttribute(net_gemm_kernel<0, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBytes));
        TS_CUDA(cudaFuncSetAttribute(net_gemm_kernel<0, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBytes));
        TS_CUDA(cudaFuncSetAttribute(net_gemm_kernel<1, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBytes));
        TS_CUDA(cudaFuncSetAttribute(net_gemm_kernel<1, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBytes));
        configured[dev] = true;
    }
    if (M <= 0 || N <= 0) return 0;
    GemmParams P;
    P.a = Operand{a, lda, a_mn, M};
    P.b = Operand{b, ldb, b_mn, N};
    P.c = c; P.ldc = ldc; P.M = M; P.N = N; P.K = K;
    P.bias = bias; P.act = act; P.mask = mask; P.ld_mask = ld_mask; P.mask_kind = mask_kind; P.accumulate = accumulate;
    int splits = 1;
    const size_t need = net_gemm_workspace_floats(M, N, K, &splits);
    if (splits > 1 && (workspace == nullptr || workspace_floats < need)) splits = 1;     // no room: run unsplit
    const int chunks = (K + BK - 1) / BK;
    P.splits = splits;
    P.k_per_split = splits > 1 ? ((chunks + splits - 1) / splits) * BK : K;
    if (splits > 1) {
        splits = (K + P.k_per_split - 1) / P.k_per_split;       // drop empty tail splits
        P.splits = splits;
        P.c = workspace;
    }
    const dim3 grid((M + BM - 1) / BM, (N + BN - 1) / BN, splits);
    if (a_mn && b_mn) net_gemm_kernel<1, 1><<<grid, kThreads, kSmemBytes, st>>>(P);
    else if (a_mn) net_gemm_kernel<1, 0><<<grid, kThreads, kSmemBytes, st>>>(P);
    else if (b_mn) net_gemm_kernel<0, 1><<<grid, kThreads, kSmemBytes, st>>>(P);
    else net_gemm_kernel<0, 0><<<grid, kThreads, kSmemBytes, st>>>(P);
    if (check_launch("ts_net_gemm")) return 1;
    if (splits > 1) {
        const int64_t total = (int64_t)M * N;
        splitk_reduce_kernel<<<(unsigned)imin((total + 255) / 256, num_sms() * 8), 256, 0, st>>>(workspace, splits, c, ldc, M, N, bias, act,
                                                                                           mask, ld_mask, mask_kind, accumulate);
        if (check_launch("ts_net_gemm/splitk")) return 1;
    }
    return 0;
}

int net_colsum(const float* x, int64_t ld, int M, int N, float* out, int accumulate, cudaStream_t st) {
    if (N <= 0) return 0;
    colsum_kernel<<<(N + 31) / 32, 256, 0, st>>>(x, ld, M, N, out, accumulate);
    return check_launch("ts_net_colsum");
}

}  // namespace tsb

extern "C" int ts_net_gemm(const float* a, int64_t lda, int32_t a_mn_major, const float* b, int64_t ldb, int32_t b_mn_major,
                           float* c, int64_t ldc, int32_t M, int32_t N, int32_t K, const float* bias, int32_t act,
                           const float* act_grad_src, int64_t ld_mask, int32_t act_grad_kind, int32_t accumulate, float* workspace,
                           int64_t workspace_floats, ts_stream_t stream) {
    TS_REQUIRE(a && b && c && M >= 0 && N >= 0 && K >= 0, "ts_net_gemm: null pointer / negative size");
    TS_REQUIRE(act >= TS_ACT_NONE && act <= TS_ACT_TANH, "ts_net_gemm: unknown activation %d", act);
    TS_REQUIRE(!act_grad_src || act_grad_kind == TS_ACT_RELU || act_grad_kind == TS_ACT_TANH, "ts_net_gemm: unknown act_grad_kind %d", act_grad_kind);
    return tsb::net_gemm(a, lda, a_mn_major, b, ldb, b_mn_major, c, ldc, M, N, K, bias, act, act_grad_src, ld_mask, act_grad_kind, accumulate,
                         workspace, (size_t)(workspace_floats > 0 ? workspace_floats : 0), tsb::as_stream(stream));
}

extern "C" int64_t ts_net_gemm_workspace_floats(int32_t M, int32_t N, int32_t K) {
    return (int64_t)tsb::net_gemm_workspace_floats(M, N, K, nullptr);
}

extern "C" int ts_net_colsum(const float* x, int64_t ld, int32_t M, int32_t N, float* out, int32_t accumulate, ts_stream_t stream) {
    TS_REQUIRE(x && out, "ts_net_colsum: null pointer");
    return tsb::net_colsum(x, ld, M, N, out, accumulate, tsb::as_stream(stream));
}
