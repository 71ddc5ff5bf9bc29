// Hardware self-test of the tensor-core building blocks in wgmma.cuh.  One CTA computes
//     D[M x N] = A[M x K] * B[N x K]^T           (a, b given row-major in global memory)
// with the 3-way bf16 split (6 wgmma per K = 16 step), M in {64, 128} (one warpgroup per 64 rows), each operand
// placed in shared memory either K-major or MN-major (blocked no-swizzle layout, see wgmma.cuh), and writes D
// row-major from the register accumulators.  B is padded with zero rows to N = 128.
#include <cuda_bf16.h>

#include "common.cuh"
#include "wgmma.cuh"

namespace {

constexpr int kThreads = 256, kN = 128;

template <int TA, int TB>
__global__ void __launch_bounds__(kThreads, 1) wgmma_selftest_kernel(const float* __restrict__ a, const float* __restrict__ b,
                                                                    float* __restrict__ d, int M, int N, int K, int swap) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int tid = threadIdx.x, wgi = tid >> 7;
    // operand X (logical [MN x K], MN rows valid) is stored as a matrix with rows = (major ? K : MN), cols = the other
    auto place = [&](const float* src, int MN, int MN_pad, int mn_major, uint8_t* base, uint32_t& RS, uint32_t& bytes) {
        const int rows = mn_major ? K : MN_pad, cols = mn_major ? MN_pad : K;
        RS = (uint32_t)(cols / 8) * 128; bytes = (uint32_t)rows * cols * 2;
        for (int e = tid; e < MN_pad * K; e += kThreads) {
            const int mn = e / K, k = e % K;
            const int r = mn_major ? k : mn, c = mn_major ? mn : k;
            const uint32_t off = (uint32_t)(r >> 3) * RS + (uint32_t)(c / 8) * 128 + (uint32_t)(r & 7) * 16 + (uint32_t)(c % 8) * 2;
            const float x = mn < MN ? src[mn * K + k] : 0.0f;
            const __nv_bfloat16 b0 = __float2bfloat16_rn(x);
            const float r1 = x - __bfloat162float(b0);
            const __nv_bfloat16 b1 = __float2bfloat16_rn(r1);
            const __nv_bfloat16 b2 = __float2bfloat16_rn(r1 - __bfloat162float(b1));
            *reinterpret_cast<__nv_bfloat16*>(base + off) = b0;
            *reinterpret_cast<__nv_bfloat16*>(base + bytes + off) = b1;
            *reinterpret_cast<__nv_bfloat16*>(base + 2 * bytes + off) = b2;
        }
    };
    uint32_t aRS, aB, bRS, bB;
    uint8_t* a_base = smem;
    place(a, M, M, TA, a_base, aRS, aB);
    uint8_t* b_base = a_base + 3 * (size_t)aB;
    place(b, N, kN, TB, b_base, bRS, bB);
    wg::fence_async_smem();
    __syncthreads();
    if (64 * wgi >= M) return;                  // warpgroup-uniform
    auto strides = [&](int mn_major, uint32_t RS, uint32_t& lbo, uint32_t& sbo, uint32_t& step) {
        if (!mn_major) { lbo = 128; sbo = RS; step = 256; }       // K-major: 2 chunks of 16 B per MMA
        else { lbo = RS; sbo = 128; step = 2 * RS; }               // MN-major: 2 row groups per MMA
        if (swap) { const uint32_t t = lbo; lbo = sbo; sbo = t; }
    };
    uint32_t albo, asbo, astep, blbo, bsbo, bstep;
    strides(TA, aRS, albo, asbo, astep);
    strides(TB, bRS, blbo, bsbo, bstep);
    const uint32_t A0 = wg::smem_u32(a_base) + 8u * (TA ? 128u : aRS) * (uint32_t)wgi, B0 = wg::smem_u32(b_base);
    float acc[kN / 2];
    wg::fence();
    for (int k = 0; k < K / 16; ++k)
        wg::gemm_bf16x3<kN, 1, TA, TB>(acc, A0 + k * astep, aB, albo, asbo, astep, B0 + k * bstep, bB, blbo, bsbo, bstep, k > 0);
    wg::commit();
    wg::wait<0>();
    for (int e = 0; e < kN / 2; ++e) {
        const int m = 64 * wgi + wg::frag_row(e), n = wg::frag_col(e);
        if (n < N) d[m * N + n] = acc[e];
    }
}

}  // namespace

extern "C" int ts_umma_selftest(const float* a, const float* b, float* d, int32_t M, int32_t N, int32_t K,
                                int32_t dtype, int32_t a_mn, int32_t b_mn, int32_t swap, ts_stream_t stream) {
    TS_REQUIRE(a && b && d, "ts_umma_selftest: null pointer");
    TS_REQUIRE(dtype == 1, "ts_umma_selftest: only the bf16x3 split (dtype 1) exists on this architecture");
    TS_REQUIRE(M == 64 || M == 128, "ts_umma_selftest: M must be 64 or 128");
    TS_REQUIRE(N % 8 == 0 && N >= 8 && N <= kN && K % 16 == 0 && K >= 16 && K <= 128, "ts_umma_selftest: bad N/K");
    TS_REQUIRE((a_mn == 0 || a_mn == 1) && (b_mn == 0 || b_mn == 1), "ts_umma_selftest: operands are K-major (0) or MN-major (1)");
    const size_t smem = (size_t)6 * (size_t)(M * K + kN * K);
    auto kern = a_mn ? (b_mn ? wgmma_selftest_kernel<1, 1> : wgmma_selftest_kernel<1, 0>)
                     : (b_mn ? wgmma_selftest_kernel<0, 1> : wgmma_selftest_kernel<0, 0>);
    TS_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<1, kThreads, smem, tsb::as_stream(stream)>>>(a, b, d, M, N, K, swap);
    return tsb::check_launch("ts_umma_selftest");
}
