// Hopper (sm_90a) tensor-core, mbarrier and bulk-copy primitives (inline PTX), plus the shared-memory operand
// layout used by every tensor-core GEMM in this library.
//
// Operand layout ("blocked", no swizzle).  A matrix X[R][C] of 16-bit elements (R % 8 == 0, C % 8 == 0) is stored
// as 8-row x 8-column "core matrices" of 128 contiguous bytes:
//     byte_off(r, c) = (r / 8) * RS + (c / 8) * 128 + (r % 8) * 16 + (c % 8) * 2
// A wgmma shared-memory descriptor (no swizzle) names the byte stride between core matrices along K (LBO) and
// along M / N (SBO):
//   * used K-major  (rows = M or N index, cols = K):  LBO = 128, SBO = RS; one K = 16 step = 2 core matrices, the
//     next step starts 256 bytes further.
//   * used MN-major (rows = K index, cols = M or N):  LBO = RS, SBO = 128; one K = 16 step = 2 row groups, the next
//     step starts 2 * RS further.  (wgmma transposes 16-bit operands itself: imm-trans-a / imm-trans-b = 1.)
// So one copy of an activation / weight matrix in shared memory serves the forward GEMM (K-major), the
// weight-gradient GEMM (MN-major, reduction over rows) and the input-gradient GEMM.
//
// bf16x3: x = b0 + b1 + b2 with three bf16 pieces (24 significant bits); the six partial products of weight
// >= 2^-16 accumulated in fp32 give fp32-faithful products from bf16 tensor-core MMAs.
//
// Accumulators live in registers (wgmma.mma_async, one warpgroup = 128 threads computes a 64 x N tile).  Thread
// t of the warpgroup (warp w = t / 32, lane l) holds, for column block i (8 columns) and j in 0..3,
//     d[4 i + j] = D[16 w + l / 4 + 8 (j >> 1)][8 i + 2 (l % 4) + (j & 1)]                  (frag_row / frag_col)
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace wg {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// row / column of accumulator element e of the calling thread within its warpgroup's 64 x N tile
__device__ __forceinline__ int frag_row(int e) { return 16 * ((threadIdx.x >> 5) & 3) + ((threadIdx.x & 31) >> 2) + 8 * ((e >> 1) & 1); }
__device__ __forceinline__ int frag_col(int e) { return 8 * (e >> 2) + 2 * (threadIdx.x & 3) + (e & 1); }

// ---- descriptors ------------------------------------------------------------------------------
// 64-bit shared-memory matrix descriptor, no swizzle: lo32 = (addr >> 4) | (LBO >> 4) << 16 ; hi32 = SBO >> 4
__device__ __forceinline__ uint32_t desc_lo(uint32_t saddr, uint32_t lbo) { return ((saddr >> 4) & 0x3FFFu) | (((lbo >> 4) & 0x3FFFu) << 16); }
__device__ __forceinline__ uint32_t desc_hi(uint32_t sbo) { return (sbo >> 4) & 0x3FFFu; }
__device__ __forceinline__ uint64_t desc_pack(uint32_t lo, uint32_t hi) { return (uint64_t)lo | ((uint64_t)hi << 32); }

// ---- wgmma ------------------------------------------------------------------------------------
// all four functions: every thread of the warpgroup, converged
__device__ __forceinline__ void fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// D[64 x N] (+)= A * B, A and B from shared memory (descriptors); TA / TB = 1: operand used MN-major
template <int N, int TA, int TB>
__device__ __forceinline__ void mma(float (&d)[N / 2], uint64_t a, uint64_t b, uint32_t scale_d) {
    if constexpr (N == 8) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %6, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n8k16.f32.bf16.bf16 {"
            "%0, %1, %2, %3"
            "}, %4, %5, p, 1, 1, %7, %8;\n\t}"
          : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
          : "l"(a), "l"(b), "r"(scale_d), "n"(TA), "n"(TB));
    } else if constexpr (N == 16) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {"
            "%0, %1, %2, %3, %4, %5, %6, %7"
            "}, %8, %9, p, 1, 1, %11, %12;\n\t}"
          : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
          : "l"(a), "l"(b), "r"(scale_d), "n"(TA), "n"(TB));
    } else if constexpr (N == 24) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %14, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n24k16.f32.bf16.bf16 {"
            "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11"
            "}, %12, %13, p, 1, 1, %15, %16;\n\t}"
          : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11])
          : "l"(a), "l"(b), "r"(scale_d), "n"(TA), "n"(TB));
    } else if constexpr (N == 32) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {"
            "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15"
            "}, %16, %17, p, 1, 1, %19, %20;\n\t}"
          : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
          : "l"(a), "l"(b), "r"(scale_d), "n"(TA), "n"(TB));
    } else if constexpr (N == 40) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %22, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n40k16.f32.bf16.bf16 {"
            "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
            "%16, %17, %18, %19"
            "}, %20, %21, p, 1, 1, %23, %24;\n\t}"
          : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19])
          : "l"(a), "l"(b), "r"(scale_d), "n"(TA), "n"(TB));
    } else if constexpr (N == 128) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {"
            "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
            "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
            "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
            "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
            "}, %64, %65, p, 1, 1, %67, %68;\n\t}"
          : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
          : "l"(a), "l"(b), "r"(scale_d), "n"(TA), "n"(TB));
    }

}

// make generic-proxy shared-memory writes visible to the async proxy (wgmma operand reads, bulk copies)
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// orders generic-proxy accesses (any state space) against later async-proxy accesses
__device__ __forceinline__ void fence_proxy_async_all() { asm volatile("fence.proxy.async;" ::: "memory"); }

// fp32-faithful D[64 x N] (+)= A * B from three bf16 pieces per operand over KSTEPS K = 16 steps.  Piece p of an
// operand lives p * *_part bytes after piece 0; *_step = bytes to the next K step.  FULL = false: three products
// only -- A0 B0 + A1 B0 + A0 B1 (relative error ~2^-16 per term instead of ~2^-22): the weight-gradient GEMMs.
// Issues the MMAs only (no fence / commit / wait).
template <int N, int KSTEPS, int TA, int TB, bool FULL = true>
__device__ __forceinline__ void gemm_bf16x3(float (&d)[N / 2], uint32_t a0, uint32_t a_part, uint32_t a_lbo, uint32_t a_sbo,
                                            uint32_t a_step, uint32_t b0, uint32_t b_part, uint32_t b_lbo, uint32_t b_sbo,
                                            uint32_t b_step, bool accumulate) {
    const uint32_t ahi = desc_hi(a_sbo), bhi = desc_hi(b_sbo);
    uint32_t alo[3], blo[3];
#pragma unroll
    for (int p = 0; p < 3; ++p) {
        alo[p] = desc_lo(a0 + p * a_part, a_lbo);
        blo[p] = desc_lo(b0 + p * b_part, b_lbo);
    }
    const uint32_t astep = a_step >> 4, bstep = b_step >> 4;
#pragma unroll
    for (int k = 0; k < KSTEPS; ++k) {
        uint64_t A[3], B[3];
#pragma unroll
        for (int p = 0; p < 3; ++p) {
            A[p] = desc_pack(alo[p] + k * astep, ahi);
            B[p] = desc_pack(blo[p] + k * bstep, bhi);
        }
        const uint32_t first = (k == 0 && !accumulate) ? 0u : 1u;
        // smallest terms first; pairs (i, j) with i + j <= 2
        if (FULL) {
            mma<N, TA, TB>(d, A[2], B[0], first);
            mma<N, TA, TB>(d, A[0], B[2], 1u);
            mma<N, TA, TB>(d, A[1], B[1], 1u);
            mma<N, TA, TB>(d, A[1], B[0], 1u);
        } else {
            mma<N, TA, TB>(d, A[1], B[0], first);
        }
        mma<N, TA, TB>(d, A[0], B[1], 1u);
        mma<N, TA, TB>(d, A[0], B[0], 1u);
    }
}

// ---- mbarrier / bulk copy ---------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* mbar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(mbar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_wait(uint64_t* mbar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra.uni WAIT_DONE;\n\t"
        "bra.uni WAIT_LOOP;\n\t"
        "WAIT_DONE:\n\t}"
        ::"r"(smem_u32(mbar)), "r"(parity) : "memory");
}
// transaction-count arrive + 1-D bulk copy global -> shared (TMA engine, completes on the mbarrier)
__device__ __forceinline__ void mbar_expect_tx(uint64_t* mbar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(mbar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t smem_dst, const void* gsrc, uint32_t bytes, uint64_t* mbar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_dst), "l"(gsrc), "r"(bytes), "r"(smem_u32(mbar)) : "memory");
}

}  // namespace wg
