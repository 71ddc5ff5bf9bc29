// Shared helpers for the ts_b200 kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/ts_b200.h"

namespace tsb {

void set_error(const char* fmt, ...);
void count_launch(int n = 1);

// Peer exchange of the multi-GPU fused update (one process per GPU, buffers shared through CUDA IPC).
// Every rank owns one exchange buffer:  [256-byte header: uint32 seq][world][2][width] 8-byte packets.
// A packet is (fp32 value, uint32 sequence number) written with ONE 8-byte store by the producing rank
// directly into the consumer's buffer over NVLink; the consumer polls the sequence half (no fences, no
// separate flags: the NCCL "LL" idea).  Slot parity = seq & 1.
constexpr int kMaxPeers = 8;
struct PeerArgs {
    int rank = 0, world = 1;
    unsigned long long* recv[kMaxPeers] = {};   // packet areas of every rank's buffer (device pointers valid on THIS device)
    unsigned int* hdr = nullptr;                // this rank's header (sequence number of the last completed step)
};
constexpr size_t kPeerHeaderBytes = 256;

inline int check_launch(const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
        set_error("%s: %s", what, cudaGetErrorString(e));
        return 1;
    }
    count_launch();
    return 0;
}

#define TS_REQUIRE(cond, ...)        \
    do {                             \
        if (!(cond)) {               \
            tsb::set_error(__VA_ARGS__); \
            return 2;                \
        }                            \
    } while (0)

#define TS_CUDA(call)                                                        \
    do {                                                                     \
        cudaError_t e_ = (call);                                             \
        if (e_ != cudaSuccess) {                                             \
            tsb::set_error("%s failed: %s", #call, cudaGetErrorString(e_)); \
            return 1;                                                        \
        }                                                                    \
    } while (0)

inline cudaStream_t as_stream(ts_stream_t s) { return reinterpret_cast<cudaStream_t>(s); }

constexpr int kMaxDevices = 64;
int device_ordinal();   // cudaGetDevice(), clamped to [0, kMaxDevices): key of per-device one-time setup caches
int num_sms();

__host__ __device__ inline int64_t imin(int64_t a, int64_t b) { return a < b ? a : b; }

__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }
__device__ __forceinline__ int warp_id() { return threadIdx.x >> 5; }

__device__ __forceinline__ double shfl_down_f64(double v, int d) {
    return __shfl_down_sync(0xffffffffu, v, d);
}
__device__ __forceinline__ double shfl_xor_f64(double v, int d) {
    return __shfl_xor_sync(0xffffffffu, v, d);
}

// floor-mod for possibly negative a, positive m (python semantics)
__device__ __forceinline__ int64_t pymod(int64_t a, int64_t m) {
    int64_t r = a % m;
    return r < 0 ? r + m : r;
}

// largest e in [0, E) with offset[e] <= i   (offset is ascending, offset[0] <= i < offset[E])
__device__ __forceinline__ int64_t find_subbuffer(const int64_t* __restrict__ offset, int64_t E,
                                                  int64_t i) {
    int64_t lo = 0, hi = E;  // invariant: offset[lo] <= i < offset[hi]
    while (hi - lo > 1) {
        int64_t mid = (lo + hi) >> 1;
        if (__ldg(offset + mid) <= i) lo = mid; else hi = mid;
    }
    return lo;
}

}  // namespace tsb
