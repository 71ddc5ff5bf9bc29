// Replay-buffer index kernels (bit-exact int64) and row gathers, sm_90a.
//
// Reference semantics (all under tianshou/data/buffer/):
//   numba _next_index / _prev_index        manager.py:339-363 / :311-336
//   ReplayBuffer.next / prev               buffer_base.py:319-334   (the E = 1 case)
//   unfinished_index                       manager.py:85-91, buffer_base.py:314-317
//   sample_indices(0)                      manager.py:217-234, buffer_base.py:519-525
// The reference loops over ALL sub-buffers with a boolean mask per index batch (O(E * n)); here
// each index finds its owner by binary search over the E+1 edges (O(n log E)), one thread per
// index, coalesced 8-byte loads/stores; `done` is a random 1-byte gather (latency bound).
#include "common.cuh"

namespace {

using tsb::find_subbuffer;
using tsb::pymod;

struct BufMeta {
    const int64_t* offset;  // E+1 edges
    int64_t E;
    const uint8_t* done;
    const int64_t* last_index;
    const int64_t* lengths;
};

__device__ __forceinline__ int64_t next_one(const BufMeta& m, int64_t i) {
    const int64_t total = __ldg(m.offset + m.E);
    i = pymod(i, total);                               // manager.py:347
    const int64_t e = find_subbuffer(m.offset, m.E, i);
    const int64_t start = __ldg(m.offset + e);
    int64_t len = __ldg(m.lengths + e);
    if (len < 1) len = 1;                              // max(1, cur_len), :357
    const int64_t last = __ldg(m.last_index + e);
    const int64_t end_flag = (m.done[i] != 0) | (i == last);
    return pymod(i - start + 1 - end_flag, len) + start;  // :362
}

__device__ __forceinline__ int64_t prev_one(const BufMeta& m, int64_t i) {
    const int64_t total = __ldg(m.offset + m.E);
    i = pymod(i, total);                               // manager.py:319
    const int64_t e = find_subbuffer(m.offset, m.E, i);
    const int64_t start = __ldg(m.offset + e);
    int64_t len = __ldg(m.lengths + e);
    if (len < 1) len = 1;
    const int64_t last = __ldg(m.last_index + e);
    const int64_t sub = pymod(i - start - 1, len);     // :333
    const int64_t end_flag = (m.done[sub + start] != 0) | (sub + start == last);
    return pymod(sub + end_flag, len) + start;         // :335
}

template <bool kNext>
__global__ void step_index_kernel(BufMeta m, const int64_t* __restrict__ index, int64_t n,
                                  int64_t* __restrict__ out) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    out[t] = kNext ? next_one(m, index[t]) : prev_one(m, index[t]);
}

__global__ void stack_next_kernel(BufMeta m, const int64_t* __restrict__ index, int64_t n,
                                  int n_step, int64_t* __restrict__ out) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    int64_t i = index[t];
    out[t] = i;                                         // row 0 is the raw index (not wrapped)
    for (int k = 1; k < n_step; ++k) {
        i = next_one(m, i);
        out[(int64_t)k * n + t] = i;
    }
}

// Single CTA: ordered compaction over the E sub-buffers.
__global__ void __launch_bounds__(1024) unfinished_kernel(BufMeta m, const int64_t* __restrict__ ins_idx /* nullable */,
                                                          int64_t* __restrict__ out, int64_t* __restrict__ count_out) {
    __shared__ int s_warp[32];
    __shared__ int64_t s_base;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) s_base = 0;
    __syncthreads();
    for (int64_t e0 = 0; e0 < m.E; e0 += blockDim.x) {
        const int64_t e = e0 + tid;
        int64_t last = 0;
        int keep = 0;
        if (e < m.E && m.lengths[e] > 0) {
            // buffer_base.py:314-317: the slot BEFORE the insertion index (== last_index for buffers filled by add();
            // from_data() / dropnull() move the insertion index without touching last_index)
            last = ins_idx ? m.offset[e] + tsb::pymod(ins_idx[e] - 1, m.lengths[e]) : m.last_index[e];
            keep = (m.done[last] == 0);
        }
        const unsigned bal = __ballot_sync(0xffffffffu, keep);
        const int within = __popc(bal & ((1u << lane) - 1u));
        if (lane == 0) s_warp[warp] = __popc(bal);
        __syncthreads();
        int before = 0, total = 0;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) {
            if (w < warp) before += s_warp[w];
            total += s_warp[w];
        }
        if (keep) out[s_base + before + within] = last;
        __syncthreads();
        if (tid == 0) s_base += total;
        __syncthreads();
    }
    if (tid == 0) *count_out = s_base;
}

// Single CTA exclusive scan of lengths -> seg_start[0..E], total.
__global__ void __launch_bounds__(1024) seg_start_kernel(const int64_t* __restrict__ lengths,
                                                         int64_t E, int64_t* __restrict__ seg_start,
                                                         int64_t* __restrict__ total_out) {
    __shared__ int64_t s_warp[32];
    __shared__ int64_t s_base;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) s_base = 0;
    __syncthreads();
    for (int64_t e0 = 0; e0 < E; e0 += blockDim.x) {
        const int64_t e = e0 + tid;
        const int64_t v = e < E ? lengths[e] : 0;
        int64_t inc = v;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
            const int64_t o = __shfl_up_sync(0xffffffffu, inc, off);
            if (lane >= off) inc += o;
        }
        if (lane == 31) s_warp[warp] = inc;
        __syncthreads();
        int64_t before = 0, total = 0;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) {
            if (w < warp) before += s_warp[w];
            total += s_warp[w];
        }
        if (e < E) seg_start[e] = s_base + before + inc - v;
        __syncthreads();
        if (tid == 0) s_base += total;
        __syncthreads();
    }
    if (tid == 0) { seg_start[E] = s_base; *total_out = s_base; }
}

__global__ void sample_all_kernel(const int64_t* __restrict__ offset, int64_t E,
                                  const int64_t* __restrict__ last_index,
                                  const int64_t* __restrict__ lengths,
                                  const int64_t* __restrict__ ins_idx /* nullable */,
                                  const int64_t* __restrict__ seg_start, int64_t* __restrict__ out,
                                  int64_t capacity) {
    const int64_t total = seg_start[E];
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < total && p < capacity;
         p += (int64_t)gridDim.x * blockDim.x) {
        // owner: largest e with seg_start[e] <= p; empty sub-buffers share a start, the search
        // below lands on the last of them or on the non-empty one: advance to size > 0.
        int64_t lo = 0, hi = E;
        while (hi - lo > 1) {
            const int64_t mid = (lo + hi) >> 1;
            if (seg_start[mid] <= p) lo = mid; else hi = mid;
        }
        const int64_t e = lo;
        const int64_t j = p - seg_start[e];
        const int64_t size = lengths[e];
        const int64_t start = offset[e];
        const int64_t cap = offset[e + 1] - start;
        // child's _insertion_idx (buffer_base.py:519-525).  It is NOT always last_index + 1: from_data() / dropnull()
        // / set_batch() leave last_index untouched, so the caller passes the buffer's own counter when it has one.
        const int64_t ins = ins_idx ? ins_idx[e] : (last_index[e] - start + 1) % cap;
        out[p] = start + (ins % size + j) % size;               // [ins..size) ++ [0..ins)  (ins == size: arange(size))
    }
}

__global__ void end_flags_kernel(const uint8_t* __restrict__ done, const int64_t* __restrict__ offset,
                                 const int64_t* __restrict__ last_index,
                                 const int64_t* __restrict__ lengths, int64_t E,
                                 uint8_t* __restrict__ out) {
    const int64_t B = offset[E];
    const int64_t nw = (B + 15) / 16;
    for (int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; w < nw;
         w += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i0 = w * 16;
        if (i0 + 16 <= B && ((reinterpret_cast<uintptr_t>(done) | reinterpret_cast<uintptr_t>(out)) & 15u) == 0) {
            *reinterpret_cast<uint4*>(out + i0) = *reinterpret_cast<const uint4*>(done + i0);
        } else {
            for (int64_t i = i0; i < B && i < i0 + 16; ++i) out[i] = done[i];
        }
    }
}
__global__ void end_flags_mark_kernel(const int64_t* __restrict__ last_index,
                                      const int64_t* __restrict__ lengths, int64_t E,
                                      uint8_t* __restrict__ out) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e < E && lengths[e] > 0) out[last_index[e]] = 1;
}

__global__ void value_mask_kernel(float* __restrict__ tq, const uint8_t* __restrict__ terminated,
                                  const int64_t* __restrict__ idx, int64_t I, int64_t A) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= I * A) return;
    const int64_t i = t / A;
    if (terminated[idx[i]]) tq[t] = tq[t] * 0.0f;  // `*= mask` keeps sign/NaN like numpy
}

__global__ void mark_set_kernel(const int64_t* __restrict__ members,
                                const int64_t* __restrict__ count, int64_t capacity,
                                uint8_t* __restrict__ table, int64_t table_size, uint8_t v) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t c = count ? *count : capacity;
    if (t < c && t < capacity) {
        const int64_t m = members[t];
        if (m >= 0 && m < table_size) table[m] = v;
    }
}
__global__ void mark_lookup_kernel(const int64_t* __restrict__ idx, int64_t n,
                                   const uint8_t* __restrict__ table, int64_t table_size,
                                   uint8_t* __restrict__ out) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    const int64_t i = idx[t];
    out[t] = (i >= 0 && i < table_size) ? table[i] : 0;
}

// dst[p][w] = src[idx[p]][w] over 4-byte words; one warp-coalesced pass, 16 B per thread when
// the row size allows.
template <typename W>
__global__ void gather_rows_kernel(const W* __restrict__ src, int64_t row_words,
                                   const int64_t* __restrict__ idx, int64_t n, W* __restrict__ dst) {
    const int64_t total = n * row_words;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total;
         t += (int64_t)gridDim.x * blockDim.x) {
        const int64_t p = t / row_words, w = t - p * row_words;
        dst[t] = src[idx[p] * row_words + w];
    }
}
// inverse: dst[idx[p]] = src[p] (device mirror of ReplayBuffer.add: rows staged contiguously, slots scattered)
template <typename W>
__global__ void scatter_rows_kernel(const W* __restrict__ src, int64_t row_words,
                                    const int64_t* __restrict__ idx, int64_t n, W* __restrict__ dst) {
    const int64_t total = n * row_words;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total;
         t += (int64_t)gridDim.x * blockDim.x) {
        const int64_t p = t / row_words, w = t - p * row_words;
        dst[idx[p] * row_words + w] = src[t];
    }
}
__global__ void gather_bytes_kernel(const uint8_t* __restrict__ src, const int64_t* __restrict__ idx,
                                    int64_t n, uint8_t* __restrict__ dst) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t < n) dst[t] = src[idx[t]];
}

__global__ void narrow_kernel(const int64_t* __restrict__ src, int64_t n, int32_t* __restrict__ dst) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t < n) dst[t] = (int32_t)src[t];
}

// ---- next-observation alias map ---------------------------------------------------------------------
// In a rollout obs_next[i] is obs[i + 1] except where an episode or an env's segment ends, so critic(obs_next[i]) is
// the value already computed for row i + 1.  alias[i] = 1 iff the two rows hold the same 32-bit words (a bitwise test:
// -0.0 vs 0.0 and different NaN payloads count as different, which only costs an evaluation); the rows with alias == 0
// are listed in ascending order in `extra`.  Nothing is assumed about the buffer layout: a shuffled batch lists every row.
constexpr int kAliasThreads = 256;      // rows per block: one warp compares 32 consecutive rows, coalesced over their words

__global__ void __launch_bounds__(kAliasThreads) next_alias_mark_kernel(
    const uint32_t* __restrict__ obs, const uint32_t* __restrict__ obs_next, int64_t n, int width,
    uint8_t* __restrict__ alias, int32_t* __restrict__ block_extra) {
    const int lane = threadIdx.x & 31;
    const int64_t i0 = (int64_t)blockIdx.x * kAliasThreads + (threadIdx.x & ~31);     // first row of the warp
    const int64_t rows = tsb::imin(32, n - 1 - i0);          // rows of the warp that have a successor (may be <= 0)
    const uint32_t* a = obs_next + i0 * width;
    const uint32_t* b = obs + (i0 + 1) * width;
    unsigned differs = 0u;                                   // bit r: row i0 + r differs in a word this lane compared
    for (int64_t w = lane; w < rows * width; w += 32) {
        if (a[w] != b[w]) differs |= 1u << (unsigned)(w / width);
    }
    differs = __reduce_or_sync(0xffffffffu, differs);
    const int64_t i = i0 + lane;
    const bool same = lane < rows && !((differs >> lane) & 1u);
    if (i < n) alias[i] = same ? 1 : 0;
    const int cnt = __syncthreads_count(i < n && !same);
    if (threadIdx.x == 0) block_extra[blockIdx.x] = cnt;
}

// Ordered compaction of the rows with alias == 0: a block's first slot is the sum of the earlier blocks' counts, the
// order inside a block comes from a ballot scan -- no atomics, so `extra` is the same list on every run.
__global__ void __launch_bounds__(kAliasThreads) next_alias_compact_kernel(
    const uint8_t* __restrict__ alias, int64_t n, const int32_t* __restrict__ block_extra,
    int32_t* __restrict__ extra, int32_t* __restrict__ n_extra) {
    __shared__ int s_warp[kAliasThreads / 32];
    __shared__ int s_base;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    int before_blocks = 0;
    for (int b = tid; b < (int)blockIdx.x; b += kAliasThreads) before_blocks += block_extra[b];
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) before_blocks += __shfl_xor_sync(0xffffffffu, before_blocks, off);
    if (lane == 0) s_warp[warp] = before_blocks;
    __syncthreads();
    if (tid == 0) {
        int base = 0;
        for (int w = 0; w < kAliasThreads / 32; ++w) base += s_warp[w];
        s_base = base;
    }
    __syncthreads();
    const int64_t i = (int64_t)blockIdx.x * kAliasThreads + tid;
    const bool keep = i < n && alias[i] == 0;
    const unsigned bal = __ballot_sync(0xffffffffu, keep);
    const int base = s_base;
    __syncthreads();                                          // s_warp is reused
    if (lane == 0) s_warp[warp] = __popc(bal);
    __syncthreads();
    int before = 0, total = 0;
    for (int w = 0; w < kAliasThreads / 32; ++w) {
        if (w < warp) before += s_warp[w];
        total += s_warp[w];
    }
    if (keep) extra[base + before + __popc(bal & ((1u << lane) - 1u))] = (int32_t)i;
    if (blockIdx.x == gridDim.x - 1 && tid == 0) *n_extra = base + total;
}

inline unsigned blocks_for(int64_t n, int threads) { return (unsigned)((n + threads - 1) / threads); }

}  // namespace

extern "C" int64_t ts_next_alias_workspace_bytes(int64_t n) {
    return n > 0 ? 4 * (int64_t)blocks_for(n, kAliasThreads) : 0;
}

extern "C" int ts_next_alias_map(const float* obs, const float* obs_next, int64_t n, int32_t obs_dim, uint8_t* alias,
                                 int32_t* extra, int32_t* n_extra, void* workspace, ts_stream_t stream) {
    TS_REQUIRE(n >= 0 && n < (1ll << 31) && obs_dim >= 1, "ts_next_alias_map: bad shape");
    TS_REQUIRE(n_extra, "ts_next_alias_map: null n_extra");
    cudaStream_t st = tsb::as_stream(stream);
    if (n == 0) {
        TS_CUDA(cudaMemsetAsync(n_extra, 0, sizeof(int32_t), st));
        return 0;
    }
    TS_REQUIRE(obs && obs_next && alias && extra && workspace, "ts_next_alias_map: null pointer");
    int32_t* block_extra = static_cast<int32_t*>(workspace);
    const unsigned grid = blocks_for(n, kAliasThreads);
    next_alias_mark_kernel<<<grid, kAliasThreads, 0, st>>>(reinterpret_cast<const uint32_t*>(obs),
                                                           reinterpret_cast<const uint32_t*>(obs_next), n, obs_dim, alias, block_extra);
    if (tsb::check_launch("ts_next_alias_map/mark")) return 1;
    next_alias_compact_kernel<<<grid, kAliasThreads, 0, st>>>(alias, n, block_extra, extra, n_extra);
    return tsb::check_launch("ts_next_alias_map");
}

#define META_ARGS_OK(fn) \
    TS_REQUIRE(offset && done && last_index && lengths && E > 0, fn ": null buffer metadata")

extern "C" int ts_next_index(const int64_t* index, int64_t n, const int64_t* offset, int64_t E,
                             const uint8_t* done, const int64_t* last_index,
                             const int64_t* lengths, int64_t* out, ts_stream_t stream) {
    if (n == 0) return 0;
    META_ARGS_OK("ts_next_index");
    TS_REQUIRE(index && out, "ts_next_index: null index/out");
    BufMeta m{offset, E, done, last_index, lengths};
    step_index_kernel<true><<<blocks_for(n, 256), 256, 0, tsb::as_stream(stream)>>>(m, index, n, out);
    return tsb::check_launch("ts_next_index");
}

extern "C" int ts_prev_index(const int64_t* index, int64_t n, const int64_t* offset, int64_t E,
                             const uint8_t* done, const int64_t* last_index,
                             const int64_t* lengths, int64_t* out, ts_stream_t stream) {
    if (n == 0) return 0;
    META_ARGS_OK("ts_prev_index");
    TS_REQUIRE(index && out, "ts_prev_index: null index/out");
    BufMeta m{offset, E, done, last_index, lengths};
    step_index_kernel<false><<<blocks_for(n, 256), 256, 0, tsb::as_stream(stream)>>>(m, index, n, out);
    return tsb::check_launch("ts_prev_index");
}

extern "C" int ts_stack_next_indices(const int64_t* index, int64_t n, int32_t n_step,
                                     const int64_t* offset, int64_t E, const uint8_t* done,
                                     const int64_t* last_index, const int64_t* lengths,
                                     int64_t* out, ts_stream_t stream) {
    TS_REQUIRE(n_step >= 1, "ts_stack_next_indices: n_step must be >= 1");
    if (n == 0) return 0;
    META_ARGS_OK("ts_stack_next_indices");
    TS_REQUIRE(index && out, "ts_stack_next_indices: null index/out");
    BufMeta m{offset, E, done, last_index, lengths};
    stack_next_kernel<<<blocks_for(n, 128), 128, 0, tsb::as_stream(stream)>>>(m, index, n, n_step, out);
    return tsb::check_launch("ts_stack_next_indices");
}

extern "C" int ts_unfinished_index(const int64_t* offset, int64_t E, const uint8_t* done,
                                   const int64_t* last_index, const int64_t* lengths, const int64_t* insertion_idx,
                                   int64_t* out, int64_t* count_out, ts_stream_t stream) {
    META_ARGS_OK("ts_unfinished_index");
    TS_REQUIRE(out && count_out, "ts_unfinished_index: null out");
    BufMeta m{offset, E, done, last_index, lengths};
    unfinished_kernel<<<1, 1024, 0, tsb::as_stream(stream)>>>(m, insertion_idx, out, count_out);
    return tsb::check_launch("ts_unfinished_index");
}

extern "C" int ts_sample_all_indices(const int64_t* offset, int64_t E, const int64_t* last_index,
                                     const int64_t* lengths, const int64_t* insertion_idx, int64_t* seg_start,
                                     int64_t* out, int64_t out_capacity, int64_t* total_out, ts_stream_t stream) {
    TS_REQUIRE(offset && last_index && lengths && seg_start && out && total_out && E > 0,
               "ts_sample_all_indices: null pointer");
    cudaStream_t st = tsb::as_stream(stream);
    seg_start_kernel<<<1, 1024, 0, st>>>(lengths, E, seg_start, total_out);
    if (tsb::check_launch("ts_sample_all_indices/scan")) return 1;
    if (out_capacity == 0) return 0;
    const unsigned grid = (unsigned)tsb::imin((int64_t)blocks_for(out_capacity, 256), tsb::num_sms() * 16);
    sample_all_kernel<<<grid, 256, 0, st>>>(offset, E, last_index, lengths, insertion_idx, seg_start, out, out_capacity);
    return tsb::check_launch("ts_sample_all_indices");
}

extern "C" int ts_buffer_end_flags(const uint8_t* done, const int64_t* offset,
                                   const int64_t* last_index, const int64_t* lengths, int64_t E,
                                   uint8_t* end_flag_out, ts_stream_t stream) {
    TS_REQUIRE(done && offset && last_index && lengths && end_flag_out && E > 0,
               "ts_buffer_end_flags: null pointer");
    cudaStream_t st = tsb::as_stream(stream);
    end_flags_kernel<<<tsb::num_sms() * 4, 256, 0, st>>>(done, offset, last_index, lengths, E, end_flag_out);
    if (tsb::check_launch("ts_buffer_end_flags/copy")) return 1;
    end_flags_mark_kernel<<<blocks_for(E, 256), 256, 0, st>>>(last_index, lengths, E, end_flag_out);
    return tsb::check_launch("ts_buffer_end_flags");
}

extern "C" int ts_value_mask_rows(float* target_q, const uint8_t* terminated, const int64_t* idx,
                                  int64_t I, int64_t A, ts_stream_t stream) {
    if (I * A == 0) return 0;
    TS_REQUIRE(target_q && terminated && idx, "ts_value_mask_rows: null pointer");
    value_mask_kernel<<<blocks_for(I * A, 256), 256, 0, tsb::as_stream(stream)>>>(target_q, terminated, idx, I, A);
    return tsb::check_launch("ts_value_mask_rows");
}

extern "C" int ts_mark_members(const int64_t* idx, int64_t n, const int64_t* members,
                               const int64_t* member_count, int64_t member_capacity, uint8_t* table,
                               int64_t table_size, uint8_t* mark_out, ts_stream_t stream) {
    if (n == 0) return 0;
    TS_REQUIRE(idx && table && mark_out, "ts_mark_members: null pointer");
    cudaStream_t st = tsb::as_stream(stream);
    if (member_capacity > 0) {
        TS_REQUIRE(members, "ts_mark_members: null members");
        mark_set_kernel<<<blocks_for(member_capacity, 256), 256, 0, st>>>(members, member_count, member_capacity, table, table_size, 1);
        if (tsb::check_launch("ts_mark_members/set")) return 1;
    }
    mark_lookup_kernel<<<blocks_for(n, 256), 256, 0, st>>>(idx, n, table, table_size, mark_out);
    if (tsb::check_launch("ts_mark_members/lookup")) return 1;
    if (member_capacity > 0) {
        mark_set_kernel<<<blocks_for(member_capacity, 256), 256, 0, st>>>(members, member_count, member_capacity, table, table_size, 0);
        if (tsb::check_launch("ts_mark_members/clear")) return 1;
    }
    return 0;
}

extern "C" int ts_gather_rows(const void* src, int64_t row_bytes, const int64_t* idx, int64_t n,
                              void* dst, ts_stream_t stream) {
    if (n == 0 || row_bytes == 0) return 0;
    TS_REQUIRE(src && idx && dst, "ts_gather_rows: null pointer");
    cudaStream_t st = tsb::as_stream(stream);
    const bool a16 = ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15u) == 0;
    if (row_bytes % 16 == 0 && a16) {
        const int64_t rw = row_bytes / 16;
        const unsigned grid = (unsigned)tsb::imin((int64_t)blocks_for(n * rw, 256), tsb::num_sms() * 32);
        gather_rows_kernel<uint4><<<grid, 256, 0, st>>>(static_cast<const uint4*>(src), rw, idx, n, static_cast<uint4*>(dst));
    } else if (row_bytes % 4 == 0 && (((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 3u) == 0)) {
        const int64_t rw = row_bytes / 4;
        const unsigned grid = (unsigned)tsb::imin((int64_t)blocks_for(n * rw, 256), tsb::num_sms() * 32);
        gather_rows_kernel<uint32_t><<<grid, 256, 0, st>>>(static_cast<const uint32_t*>(src), rw, idx, n, static_cast<uint32_t*>(dst));
    } else if (row_bytes == 1) {
        gather_bytes_kernel<<<blocks_for(n, 256), 256, 0, st>>>(static_cast<const uint8_t*>(src), idx, n, static_cast<uint8_t*>(dst));
    } else {
        const unsigned grid = (unsigned)tsb::imin((int64_t)blocks_for(n * row_bytes, 256), tsb::num_sms() * 32);
        gather_rows_kernel<uint8_t><<<grid, 256, 0, st>>>(static_cast<const uint8_t*>(src), row_bytes, idx, n, static_cast<uint8_t*>(dst));
    }
    return tsb::check_launch("ts_gather_rows");
}

extern "C" int ts_scatter_rows(const void* src, int64_t row_bytes, const int64_t* idx, int64_t n,
                               void* dst, ts_stream_t stream) {
    if (n == 0 || row_bytes == 0) return 0;
    TS_REQUIRE(src && idx && dst, "ts_scatter_rows: null pointer");
    cudaStream_t st = tsb::as_stream(stream);
    const bool a16 = ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15u) == 0;
    if (row_bytes % 16 == 0 && a16) {
        const int64_t rw = row_bytes / 16;
        const unsigned grid = (unsigned)tsb::imin((int64_t)blocks_for(n * rw, 256), tsb::num_sms() * 32);
        scatter_rows_kernel<uint4><<<grid, 256, 0, st>>>(static_cast<const uint4*>(src), rw, idx, n, static_cast<uint4*>(dst));
    } else if (row_bytes % 4 == 0 && (((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 3u) == 0)) {
        const int64_t rw = row_bytes / 4;
        const unsigned grid = (unsigned)tsb::imin((int64_t)blocks_for(n * rw, 256), tsb::num_sms() * 32);
        scatter_rows_kernel<uint32_t><<<grid, 256, 0, st>>>(static_cast<const uint32_t*>(src), rw, idx, n, static_cast<uint32_t*>(dst));
    } else {
        const unsigned grid = (unsigned)tsb::imin((int64_t)blocks_for(n * row_bytes, 256), tsb::num_sms() * 32);
        scatter_rows_kernel<uint8_t><<<grid, 256, 0, st>>>(static_cast<const uint8_t*>(src), row_bytes, idx, n, static_cast<uint8_t*>(dst));
    }
    return tsb::check_launch("ts_scatter_rows");
}

extern "C" int ts_narrow_i64_i32(const int64_t* src, int64_t n, int32_t* dst, ts_stream_t stream) {
    if (n == 0) return 0;
    TS_REQUIRE(src && dst, "ts_narrow_i64_i32: null pointer");
    narrow_kernel<<<blocks_for(n, 256), 256, 0, tsb::as_stream(stream)>>>(src, n, dst);
    return tsb::check_launch("ts_narrow_i64_i32");
}
