// Sum tree for prioritized experience replay (f64 tree resident in HBM), sm_90a.
//
// Reference: tianshou/data/utils/segtree.py (numba `_setitem` :95-101, `_reduce` :104-116,
// `_get_prefix_sum_idx` :119-134) and tianshou/data/buffer/prio.py (:46-47,:63-90,:104-106).
// Layout: tree[1] = root, children of k are 2k and 2k+1, leaves at [bound, 2*bound).
// Every sum is the same single f64 addition `left + right` as the reference, so tree contents --
// and therefore the sampled indices -- are bit-identical.
//
// setitem runs in ONE CTA: phase 0 resolves duplicate indices ("last write wins", numpy fancy
// assignment), phase 1 writes leaves, then log2(bound) levels separated by __syncthreads; every
// thread owns batch items k, k+T, ... and recomputes its ancestor at each level (siblings that
// share an ancestor write the same value).  Batches are a few hundred indices (32..256 per
// update, #envs per add) over a 2^20..2^22-leaf tree, so the work is latency- not bandwidth-bound.
// The prefix-sum descent is one thread per query: log2(bound) dependent 8-byte loads; the top
// ~15 levels of the tree stay L2-resident.
#include <type_traits>

#include "common.cuh"

namespace {

constexpr int kSetThreads = 1024;

template <typename TV>
__global__ void __launch_bounds__(kSetThreads) setitem_kernel(
    double* __restrict__ tree, int64_t bound, const int64_t* __restrict__ index,
    const TV* __restrict__ value, int64_t n, double alpha, double eps, int prio_mode,
    double* __restrict__ prio_minmax) {
    const int tid = threadIdx.x;
    __shared__ double s_max[32], s_min[32];
    // ---- leaves: last occurrence of an index wins (numpy fancy assignment) -------------------
    // The leaf slot itself is the scratch: (1) zero it, (2) atomicMax of k+1 as u64, (3) the
    // item whose k+1 survived writes its value.  O(n), three CTA barriers.
    unsigned long long* slots = reinterpret_cast<unsigned long long*>(tree);
    for (int64_t k = tid; k < n; k += kSetThreads) slots[bound + index[k]] = 0ull;
    __syncthreads();
    for (int64_t k = tid; k < n; k += kSetThreads)
        atomicMax(slots + bound + index[k], (unsigned long long)(k + 1));
    __syncthreads();
    double lmax = -1.0e300, lmin = 1.0e300;
    // winners are decided before anyone overwrites a slot with a value
    unsigned win_mask = 0;  // bit j: item tid + j*kSetThreads wins (first 32 items per thread)
    {
        int j = 0;
        for (int64_t k = tid; k < n; k += kSetThreads, ++j) {
            const bool win = (slots[bound + index[k]] == (unsigned long long)(k + 1));
            if (j < 32) { if (win) win_mask |= (1u << j); }
        }
    }
    __syncthreads();
    {
        int j = 0;
        for (int64_t k = tid; k < n; k += kSetThreads, ++j) {
            double v = (double)value[k];
            if (prio_mode) {          // prio.py:82-85: w = |td| + eps ; tree = w ** alpha
                if constexpr (std::is_same_v<TV, float>) {
                    // numpy keeps a float32 array combined with a Python float in float32: eps and alpha are
                    // rounded to float32, |td| + eps and the power are float32 operations, the tree widens after
                    const float w = fabsf(value[k]) + (float)eps;
                    lmax = fmax(lmax, (double)w);
                    lmin = fmin(lmin, (double)w);
                    v = (double)powf(w, (float)alpha);
                } else {
                    v = fabs(v) + eps;
                    lmax = fmax(lmax, v);
                    lmin = fmin(lmin, v);
                    v = pow(v, alpha);
                }
            }
            if ((win_mask >> j) & 1u) tree[bound + index[k]] = v;
        }
    }
    __syncthreads();
    // ---- parents, bottom-up: level l holds nodes (bound + leaf) >> l -------------------------
    for (int l = 1; (bound >> l) >= 1; ++l) {
        for (int64_t k = tid; k < n; k += kSetThreads) {
            const int64_t parent = (bound + index[k]) >> l;
            tree[parent] = tree[2 * parent] + tree[2 * parent + 1];
        }
        __syncthreads();
    }
    if (prio_mode && prio_minmax) {
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
            lmax = fmax(lmax, tsb::shfl_xor_f64(lmax, off));
            lmin = fmin(lmin, tsb::shfl_xor_f64(lmin, off));
        }
        if ((tid & 31) == 0) { s_max[tid >> 5] = lmax; s_min[tid >> 5] = lmin; }
        __syncthreads();
        if (tid == 0) {
            double mx = prio_minmax[0], mn = prio_minmax[1];
            for (int w = 0; w < kSetThreads / 32; ++w) { mx = fmax(mx, s_max[w]); mn = fmin(mn, s_min[w]); }
            prio_minmax[0] = mx;   // prio.py:86-87
            prio_minmax[1] = mn;
        }
    }
}

__global__ void reduce_kernel(const double* __restrict__ tree, int64_t start, int64_t end,
                              double* __restrict__ out) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    double result = 0.0;           // segtree.py:104-116, same order of additions
    while (end - start > 1) {
        if (start % 2 == 0) result += tree[start + 1];
        start /= 2;
        if (end % 2 == 1) result += tree[end - 1];
        end /= 2;
    }
    *out = result;
}

template <bool kScaleByRoot>
__global__ void prefix_sum_idx_kernel(const double* __restrict__ tree, int64_t bound,
                                      const double* __restrict__ value, int64_t n,
                                      int64_t* __restrict__ out) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    double v = value[t];
    if (kScaleByRoot) v = __dmul_rn(v, tree[1]);   // np.random.rand(bs) * weight.reduce()
    int64_t index = 1;
    while (index < bound) {        // segtree.py:126-131
        index *= 2;
        const double lsons = __ldg(tree + index);
        if (lsons < v) {           // strict: ties go left
            v = __dsub_rn(v, lsons);
            index += 1;
        }
    }
    out[t] = index - bound;
}

__global__ void __launch_bounds__(1024) get_weight_kernel(
    const double* __restrict__ tree, int64_t bound, const int64_t* __restrict__ index, int64_t n,
    const double* __restrict__ prio_minmax, double beta, int weight_norm, double* __restrict__ out) {
    __shared__ double s_max[32];
    __shared__ double s_all;
    const int tid = threadIdx.x;
    const double min_prio = prio_minmax[1];
    double lmax = -1.0e300;
    for (int64_t k = tid; k < n; k += blockDim.x) {
        const double w = pow(tree[bound + index[k]] / min_prio, -beta);   // prio.py:79
        out[k] = w;
        lmax = fmax(lmax, w);
    }
    if (!weight_norm) return;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) lmax = fmax(lmax, tsb::shfl_xor_f64(lmax, off));
    if ((tid & 31) == 0) s_max[tid >> 5] = lmax;
    __syncthreads();
    if (tid == 0) {
        double mx = s_max[0];
        for (int w = 1; w < (int)(blockDim.x >> 5); ++w) mx = fmax(mx, s_max[w]);
        s_all = mx;
    }
    __syncthreads();
    const double mx = s_all;
    for (int64_t k = tid; k < n; k += blockDim.x) out[k] = out[k] / mx;      // prio.py:105
}

}  // namespace

extern "C" int ts_segtree_setitem(double* tree, int64_t bound, const int64_t* index,
                                  const void* value, int value_dtype, int64_t n,
                                  ts_stream_t stream) {
    if (n == 0) return 0;
    TS_REQUIRE(tree && index && value && bound >= 1, "ts_segtree_setitem: bad arguments");
    TS_REQUIRE(n <= 32 * kSetThreads, "ts_segtree_setitem: at most %d items per call", 32 * kSetThreads);
    cudaStream_t st = tsb::as_stream(stream);
    if (value_dtype == TS_F64)
        setitem_kernel<double><<<1, kSetThreads, 0, st>>>(tree, bound, index, static_cast<const double*>(value), n, 1.0, 0.0, 0, nullptr);
    else if (value_dtype == TS_F32)
        setitem_kernel<float><<<1, kSetThreads, 0, st>>>(tree, bound, index, static_cast<const float*>(value), n, 1.0, 0.0, 0, nullptr);
    else TS_REQUIRE(false, "ts_segtree_setitem: bad dtype");
    return tsb::check_launch("ts_segtree_setitem");
}

extern "C" int ts_prio_update_weight(double* tree, int64_t bound, const int64_t* index,
                                     const void* td, int td_dtype, int64_t n, double alpha,
                                     double eps, double* prio_minmax, ts_stream_t stream) {
    if (n == 0) return 0;
    TS_REQUIRE(tree && index && td && prio_minmax && bound >= 1, "ts_prio_update_weight: bad arguments");
    TS_REQUIRE(n <= 32 * kSetThreads, "ts_prio_update_weight: at most %d items per call", 32 * kSetThreads);
    cudaStream_t st = tsb::as_stream(stream);
    if (td_dtype == TS_F64)
        setitem_kernel<double><<<1, kSetThreads, 0, st>>>(tree, bound, index, static_cast<const double*>(td), n, alpha, eps, 1, prio_minmax);
    else if (td_dtype == TS_F32)
        setitem_kernel<float><<<1, kSetThreads, 0, st>>>(tree, bound, index, static_cast<const float*>(td), n, alpha, eps, 1, prio_minmax);
    else TS_REQUIRE(false, "ts_prio_update_weight: bad dtype");
    return tsb::check_launch("ts_prio_update_weight");
}

extern "C" int ts_segtree_reduce(const double* tree, int64_t bound, int64_t start, int64_t end,
                                 double* out, ts_stream_t stream) {
    TS_REQUIRE(tree && out && bound >= 1, "ts_segtree_reduce: bad arguments");
    // caller passes leaf positions [start, end); the reference walks (start+bound-1, end+bound)
    reduce_kernel<<<1, 32, 0, tsb::as_stream(stream)>>>(tree, start + bound - 1, end + bound, out);
    return tsb::check_launch("ts_segtree_reduce");
}

extern "C" int ts_segtree_prefix_sum_idx(const double* tree, int64_t bound, const double* value,
                                         int64_t n, int64_t* out, ts_stream_t stream) {
    if (n == 0) return 0;
    TS_REQUIRE(tree && value && out && bound >= 1, "ts_segtree_prefix_sum_idx: bad arguments");
    prefix_sum_idx_kernel<false><<<(unsigned)((n + 127) / 128), 128, 0, tsb::as_stream(stream)>>>(tree, bound, value, n, out);
    return tsb::check_launch("ts_segtree_prefix_sum_idx");
}

extern "C" int ts_segtree_sample(const double* tree, int64_t bound, const double* u, int64_t n,
                                 int64_t* out, ts_stream_t stream) {
    if (n == 0) return 0;
    TS_REQUIRE(tree && u && out && bound >= 1, "ts_segtree_sample: bad arguments");
    prefix_sum_idx_kernel<true><<<(unsigned)((n + 127) / 128), 128, 0, tsb::as_stream(stream)>>>(tree, bound, u, n, out);
    return tsb::check_launch("ts_segtree_sample");
}

extern "C" int ts_prio_get_weight(const double* tree, int64_t bound, const int64_t* index,
                                  int64_t n, const double* prio_minmax, double beta,
                                  int weight_norm, double* out, ts_stream_t stream) {
    if (n == 0) return 0;
    TS_REQUIRE(tree && index && prio_minmax && out, "ts_prio_get_weight: bad arguments");
    get_weight_kernel<<<1, 1024, 0, tsb::as_stream(stream)>>>(tree, bound, index, n, prio_minmax, beta, weight_norm, out);
    return tsb::check_launch("ts_prio_get_weight");
}
