// Posterior sampling RL (algorithm/modelbased/psrl.py): the posterior update of PSRL._update_with_batch + PSRLModel.observe, and
// PSRLModel.value_iteration as one persistent kernel.
//
// Reference: tianshou/algorithm/modelbased/psrl.py:65-98 (observe), :116-150 (value_iteration), :245-276 (the per-row loop over
// batch.split(size=1), whose order is np.random.permutation(len(batch))).
//
// Update: check (one pass over the rows, error flag) -> count (keys in permuted order, integer counts by atomics) -> CUB's stable
// radix sort of (key, reward) -> segment starts -> one thread per (s, a) sums its rows in permuted order and applies observe's
// formula -> the transition counts, one add per element -> the two stat means, fixed order.  Every kernel after the check does
// nothing when the flag is set, so a refused batch leaves the posterior bit-for-bit unchanged.
#include <math.h>

#include <cub/device/device_radix_sort.cuh>

#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kViThreads = 256;                              // 8 warps: one CTA covers 8 states per pass
constexpr double kEps32 = 1.1920928955078125e-07;            // np.finfo(np.float32).eps
constexpr double kAtol = 1e-8;                               // np.allclose's default atol

// the model-sized part of the update workspace comes first, so its layout does not depend on the row count: the transition
// counts stay zero between updates (the transition kernel consumes and clears them)
struct UpdateLayout {
    size_t err, trans_cnt, key_cnt, loop_cnt, seg, keys_in, vals_in, keys_out, vals_out, cub, total;
};

inline size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

inline UpdateLayout update_layout(int64_t n, int64_t n_s, int64_t n_a, size_t cub_bytes) {
    UpdateLayout L{};
    const int64_t K = n_s * n_a;
    size_t o = 0;
    L.err = o;       o += align256(sizeof(int));
    L.trans_cnt = o; o += align256((size_t)(K * n_s) * sizeof(unsigned int));
    L.key_cnt = o;   o += align256((size_t)K * sizeof(unsigned int));
    L.loop_cnt = o;  o += align256((size_t)n_s * sizeof(unsigned int));
    L.seg = o;       o += align256((size_t)K * sizeof(int));
    L.keys_in = o;   o += align256((size_t)n * sizeof(int));
    L.vals_in = o;   o += align256((size_t)n * sizeof(double));
    L.keys_out = o;  o += align256((size_t)n * sizeof(int));
    L.vals_out = o;  o += align256((size_t)n * sizeof(double));
    L.cub = o;       o += align256(cub_bytes);
    L.total = o;
    return L;
}

inline int key_bits(int64_t K) {
    int b = 1;
    while (b < 31 && ((int64_t)1 << b) < K) ++b;
    return b;
}

inline size_t cub_sort_bytes(int64_t n, int bits) {
    size_t bytes = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, bytes, (const int*)nullptr, (int*)nullptr, (const double*)nullptr, (double*)nullptr,
                                    (int)n, 0, bits);
    return bytes;
}

// index column value of row r: int64, or float32 holding an integer (the device mirror's columns)
__device__ __forceinline__ bool read_index(const void* col, int f32, int64_t r, int64_t n, int64_t& out) {
    if (f32) {
        const float v = static_cast<const float*>(col)[r];
        if (!(v >= 0.0f && v < (float)n && v == truncf(v))) return false;
        out = (int64_t)v;
        return out < n;
    }
    out = static_cast<const int64_t*>(col)[r];
    return out >= 0 && out < n;
}

__global__ void __launch_bounds__(kThreads) psrl_check_kernel(const void* __restrict__ obs, const void* __restrict__ act,
                                                              const void* __restrict__ obs_next, int idx_f32, int64_t N, int n_s,
                                                              int n_a, int* __restrict__ err) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < N; r += (int64_t)gridDim.x * blockDim.x) {
        int64_t s, a, t;
        if (!read_index(obs, idx_f32, r, n_s, s) || !read_index(act, idx_f32, r, n_a, a) || !read_index(obs_next, idx_f32, r, n_s, t))
            *err = 1;
    }
}

// position j of the permuted order holds row perm[j]: key s n_a + a and the row's reward (widened to float64, exactly), for the
// stable sort, which then hands every key its rewards contiguous and in permuted order; the integer counts of the batch (exact
// in any order) by atomics.  With add_done_loop a done row also counts the self-loops of its next state.
__global__ void __launch_bounds__(kThreads) psrl_count_kernel(const void* __restrict__ obs, const void* __restrict__ act,
                                                              const void* __restrict__ obs_next, int idx_f32,
                                                              const void* __restrict__ rew, int rew_f64,
                                                              const uint8_t* __restrict__ done, int add_done_loop,
                                                              const int64_t* __restrict__ perm, int64_t N, int n_s, int n_a,
                                                              const int* __restrict__ err, int* __restrict__ keys,
                                                              double* __restrict__ vals, unsigned int* __restrict__ trans_cnt,
                                                              unsigned int* __restrict__ key_cnt, unsigned int* __restrict__ loop_cnt) {
    const bool bad = *err != 0;
    for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < N; j += (int64_t)gridDim.x * blockDim.x) {
        if (bad) {              // the sort still runs: give it defined keys
            keys[j] = 0;
            vals[j] = 0.0;
            continue;
        }
        const int64_t r = perm[j];
        int64_t s = 0, a = 0, t = 0;
        read_index(obs, idx_f32, r, n_s, s);
        read_index(act, idx_f32, r, n_a, a);
        read_index(obs_next, idx_f32, r, n_s, t);
        const int64_t k = s * n_a + a;
        keys[j] = (int)k;
        vals[j] = rew_f64 ? static_cast<const double*>(rew)[r] : (double)static_cast<const float*>(rew)[r];
        atomicAdd(&trans_cnt[k * n_s + t], 1u);
        atomicAdd(&key_cnt[k], 1u);
        if (add_done_loop && done[r]) atomicAdd(&loop_cnt[t], 1u);
    }
}

// first sorted position of every key that has rows
__global__ void __launch_bounds__(kThreads) psrl_segment_kernel(const int* __restrict__ keys, int64_t N, const int* __restrict__ err,
                                                                int* __restrict__ seg) {
    if (*err) return;
    for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < N; j += (int64_t)gridDim.x * blockDim.x) {
        if (j == 0 || keys[j] != keys[j - 1]) seg[keys[j]] = (int)j;
    }
}

// observe's update of one (s, a) from the batch's count n, reward sum rs and square sum rq, in the reference's operation order
// with explicitly rounded operations (no contraction):
//   sum_count = rew_count + n;  rew_mean = (rew_mean rew_count + rs) / sum_count;  rew_square_sum += rq;
//   raw = rew_square_sum / sum_count - rew_mean^2;  rew_std = sqrt(1 / (sum_count / (raw + eps32) + 1 / prior^2));
//   rew_count = sum_count.
__device__ __forceinline__ void observe_one(int64_t k, double n, double rs, double rq, double* __restrict__ rew_mean,
                                            double* __restrict__ rew_std, double* __restrict__ rew_square_sum,
                                            double* __restrict__ rew_count, const double* __restrict__ std_prior) {
    const double cnt = rew_count[k];
    const double sc = __dadd_rn(cnt, n);
    const double mean = __ddiv_rn(__dadd_rn(__dmul_rn(rew_mean[k], cnt), rs), sc);
    const double sq = __dadd_rn(rew_square_sum[k], rq);
    const double raw = __dsub_rn(__ddiv_rn(sq, sc), __dmul_rn(mean, mean));
    const double p = std_prior[k];
    const double inner = __dadd_rn(__ddiv_rn(sc, __dadd_rn(raw, kEps32)), __ddiv_rn(1.0, __dmul_rn(p, p)));
    rew_std[k] = __dsqrt_rn(__ddiv_rn(1.0, inner));
    rew_mean[k] = mean;
    rew_square_sum[k] = sq;
    rew_count[k] = sc;
}

// One thread per (s, a): rew_sum and rew_square_sum of its rewards (contiguous after the sort), summed from 0.0 in the permuted
// order, then observe_one.  A float32 reward is squared in float32 (sq_f32) before it is widened, as numpy squares the batch's
// dtype.  The sums must run in order, so the key with the most rows bounds the update; its loads do not depend on each other
// and are issued ahead of the additions.
__global__ void __launch_bounds__(kThreads) psrl_observe_kernel(int sq_f32, const int* __restrict__ seg,
                                                                const double* __restrict__ sorted_rew,
                                                                const unsigned int* __restrict__ key_cnt,
                                                                const unsigned int* __restrict__ loop_cnt, int n_s, int n_a,
                                                                const int* __restrict__ err, double* __restrict__ rew_mean,
                                                                double* __restrict__ rew_std, double* __restrict__ rew_square_sum,
                                                                double* __restrict__ rew_count, const double* __restrict__ std_prior) {
    if (*err) return;
    const int64_t K = (int64_t)n_s * n_a;
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < K; k += (int64_t)gridDim.x * blockDim.x) {
        const unsigned int c = key_cnt[k];
        double rs = 0.0, rq = 0.0;
        if (c) {
            const double* rk = sorted_rew + seg[k];
#pragma unroll 8
            for (unsigned int i = 0; i < c; ++i) {
                const double x = rk[i];
                double x2;
                if (sq_f32) {
                    const float xf = (float)x;
                    x2 = (double)__fmul_rn(xf, xf);
                } else {
                    x2 = __dmul_rn(x, x);
                }
                rs = __dadd_rn(rs, x);
                rq = __dadd_rn(rq, x2);
            }
        }
        observe_one(k, (double)(c + loop_cnt[k / n_a]), rs, rq, rew_mean, rew_std, rew_square_sum, rew_count, std_prior);
    }
}

// trans_count += batch counts, one add per element (the done-loop counts on the diagonal), and the counts cleared for the next
// update
__global__ void __launch_bounds__(kThreads) psrl_trans_kernel(unsigned int* __restrict__ trans_cnt,
                                                              const unsigned int* __restrict__ loop_cnt, int n_s, int n_a,
                                                              const int* __restrict__ err, double* __restrict__ trans_count) {
    if (*err) return;
    const int64_t total = (int64_t)n_s * n_a * n_s;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t k = e / n_s, t = e - k * n_s, s = k / n_a;
        const unsigned int c = trans_cnt[e] + (s == t ? loop_cnt[s] : 0u);
        trans_count[e] = __dadd_rn(trans_count[e], (double)c);
        if (trans_cnt[e]) trans_cnt[e] = 0u;
    }
}

// PSRLModel.observe with the batch's dense arrays: trans_count += tc (one add per element) and observe_one per (s, a)
__global__ void __launch_bounds__(kThreads) psrl_observe_dense_kernel(const double* __restrict__ tc, const double* __restrict__ rs,
                                                                      const double* __restrict__ rq, const double* __restrict__ rc,
                                                                      int64_t K, int n_s, double* __restrict__ trans_count,
                                                                      double* __restrict__ rew_mean, double* __restrict__ rew_std,
                                                                      double* __restrict__ rew_square_sum,
                                                                      double* __restrict__ rew_count,
                                                                      const double* __restrict__ std_prior) {
    const int64_t total = K * n_s;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
        trans_count[e] = __dadd_rn(trans_count[e], tc[e]);
        if (e < K) observe_one(e, rc[e], rs[e], rq[e], rew_mean, rew_std, rew_square_sum, rew_count, std_prior);
    }
}

// result = (error flag, mean(rew_mean), mean(rew_std)): strided per-thread sums then a tree over the block, a fixed order
__global__ void __launch_bounds__(kThreads) psrl_stats_kernel(const double* __restrict__ rew_mean, const double* __restrict__ rew_std,
                                                              int64_t K, const int* __restrict__ err, double* __restrict__ result) {
    __shared__ double sm[2][kThreads];
    double a = 0.0, b = 0.0;
    for (int64_t k = threadIdx.x; k < K; k += kThreads) {
        a = __dadd_rn(a, rew_mean[k]);
        b = __dadd_rn(b, rew_std[k]);
    }
    sm[0][threadIdx.x] = a;
    sm[1][threadIdx.x] = b;
    __syncthreads();
    for (int w = kThreads / 2; w > 0; w >>= 1) {
        if ((int)threadIdx.x < w) {
            sm[0][threadIdx.x] = __dadd_rn(sm[0][threadIdx.x], sm[0][threadIdx.x + w]);
            sm[1][threadIdx.x] = __dadd_rn(sm[1][threadIdx.x], sm[1][threadIdx.x + w]);
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        result[0] = (double)*err;
        result[1] = sm[0][0] / (double)K;
        result[2] = sm[1][0] / (double)K;
    }
}

// ---------------------------------------------------------------------------------------------------------- value iteration
// Barrier and convergence state of one solve, zeroed by the host before the launch.  flag[k % 3] is set by any state of sweep k
// whose new value is not close to the old one; CTA 0 clears flag[(k + 1) % 3] during sweep k: every CTA read it last after
// barrier k - 2 and wrote nothing to it since, and it is written again only after barrier k.
struct ViCtl {
    unsigned long long arrive;        // grid-barrier arrivals: 64 bits, so no sweep count can wrap it
    unsigned int flag[3], pad2;
    unsigned long long maxdiff;       // bits of max |V' - V| of the last permitted sweep (a non-negative double; NaN sorts above)
};

__device__ __forceinline__ double warp_sum_f64(double v) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) v += tsb::shfl_xor_f64(v, off);
    return v;
}

// np.isclose(new, old, rtol=eps): |new - old| <= atol + eps |old| with old finite, or new == old
__device__ __forceinline__ bool vi_close(double nv, double ov, double eps) {
    return (fabs(nv - ov) <= __dadd_rn(kAtol, __dmul_rn(eps, fabs(ov))) && isfinite(ov)) || nv == ov;
}

// Sweep k: V (value for k = 0, else vbuf[k & 1]) staged in shared memory; one warp per state s (grid-stride over states), for
// each action a the dot P[s, a, :] . V in one fixed order (lane-strided FMAs, then the xor butterfly), Q = rew + gamma dot,
// V'[s] = max_a Q (NaN propagates) into vbuf[(k + 1) & 1] and Q into qbuf; then a grid barrier and the sweep's flag.  Converged
// (no state not close) -> epilogue: policy = first argmax_a (Q + eps noise) (a NaN wins, as in numpy), value = V'.  Not converged
// after max_iter sweeps -> nothing is written but out[n_s:].  out = [policy (n_s)][sweeps][converged][max |V' - V| bits].
__global__ void __launch_bounds__(kViThreads, 1) psrl_value_iteration_kernel(const double* __restrict__ P, const double* __restrict__ R,
                                                                          const double* __restrict__ noise, int n_s, int n_a,
                                                                          double gamma, double eps, int64_t max_iter, double* value,
                                                                          double* vbuf, double* __restrict__ qbuf, ViCtl* ctl,
                                                                          int64_t* __restrict__ out) {
    extern __shared__ double sv[];
    __shared__ int s_more;
    const int lane = tsb::lane_id();
    const int nw = kViThreads / 32;
    const int64_t gw0 = (int64_t)blockIdx.x * nw + tsb::warp_id(), tw = (int64_t)gridDim.x * nw;
    unsigned long long target = 0;
    int64_t k = 0;
    bool converged = false;
    for (;; ++k) {
        const double* vin = k == 0 ? value : vbuf + (k & 1) * (int64_t)n_s;
        double* vout = vbuf + ((k + 1) & 1) * (int64_t)n_s;
        for (int i = threadIdx.x; i < n_s; i += kViThreads) sv[i] = __ldcg(vin + i);
        if (blockIdx.x == 0 && threadIdx.x == 0) {
            volatile unsigned int* f = ctl->flag;
            f[(k + 1) % 3] = 0u;
        }
        __syncthreads();
        const bool last = k + 1 >= max_iter;
        for (int64_t s = gw0; s < n_s; s += tw) {
            double vmax = 0.0;
            for (int a = 0; a < n_a; ++a) {
                const double* prow = P + ((int64_t)s * n_a + a) * n_s;
                double acc = 0.0;
                for (int t = lane; t < n_s; t += 32) acc = fma(__ldg(prow + t), sv[t], acc);
                acc = warp_sum_f64(acc);
                const double q = __dadd_rn(R[s * n_a + a], __dmul_rn(gamma, acc));
                if (lane == 0) qbuf[s * n_a + a] = q;
                vmax = (a == 0 || q > vmax || isnan(q)) ? q : vmax;
            }
            if (lane == 0) {
                const double ov = sv[s];
                __stcg(vout + s, vmax);
                if (!vi_close(vmax, ov, eps)) {
                    volatile unsigned int* f = ctl->flag;
                    f[k % 3] = 1u;
                }
                if (last) atomicMax(&ctl->maxdiff, (unsigned long long)__double_as_longlong(fabs(vmax - ov)));
            }
        }
        // grid barrier (every CTA is resident: cooperative launch)
        __syncthreads();
        if (threadIdx.x == 0) {
            target += gridDim.x;
            asm volatile("red.release.gpu.global.add.u64 [%0], 1;" ::"l"(&ctl->arrive) : "memory");
            unsigned long long seen;
            do {
                asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(seen) : "l"(&ctl->arrive) : "memory");
            } while (seen < target);
            unsigned int more;
            asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(more) : "l"(&ctl->flag[k % 3]) : "memory");
            s_more = (int)more;
        }
        __syncthreads();
        if (!s_more) {
            converged = true;
            break;
        }
        if (last) break;
    }
    if (converged) {
        const double* vfin = vbuf + ((k + 1) & 1) * (int64_t)n_s;
        for (int64_t s = gw0; s < n_s; s += tw) {
            if (lane != 0) continue;
            int best = 0;
            double bq = 0.0;
            for (int a = 0; a < n_a; ++a) {
                const double x = __dadd_rn(qbuf[s * n_a + a], __dmul_rn(eps, noise[s * n_a + a]));
                if (a == 0 || (!isnan(bq) && (x > bq || isnan(x)))) {
                    bq = x;
                    best = a;
                }
            }
            out[s] = best;
            value[s] = __ldcg(vfin + s);
        }
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        out[n_s] = k + 1;
        out[n_s + 1] = converged ? 1 : 0;
        out[n_s + 2] = (int64_t)*(volatile unsigned long long*)&ctl->maxdiff;
    }
}

inline unsigned grid_for(int64_t items) {
    int64_t b = (items + kThreads - 1) / kThreads;
    const int64_t cap = (int64_t)tsb::num_sms() * 8;
    return (unsigned)(b > cap ? cap : (b < 1 ? 1 : b));
}

inline size_t vi_static_smem() { return 1024; }       // s_more and alignment headroom

}  // namespace

extern "C" int64_t ts_psrl_update_workspace_bytes(int64_t n, int32_t n_state, int32_t n_action) {
    if (n < 1 || n_state < 1 || n_action < 1) return 0;
    const int64_t K = (int64_t)n_state * n_action;
    return (int64_t)update_layout(n, n_state, n_action, cub_sort_bytes(n, key_bits(K))).total;
}

extern "C" int ts_psrl_update(const void* obs, const void* act, const void* obs_next, int32_t idx_f32, const void* rew, int32_t rew_dtype,
                              int32_t sq_f32, const uint8_t* done, int32_t add_done_loop, const int64_t* perm, int64_t n,
                              int32_t n_state, int32_t n_action, double* trans_count, double* rew_mean, double* rew_std,
                              double* rew_square_sum, double* rew_count, const double* rew_std_prior, void* workspace,
                              int64_t workspace_bytes, double* result, ts_stream_t stream) {
    TS_REQUIRE(obs && act && obs_next && rew && perm && trans_count && rew_mean && rew_std && rew_square_sum && rew_count &&
                   rew_std_prior && workspace && result && n >= 1 && n < ((int64_t)1 << 31) && n_state >= 1 && n_action >= 1,
               "ts_psrl_update: bad argument");
    TS_REQUIRE(!add_done_loop || done, "ts_psrl_update: add_done_loop needs done");
    TS_REQUIRE(rew_dtype == TS_F32 || rew_dtype == TS_F64, "ts_psrl_update: rew must be float32 or float64");
    const int64_t K = (int64_t)n_state * n_action;
    TS_REQUIRE(K < ((int64_t)1 << 31), "ts_psrl_update: n_state * n_action too large");
    const int bits = key_bits(K);
    size_t cub_bytes = cub_sort_bytes(n, bits);
    const UpdateLayout L = update_layout(n, n_state, n_action, cub_bytes);
    TS_REQUIRE((int64_t)L.total <= workspace_bytes, "ts_psrl_update: workspace too small (%lld < %lld bytes)",
               (long long)workspace_bytes, (long long)L.total);
    cudaStream_t st = tsb::as_stream(stream);
    uint8_t* ws = static_cast<uint8_t*>(workspace);
    int* err = reinterpret_cast<int*>(ws + L.err);
    auto* trans_cnt = reinterpret_cast<unsigned int*>(ws + L.trans_cnt);
    auto* key_cnt = reinterpret_cast<unsigned int*>(ws + L.key_cnt);
    auto* loop_cnt = reinterpret_cast<unsigned int*>(ws + L.loop_cnt);
    int* seg = reinterpret_cast<int*>(ws + L.seg);
    int* keys_in = reinterpret_cast<int*>(ws + L.keys_in);
    double* vals_in = reinterpret_cast<double*>(ws + L.vals_in);
    int* keys_out = reinterpret_cast<int*>(ws + L.keys_out);
    double* vals_out = reinterpret_cast<double*>(ws + L.vals_out);
    TS_CUDA(cudaMemsetAsync(ws, 0, L.trans_cnt, st));                                          // error flag
    TS_CUDA(cudaMemsetAsync(ws + L.key_cnt, 0, L.seg - L.key_cnt, st));                        // key and loop counts
    const int f32 = idx_f32 ? 1 : 0;
    psrl_check_kernel<<<grid_for(n), kThreads, 0, st>>>(obs, act, obs_next, f32, n, n_state, n_action, err);
    if (tsb::check_launch("ts_psrl_update/check")) return 1;
    psrl_count_kernel<<<grid_for(n), kThreads, 0, st>>>(obs, act, obs_next, f32, rew, rew_dtype == TS_F64 ? 1 : 0, done, add_done_loop ? 1 : 0, perm, n, n_state,
                                                        n_action, err, keys_in, vals_in, trans_cnt, key_cnt, loop_cnt);
    if (tsb::check_launch("ts_psrl_update/count")) return 1;
    TS_CUDA(cub::DeviceRadixSort::SortPairs(ws + L.cub, cub_bytes, keys_in, keys_out, vals_in, vals_out, (int)n, 0, bits, st));
    psrl_segment_kernel<<<grid_for(n), kThreads, 0, st>>>(keys_out, n, err, seg);
    if (tsb::check_launch("ts_psrl_update/segment")) return 1;
    psrl_observe_kernel<<<grid_for(K), kThreads, 0, st>>>(sq_f32 ? 1 : 0, seg, vals_out, key_cnt,
                                                          loop_cnt, n_state, n_action, err, rew_mean, rew_std, rew_square_sum,
                                                          rew_count, rew_std_prior);
    if (tsb::check_launch("ts_psrl_update/observe")) return 1;
    psrl_trans_kernel<<<grid_for(K * n_state), kThreads, 0, st>>>(trans_cnt, loop_cnt, n_state, n_action, err, trans_count);
    if (tsb::check_launch("ts_psrl_update/trans")) return 1;
    psrl_stats_kernel<<<1, kThreads, 0, st>>>(rew_mean, rew_std, K, err, result);
    return tsb::check_launch("ts_psrl_update/stats");
}

extern "C" int ts_psrl_observe(const double* trans_count_batch, const double* rew_sum, const double* rew_square_sum_batch,
                               const double* rew_count_batch, int32_t n_state, int32_t n_action, double* trans_count,
                               double* rew_mean, double* rew_std, double* rew_square_sum, double* rew_count,
                               const double* rew_std_prior, int* flag, double* result, ts_stream_t stream) {
    TS_REQUIRE(trans_count_batch && rew_sum && rew_square_sum_batch && rew_count_batch && trans_count && rew_mean && rew_std &&
                   rew_square_sum && rew_count && rew_std_prior && flag && result && n_state >= 1 && n_action >= 1,
               "ts_psrl_observe: bad argument");
    cudaStream_t st = tsb::as_stream(stream);
    const int64_t K = (int64_t)n_state * n_action;
    TS_CUDA(cudaMemsetAsync(flag, 0, sizeof(int), st));
    psrl_observe_dense_kernel<<<grid_for(K * n_state), kThreads, 0, st>>>(trans_count_batch, rew_sum, rew_square_sum_batch,
                                                                          rew_count_batch, K, n_state, trans_count, rew_mean,
                                                                          rew_std, rew_square_sum, rew_count, rew_std_prior);
    if (tsb::check_launch("ts_psrl_observe")) return 1;
    psrl_stats_kernel<<<1, kThreads, 0, st>>>(rew_mean, rew_std, K, flag, result);
    return tsb::check_launch("ts_psrl_observe/stats");
}

extern "C" int32_t ts_psrl_max_states(void) {
    int dev = 0, optin = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 0;
    if (cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess) return 0;
    return (int32_t)(((size_t)optin - vi_static_smem()) / sizeof(double));
}

extern "C" int64_t ts_psrl_value_iteration_scratch_bytes(int32_t n_state, int32_t n_action) {
    return (int64_t)(align256(sizeof(ViCtl)) + align256(2 * (size_t)n_state * sizeof(double)) +
                     align256((size_t)n_state * n_action * sizeof(double)));
}

extern "C" int ts_psrl_value_iteration(const double* trans_prob, const double* rew, const double* noise, int32_t n_state,
                                       int32_t n_action, double gamma, double eps, int64_t max_iterations, double* value,
                                       void* scratch, int64_t* out, ts_stream_t stream) {
    TS_REQUIRE(trans_prob && rew && noise && value && scratch && out && n_state >= 1 && n_action >= 1 && max_iterations >= 1,
               "ts_psrl_value_iteration: bad argument");
    TS_REQUIRE(n_state <= ts_psrl_max_states(), "ts_psrl_value_iteration: %d states do not fit in shared memory (at most %d)",
               (int)n_state, (int)ts_psrl_max_states());
    cudaStream_t st = tsb::as_stream(stream);
    uint8_t* ws = static_cast<uint8_t*>(scratch);
    ViCtl* ctl = reinterpret_cast<ViCtl*>(ws);
    double* vbuf = reinterpret_cast<double*>(ws + align256(sizeof(ViCtl)));
    double* qbuf = reinterpret_cast<double*>(ws + align256(sizeof(ViCtl)) + align256(2 * (size_t)n_state * sizeof(double)));
    const size_t smem = (size_t)n_state * sizeof(double);
    if (smem > 48 * 1024)
        TS_CUDA(cudaFuncSetAttribute(psrl_value_iteration_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 0;
    TS_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, psrl_value_iteration_kernel, kViThreads, smem));
    TS_REQUIRE(per_sm >= 1, "ts_psrl_value_iteration: the kernel does not fit on an SM with %zu bytes of shared memory", smem);
    const int64_t warps = kViThreads / 32;
    const unsigned grid = (unsigned)tsb::imin((n_state + warps - 1) / warps, tsb::num_sms());
    TS_CUDA(cudaMemsetAsync(ctl, 0, sizeof(ViCtl), st));
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(kViThreads);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeCooperative;
    attr[0].val.cooperative = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    TS_CUDA(cudaLaunchKernelEx(&cfg, psrl_value_iteration_kernel, trans_prob, rew, noise, (int)n_state, (int)n_action, gamma, eps,
                               max_iterations, value, vbuf, qbuf, ctl, out));
    return tsb::check_launch("ts_psrl_value_iteration");
}
