// GAE as a single-pass segmented reverse scan (decoupled look-back), sm_90a.
//
// Reference semantics: numba `_gae` (tianshou/algorithm/algorithm_base.py:1085-1140) plus the
// value-mask / end-flag / return-scaling arithmetic of compute_episodic_return (:704-719) and
// _add_returns_and_advantages (modelfree/a2c.py:131-152), and RunningMeanStd.update
// (utils/statistics.py:99-114).  See include/ts_b200.h for the exact formulae.
//
// Algorithm.  adv_i = delta_i + m_i * adv_{i+1} is the affine map T_i(g) = b_i + a_i g with
// a_i = (1-end_i) gamma lambda, b_i = delta_i.  Affine maps compose associatively, so the whole
// flat array is ONE reverse scan; episode boundaries need no special handling because end flags
// make a_i exactly 0, which also cuts the look-back chain between tiles.  Each CTA owns a tile of
// 2048 consecutive transitions (8 per thread, read with 128-bit loads), composes right-to-left in
// registers, does a warp-shuffle suffix scan of (a,b) pairs, stages the 8 warp aggregates in
// shared memory, publishes the tile aggregate, looks back over the tiles to its right for the
// carry-in and writes adv / returns.  All arithmetic is f64 (the reference accumulates in f64).
//
// HBM traffic per transition (f32 values, f64 rew, 3 flag bytes, f32 outputs): 4+4+8+3+4+4 = 27 B.
#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kItems = 8;
constexpr int kTile = kThreads * kItems;
constexpr int kWarps = kThreads / 32;

struct TileState {   // 32 B: one sector
    double A, B, G;
    int flag;        // 0 = empty, 1 = aggregate (A,B) valid, 2 = G (adv at tile start) valid
    int pad;
};
struct TileMoments { // partial (count, mean, M2) of un-scaled returns
    double n, mean, M2, pad;
};
struct WsHeader {
    int ticket;
    int done;
    int pad[14];
};

struct GaeParams {
    const void* v_s;
    const void* v_n;
    const double* rew;
    const uint8_t* terminated;
    const uint8_t* truncated;
    const uint8_t* extra_end;
    int terminated_ends;
    int vec_ok;
    int64_t n;
    int num_tiles;
    double gamma, lam;
    double* rms;  // {mean, var, count} or null
    double* batch_moments;  // {count, mean, M2} of this call's un-scaled returns, or null
    double rms_eps;
    void* adv_out;
    void* ret_out;
    WsHeader* hdr;
    TileState* tiles;
    TileMoments* moments;
};

__device__ __forceinline__ int ld_acquire(const int* p) {
    int v;
    asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release(int* p, int v) {
    asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

template <typename T>
__device__ __forceinline__ void load8(const T* __restrict__ p, int64_t base, double (&out)[kItems]);

template <>
__device__ __forceinline__ void load8<float>(const float* __restrict__ p, int64_t base,
                                             double (&out)[kItems]) {
    const float4 a = __ldcs(reinterpret_cast<const float4*>(p + base));
    const float4 b = __ldcs(reinterpret_cast<const float4*>(p + base + 4));
    out[0] = a.x; out[1] = a.y; out[2] = a.z; out[3] = a.w;
    out[4] = b.x; out[5] = b.y; out[6] = b.z; out[7] = b.w;
}
template <>
__device__ __forceinline__ void load8<double>(const double* __restrict__ p, int64_t base,
                                              double (&out)[kItems]) {
#pragma unroll
    for (int j = 0; j < kItems; j += 2) {
        const double2 a = __ldcs(reinterpret_cast<const double2*>(p + base + j));
        out[j] = a.x; out[j + 1] = a.y;
    }
}
__device__ __forceinline__ void load8_flags(const uint8_t* __restrict__ p, int64_t base,
                                            uint32_t (&out)[kItems]) {
    const uint2 w = __ldcs(reinterpret_cast<const uint2*>(p + base));
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        out[j] = (w.x >> (8 * j)) & 0xffu;
        out[4 + j] = (w.y >> (8 * j)) & 0xffu;
    }
}

template <typename T>
__device__ __forceinline__ void store8(T* p, int64_t base, const double (&v)[kItems]);
template <>
__device__ __forceinline__ void store8<float>(float* p, int64_t base, const double (&v)[kItems]) {
    float4 a = make_float4((float)v[0], (float)v[1], (float)v[2], (float)v[3]);
    float4 b = make_float4((float)v[4], (float)v[5], (float)v[6], (float)v[7]);
    __stcs(reinterpret_cast<float4*>(p + base), a);
    __stcs(reinterpret_cast<float4*>(p + base + 4), b);
}
template <>
__device__ __forceinline__ void store8<double>(double* p, int64_t base, const double (&v)[kItems]) {
#pragma unroll
    for (int j = 0; j < kItems; j += 2)
        __stcs(reinterpret_cast<double2*>(p + base + j), make_double2(v[j], v[j + 1]));
}

// Chan merge of (n, mean, M2) partials; (n2, m2, M2b) is folded into (n1, m1, M1).
__device__ __forceinline__ void chan_merge(double& n1, double& m1, double& M1, double n2, double m2,
                                           double M2b) {
    const double n = n1 + n2;
    if (n2 == 0.0) return;
    if (n1 == 0.0) { n1 = n2; m1 = m2; M1 = M2b; return; }
    const double d = m2 - m1;
    m1 = m1 + d * (n2 / n);
    M1 = M1 + M2b + d * d * (n1 * n2 / n);
    n1 = n;
}

template <typename TV, typename TO>
__global__ void __launch_bounds__(kThreads) gae_scan_kernel(const GaeParams p) {
    __shared__ int s_tile;
    __shared__ int s_is_last;
    __shared__ double s_wA[kWarps], s_wB[kWarps];
    __shared__ double s_carry;
    __shared__ double s_mn[kWarps], s_mm[kWarps], s_mM[kWarps];

    const int tid = threadIdx.x;
    const int lane = tid & 31, warp = tid >> 5;
    if (tid == 0) s_tile = atomicAdd(&p.hdr->ticket, 1);
    __syncthreads();
    const int tile = p.num_tiles - 1 - s_tile;  // tiles are claimed right-to-left

    const double scale = p.rms ? sqrt(p.rms[1] + p.rms_eps) : 1.0;  // pre-update var (a2c.py:135)
    const double gl = p.gamma * p.lam;

    const int64_t base = (int64_t)tile * kTile + (int64_t)tid * kItems;
    double vs[kItems], d[kItems], a[kItems];
    {
        double vn[kItems], rw[kItems];
        uint32_t term[kItems], endf[kItems];
        if (p.vec_ok && base + kItems <= p.n) {
            load8<TV>(static_cast<const TV*>(p.v_s), base, vs);
            load8<TV>(static_cast<const TV*>(p.v_n), base, vn);
            load8<double>(p.rew, base, rw);
#pragma unroll
            for (int j = 0; j < kItems; ++j) { term[j] = 0; endf[j] = 0; }
            if (p.terminated) {
                load8_flags(p.terminated, base, term);
                if (p.terminated_ends) {
#pragma unroll
                    for (int j = 0; j < kItems; ++j) endf[j] |= term[j];
                }
            }
            if (p.truncated) {
                uint32_t t2[kItems];
                load8_flags(p.truncated, base, t2);
#pragma unroll
                for (int j = 0; j < kItems; ++j) endf[j] |= t2[j];
            }
            if (p.extra_end) {
                uint32_t t3[kItems];
                load8_flags(p.extra_end, base, t3);
#pragma unroll
                for (int j = 0; j < kItems; ++j) endf[j] |= t3[j];
            }
        } else {
#pragma unroll
            for (int j = 0; j < kItems; ++j) {
                const int64_t i = base + j;
                if (i < p.n) {
                    vs[j] = (double)static_cast<const TV*>(p.v_s)[i];
                    vn[j] = (double)static_cast<const TV*>(p.v_n)[i];
                    rw[j] = p.rew[i];
                    term[j] = p.terminated ? p.terminated[i] : 0u;
                    uint32_t e = (p.terminated_ends ? term[j] : 0u);
                    if (p.truncated) e |= p.truncated[i];
                    if (p.extra_end) e |= p.extra_end[i];
                    endf[j] = e;
                } else {  // padding right of the data: identity map, carries adv[n] = 0 through
                    vs[j] = 0.0; vn[j] = 0.0; rw[j] = 0.0; term[j] = 0; endf[j] = 0xffffffffu;
                }
            }
        }
#pragma unroll
        for (int j = 0; j < kItems; ++j) {
            const bool pad = (endf[j] == 0xffffffffu);
            vs[j] = vs[j] * scale;
            const double vnj = vn[j] * scale * (term[j] ? 0.0 : 1.0);
            // delta = rew + v_s_ * gamma - v_s   (algorithm_base.py:1134)
            d[j] = __dsub_rn(__dadd_rn(rw[j], __dmul_rn(vnj, p.gamma)), vs[j]);
            a[j] = pad ? 1.0 : (endf[j] ? 0.0 : gl);
            if (pad) d[j] = 0.0;
        }
    }

    // thread-local composite of its 8 maps, applied right-to-left
    double A = 1.0, B = 0.0;
#pragma unroll
    for (int j = kItems - 1; j >= 0; --j) {
        B = d[j] + a[j] * B;
        A = a[j] * A;
    }
    // warp inclusive suffix scan: (A,B) of lanes [lane, 31]
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
        const double A2 = tsb::shfl_down_f64(A, off);
        const double B2 = tsb::shfl_down_f64(B, off);
        if (lane + off < 32) {
            B = B + A * B2;
            A = A * A2;
        }
    }
    if (lane == 0) { s_wA[warp] = A; s_wB[warp] = B; }
    // exclusive: composite of lanes (lane, 31]
    double eA = tsb::shfl_down_f64(A, 1), eB = tsb::shfl_down_f64(B, 1);
    if (lane == 31) { eA = 1.0; eB = 0.0; }
    __syncthreads();
#pragma unroll
    for (int w = 0; w < kWarps; ++w) {
        if (w > warp) {
            eB = eB + eA * s_wB[w];
            eA = eA * s_wA[w];
        }
    }

    if (tid == 0) {
        double tA = 1.0, tB = 0.0;  // tile aggregate = W_0 o W_1 o ... o W_7
        for (int w = kWarps - 1; w >= 0; --w) {
            tB = s_wB[w] + s_wA[w] * tB;
            tA = s_wA[w] * tA;
        }
        TileState* me = p.tiles + tile;
        volatile TileState* vt = p.tiles;
        const bool last_tile = (tile == p.num_tiles - 1);
        // G (adv at the tile's first element) is known without a carry when nothing lies to the
        // right (adv[n] = 0) or when a segment cut inside the tile makes tA exactly 0.
        const bool g_known = last_tile || tA == 0.0;
        me->A = tA; me->B = tB;
        if (g_known) me->G = tB;
        __threadfence();
        st_release(&me->flag, g_known ? 2 : 1);
        double carry = 0.0;
        if (!last_tile) {
            double cA = 1.0, cB = 0.0;  // composite of the tiles in (tile, t)
            int t = tile + 1;
            while (true) {
                if (t >= p.num_tiles) { carry = cB; break; }  // cB + cA * adv[n], adv[n] = 0
                int f;
                do { f = ld_acquire(&p.tiles[t].flag); } while (f == 0);
                if (f == 2) { carry = cB + cA * vt[t].G; break; }
                cB = cB + cA * vt[t].B;
                cA = cA * vt[t].A;
                if (cA == 0.0) { carry = cB; break; }
                ++t;
            }
            if (!g_known) {
                me->G = tB + tA * carry;
                __threadfence();
                st_release(&me->flag, 2);
            }
        }
        s_carry = carry;
    }
    __syncthreads();

    const bool want_moments = (p.rms != nullptr) || (p.batch_moments != nullptr);
    double g = eB + eA * s_carry;  // adv just right of this thread's items
    double advv[kItems], retv[kItems];
    // moments of the un-scaled returns: pivot-shifted sums (one division per thread, not per item)
    double mn = 0.0, pivot = 0.0, s1 = 0.0, s2 = 0.0;
    const bool scaled = (p.rms != nullptr);
#pragma unroll
    for (int j = kItems - 1; j >= 0; --j) {
        g = d[j] + a[j] * g;
        advv[j] = g;
        const double r = g + vs[j];  // un-scaled return (algorithm_base.py:717)
        retv[j] = scaled ? r / scale : r;   // a2c.py:146
        if (want_moments && base + j < p.n) {
            if (mn == 0.0) pivot = r;
            const double dl = r - pivot;
            mn += 1.0; s1 += dl; s2 += dl * dl;
        }
    }
    double mm = 0.0, mM = 0.0;
    if (mn > 0.0) { mm = pivot + s1 / mn; mM = s2 - s1 * s1 / mn; if (mM < 0.0) mM = 0.0; }
    if (p.vec_ok && base + kItems <= p.n) {
        store8<TO>(static_cast<TO*>(p.adv_out), base, advv);
        store8<TO>(static_cast<TO*>(p.ret_out), base, retv);
    } else {
#pragma unroll
        for (int j = 0; j < kItems; ++j) {
            if (base + j < p.n) {
                static_cast<TO*>(p.adv_out)[base + j] = (TO)advv[j];
                static_cast<TO*>(p.ret_out)[base + j] = (TO)retv[j];
            }
        }
    }

    if (!want_moments) return;
    // (count, mean, M2) of un-scaled returns: warp -> CTA -> (last CTA) whole array
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        const double n2 = tsb::shfl_xor_f64(mn, off);
        const double m2 = tsb::shfl_xor_f64(mm, off);
        const double M2 = tsb::shfl_xor_f64(mM, off);
        // symmetric merge so that all lanes agree
        const double n = mn + n2;
        if (n > 0.0) {
            const double dl = m2 - mm;
            const double mean = (mn * mm + n2 * m2) / n;
            mM = mM + M2 + dl * dl * (mn * n2 / n);
            mm = mean;
        }
        mn = n;
    }
    if (lane == 0) { s_mn[warp] = mn; s_mm[warp] = mm; s_mM[warp] = mM; }
    __syncthreads();
    if (tid == 0) {
        double n1 = 0.0, m1 = 0.0, M1 = 0.0;
        for (int w = 0; w < kWarps; ++w) chan_merge(n1, m1, M1, s_mn[w], s_mm[w], s_mM[w]);
        TileMoments* tm = p.moments + tile;
        tm->n = n1; tm->mean = m1; tm->M2 = M1;
        __threadfence();
        const int prev = atomicAdd(&p.hdr->done, 1);
        s_is_last = (prev == p.num_tiles - 1);
    }
    __syncthreads();
    if (!s_is_last || warp != 0) return;
    __threadfence();
    // last CTA: fixed-order merge of all tile partials, then RunningMeanStd.update
    double n1 = 0.0, m1 = 0.0, M1 = 0.0;
    for (int t = lane; t < p.num_tiles; t += 32) {
        const volatile TileMoments* tm = p.moments + t;
        chan_merge(n1, m1, M1, tm->n, tm->mean, tm->M2);
    }
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
        const double n2 = tsb::shfl_down_f64(n1, off);
        const double m2 = tsb::shfl_down_f64(m1, off);
        const double M2 = tsb::shfl_down_f64(M1, off);
        if (lane + off < 32) chan_merge(n1, m1, M1, n2, m2, M2);
    }
    if (lane == 0 && p.batch_moments) {  // multi-GPU: the caller merges moments across ranks
        p.batch_moments[0] = n1; p.batch_moments[1] = m1; p.batch_moments[2] = M1;
    } else if (lane == 0 && n1 > 0.0) {
        // utils/statistics.py:99-114
        const double batch_mean = m1, batch_var = M1 / n1, batch_count = n1;
        const double mean = p.rms[0], var = p.rms[1], count = p.rms[2];
        const double delta = batch_mean - mean;
        const double total = count + batch_count;
        const double new_mean = mean + delta * batch_count / total;
        const double m_a = var * count;
        const double m_b = batch_var * batch_count;
        const double m_2 = m_a + m_b + delta * delta * count * batch_count / total;
        p.rms[0] = new_mean;
        p.rms[1] = m_2 / total;
        p.rms[2] = total;
    }
}

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }
inline bool aligned8(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 7u) == 0; }

}  // namespace

namespace {
__global__ void rms_merge_kernel(double* __restrict__ rms, const double* __restrict__ moments, int parts) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    double n1 = 0.0, m1 = 0.0, M1 = 0.0;
    for (int k = 0; k < parts; ++k) chan_merge(n1, m1, M1, moments[3 * k], moments[3 * k + 1], moments[3 * k + 2]);
    if (n1 <= 0.0) return;
    const double batch_mean = m1, batch_var = M1 / n1, batch_count = n1;
    const double mean = rms[0], var = rms[1], count = rms[2];
    const double delta = batch_mean - mean;
    const double total = count + batch_count;
    rms[0] = mean + delta * batch_count / total;
    rms[1] = (var * count + batch_var * batch_count + delta * delta * count * batch_count / total) / total;
    rms[2] = total;
}
}  // namespace

extern "C" int ts_rms_merge(double* rms_state, const double* moments, int32_t parts, ts_stream_t stream) {
    TS_REQUIRE(rms_state && moments && parts >= 1, "ts_rms_merge: bad arguments");
    rms_merge_kernel<<<1, 32, 0, tsb::as_stream(stream)>>>(rms_state, moments, parts);
    return tsb::check_launch("ts_rms_merge");
}

extern "C" size_t ts_gae_workspace_bytes(int64_t n) {
    const int64_t tiles = (n + kTile - 1) / kTile;
    return sizeof(WsHeader) + (size_t)tiles * (sizeof(TileState) + sizeof(TileMoments));
}

extern "C" int ts_gae(const void* v_s, const void* v_s_next, int v_dtype, const double* rew,
                      const uint8_t* terminated, const uint8_t* truncated,
                      const uint8_t* extra_end, int terminated_ends, int64_t n, double gamma,
                      double lam, double* rms_state, double rms_eps, double* batch_moments_out,
                      void* adv_out, void* ret_out, int out_dtype, void* workspace,
                      ts_stream_t stream) {
    TS_REQUIRE(n >= 0, "ts_gae: negative n");
    if (n == 0) return 0;
    TS_REQUIRE(v_s && v_s_next && rew && adv_out && ret_out && workspace, "ts_gae: null pointer");
    TS_REQUIRE(v_dtype == TS_F32 || v_dtype == TS_F64, "ts_gae: bad v_dtype %d", v_dtype);
    TS_REQUIRE(out_dtype == TS_F32 || out_dtype == TS_F64, "ts_gae: bad out_dtype %d", out_dtype);
    TS_REQUIRE(n <= (int64_t)kTile * 0x7fffffff, "ts_gae: n too large");
    cudaStream_t st = tsb::as_stream(stream);
    GaeParams p;
    p.v_s = v_s; p.v_n = v_s_next; p.rew = rew;
    p.terminated = terminated; p.truncated = truncated; p.extra_end = extra_end;
    p.terminated_ends = terminated_ends;
    p.n = n;
    p.num_tiles = (int)((n + kTile - 1) / kTile);
    p.gamma = gamma; p.lam = lam;
    p.rms = rms_state; p.rms_eps = rms_eps; p.batch_moments = batch_moments_out;
    p.adv_out = adv_out; p.ret_out = ret_out;
    p.vec_ok = aligned16(v_s) && aligned16(v_s_next) && aligned16(rew) && aligned16(adv_out) &&
               aligned16(ret_out) && (!terminated || aligned8(terminated)) &&
               (!truncated || aligned8(truncated)) && (!extra_end || aligned8(extra_end));
    char* ws = static_cast<char*>(workspace);
    p.hdr = reinterpret_cast<WsHeader*>(ws);
    p.tiles = reinterpret_cast<TileState*>(ws + sizeof(WsHeader));
    p.moments = reinterpret_cast<TileMoments*>(ws + sizeof(WsHeader) +
                                               (size_t)p.num_tiles * sizeof(TileState));
    TS_CUDA(cudaMemsetAsync(ws, 0, sizeof(WsHeader) + (size_t)p.num_tiles * sizeof(TileState), st));
    dim3 grid(p.num_tiles), block(kThreads);
    if (v_dtype == TS_F32 && out_dtype == TS_F32) gae_scan_kernel<float, float><<<grid, block, 0, st>>>(p);
    else if (v_dtype == TS_F32) gae_scan_kernel<float, double><<<grid, block, 0, st>>>(p);
    else if (out_dtype == TS_F32) gae_scan_kernel<double, float><<<grid, block, 0, st>>>(p);
    else gae_scan_kernel<double, double><<<grid, block, 0, st>>>(p);
    return tsb::check_launch("ts_gae");
}
