// Discrete BCQ arithmetic (algorithm/imitation/discrete_bcq.py): the per-row pieces between the Q / imitator head GEMMs of the
// forward and their backward GEMMs.  The GEMMs themselves are the layered-network launches of net_gemm.cu.
//
// Reference: tianshou/algorithm/imitation/discrete_bcq.py:115-118 (the imitator's mask on the arg-max), :228-234 (the target
// Q_old(s', argmax_a masked Q(s', a))), :244-252 (smooth-L1 Q loss, NLL imitation loss, logit penalty).
#include <float.h>
#include <math.h>

#include "common.cuh"
#include "quantile.cuh"
#include "row_sums.cuh"

namespace {

using tsb::argmax_before;
using tsb::kRowsPerBlock;
using tsb::kRowThreads;

// Per row b: mask_a = (logits[b][a] - max_a logits[b]) < log_tau, a* = first argmax_a (q_online[b][a] - FLT_MAX * mask_a) in fp32
// as torch evaluates it, out[b] = q_old[b][a*].  The arg-max-logit action is never masked (log_tau < 0), so a* always exists.
__global__ void __launch_bounds__(kRowThreads) discrete_bcq_target_kernel(
        const float* __restrict__ q_online, const float* __restrict__ logits, const float* __restrict__ q_old, float log_tau, int64_t B,
        int A, float* __restrict__ out, int64_t* __restrict__ act_out) {
    const int lane = tsb::lane_id();
    for (int64_t b = (int64_t)blockIdx.x * kRowsPerBlock + tsb::warp_id(); b < B; b += (int64_t)gridDim.x * kRowsPerBlock) {
        const float* z = logits + b * A;
        const float* q = q_online + b * A;
        float mx = -INFINITY;
        for (int a = lane; a < A; a += 32) mx = fmaxf(mx, z[a]);
        mx = tsb::warp_max(mx);
        float bv = 0.0f;
        int bi = -1;
        for (int a = lane; a < A; a += 32) {
            const float mask = (z[a] - mx) < log_tau ? 1.0f : 0.0f;
            const float v = q[a] - FLT_MAX * mask;
            if (argmax_before(v, a, bv, bi)) { bv = v; bi = a; }
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, bv, off);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, off);
            if (oi >= 0 && argmax_before(ov, oi, bv, bi)) { bv = ov; bi = oi; }
        }
        if (lane == 0) {
            out[b] = q_old[b * A + bi];
            if (act_out) act_out[b] = bi;
        }
    }
}

// Per row b, with z = logits[b], p = softmax(z), td = q[b][act[b]] - returns[b]:
//   rows[0][b] = smooth_l1(td) (beta 1: 0.5 td^2 below |td| = 1, |td| - 0.5 from it on)
//   rows[1][b] = -(z[act] - logsumexp(z))
//   rows[2][b] = sum_a z_a^2
//   dq[b][a]      = 1[a == act] * (|td| < 1 ? td : sign(td)) * inv_b
//   dlogits[b][a] = (p_a - 1[a == act]) * inv_b + reg_scale * z_a          (reg_scale = 2 penalty / (B A))
__global__ void __launch_bounds__(kRowThreads) discrete_bcq_rows_kernel(
        const float* __restrict__ q, const float* __restrict__ logits, const int64_t* __restrict__ act, const float* __restrict__ returns,
        int64_t B, int A, float inv_b, float reg_scale, float* __restrict__ dq, float* __restrict__ dlogits, float* __restrict__ rows) {
    const int lane = tsb::lane_id();
    for (int64_t b = (int64_t)blockIdx.x * kRowsPerBlock + tsb::warp_id(); b < B; b += (int64_t)gridDim.x * kRowsPerBlock) {
        const float* z = logits + b * A;
        const int ab = (int)act[b];
        const float td = q[b * A + ab] - returns[b];
        const float atd = fabsf(td);
        const float gq = (atd < 1.0f ? td : copysignf(1.0f, td)) * inv_b;
        float mx = -INFINITY;
        for (int a = lane; a < A; a += 32) mx = fmaxf(mx, z[a]);
        mx = tsb::warp_max(mx);
        float s = 0.0f, sq = 0.0f;
        for (int a = lane; a < A; a += 32) {
            s += expf(z[a] - mx);
            sq += z[a] * z[a];
        }
        s = tsb::warp_sum(s);
        sq = tsb::warp_sum(sq);
        const float lse = logf(s) + (isinf(mx) ? 0.0f : mx);
        for (int a = lane; a < A; a += 32) {
            const float hit = a == ab ? 1.0f : 0.0f;
            dq[b * A + a] = hit * gq;
            dlogits[b * A + a] = (expf(z[a] - mx) / s - hit) * inv_b + reg_scale * z[a];
        }
        if (lane == 0) {
            rows[b] = atd < 1.0f ? 0.5f * td * td : atd - 0.5f;
            rows[B + b] = -(z[ab] - lse);
            rows[2 * B + b] = sq;
        }
    }
}

}  // namespace

extern "C" int ts_discrete_bcq_target(const float* q_online, const float* logits, const float* q_old, float log_tau, int64_t B,
                                      int32_t A, float* out, int64_t* act_out, ts_stream_t stream) {
    TS_REQUIRE(q_online && logits && q_old && out && B >= 0 && A >= 1, "ts_discrete_bcq_target: bad argument");
    if (B == 0) return 0;
    discrete_bcq_target_kernel<<<tsb::row_grid(B), kRowThreads, 0, tsb::as_stream(stream)>>>(q_online, logits, q_old, log_tau, B, A,
                                                                                            out, act_out);
    return tsb::check_launch("ts_discrete_bcq_target");
}

extern "C" int ts_discrete_bcq_rows(const float* q, const float* logits, const int64_t* act, const float* returns, int64_t B,
                                    int32_t A, float penalty, float* dq, float* dlogits, float* rows, float* losses,
                                    ts_stream_t stream) {
    TS_REQUIRE(q && logits && act && returns && dq && dlogits && rows && losses && B >= 1 && A >= 1,
               "ts_discrete_bcq_rows: bad argument");
    cudaStream_t st = tsb::as_stream(stream);
    const float inv_b = 1.0f / (float)B;
    const float inv_ba = (float)(1.0 / ((double)B * (double)A));
    discrete_bcq_rows_kernel<<<tsb::row_grid(B), kRowThreads, 0, st>>>(q, logits, act, returns, B, A, inv_b, 2.0f * penalty * inv_ba, dq,
                                                                      dlogits, rows);
    if (tsb::check_launch("ts_discrete_bcq_rows")) return 1;
    tsb::row_sums3_kernel<<<1, tsb::kRowSumThreads, 0, st>>>(rows, B, inv_b, inv_b, inv_ba, 1.0f, 1.0f, penalty, losses);
    return tsb::check_launch("ts_discrete_bcq_rows/sums");
}
