// GAIL discriminator arithmetic (algorithm/imitation/gail.py): the per-row pieces between the discriminator's forward GEMMs
// and its backward GEMMs.  The GEMMs themselves are the layered-network launches of net_gemm.cu.
//
// Reference: tianshou/algorithm/imitation/gail.py:193-206 (rewards -logsigmoid(-D(s, a)) before GAE) and :214-248 (the
// discriminator loss -logsigmoid(-logits_pi).mean() + -logsigmoid(logits_exp).mean(), its two accuracies), torch's
// log_sigmoid forward / backward (aten LogSigmoid: min(0, z) - log1p(exp(-|z|))).
#include <math.h>

#include "common.cuh"

namespace {

constexpr int kRowThreads = 256;
constexpr int kDiscThreads = 1024;      // one block: the loss sums and the counts are reduced in a fixed order

// torch's log_sigmoid(z) in its own formulation (not softplus: the two differ by up to 1e-6 in fp32)
__device__ __forceinline__ float log_sigmoid(float z) {
    return fminf(0.0f, z) - log1pf(expf(-fabsf(z)));
}

// d log_sigmoid(z) / dz = sigmoid(-z), as torch's log_sigmoid backward evaluates it from e = exp(-|z|)
__device__ __forceinline__ float log_sigmoid_grad(float z) {
    const float e = expf(-fabsf(z));
    const float t = e / (1.0f + e);
    return z < 0.0f ? 1.0f - t : t;
}

// rew[i] = -log_sigmoid(-logits[i]) in fp32, widened (gail.py:204: to_numpy of an fp32 tensor, then GAE in f64)
__global__ void gail_reward_kernel(const float* __restrict__ logits, int64_t n, double* __restrict__ rew) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        rew[i] = (double)(-log_sigmoid(-logits[i]));
}

// Fixed-order sum over the block of four doubles; thread 0 receives the totals.
__device__ void block_sum4(double v[4], double (*sh)[4] /* [32][4] */) {
    for (int k = 0; k < 4; ++k)
        for (int o = 16; o > 0; o >>= 1) v[k] += tsb::shfl_down_f64(v[k], o);
    if (tsb::lane_id() == 0)
        for (int k = 0; k < 4; ++k) sh[tsb::warp_id()][k] = v[k];
    __syncthreads();
    if (tsb::warp_id() == 0) {
        const bool live = tsb::lane_id() < (int)(blockDim.x >> 5);
        for (int k = 0; k < 4; ++k) {
            double t = live ? sh[tsb::lane_id()][k] : 0.0;
            for (int o = 16; o > 0; o >>= 1) t += tsb::shfl_down_f64(t, o);
            v[k] = t;
        }
    }
}

// logits [n_pi | n_exp] -> dlogits (d loss / d logit) and stats_row = (loss, acc_pi, acc_exp, n_pi)
__global__ void gail_disc_kernel(const float* __restrict__ logits, int64_t n_pi, int64_t n_exp, float* __restrict__ dlogits,
                                 float* __restrict__ stats_row) {
    __shared__ double sh[32][4];
    const float inv_pi = 1.0f / (float)n_pi, inv_exp = 1.0f / (float)n_exp;
    double v[4] = {0.0, 0.0, 0.0, 0.0};      // sum loss_pi rows, sum loss_exp rows, #(x_pi < 0), #(x_exp > 0)
    const int64_t n = n_pi + n_exp;
    for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
        const float x = logits[i];
        if (i < n_pi) {         // -log_sigmoid(-x): d / dx = sigmoid(x) = log_sigmoid_grad(-x)
            v[0] += (double)(-log_sigmoid(-x));
            v[2] += x < 0.0f ? 1.0 : 0.0;
            dlogits[i] = log_sigmoid_grad(-x) * inv_pi;
        } else {                // -log_sigmoid(x): d / dx = -sigmoid(-x)
            v[1] += (double)(-log_sigmoid(x));
            v[3] += x > 0.0f ? 1.0 : 0.0;
            dlogits[i] = -log_sigmoid_grad(x) * inv_exp;
        }
    }
    block_sum4(v, sh);
    if (threadIdx.x == 0) {
        const float loss_pi = (float)(v[0] / (double)n_pi), loss_exp = (float)(v[1] / (double)n_exp);
        stats_row[0] = loss_pi + loss_exp;                   // gail.py:232: two fp32 means, added in fp32
        stats_row[1] = (float)v[2] / (float)n_pi;           // (logits_pi < 0).float().mean()
        stats_row[2] = (float)v[3] / (float)n_exp;          // (logits_exp > 0).float().mean()
        stats_row[3] = (float)n_pi;
    }
}

inline unsigned row_grid(int64_t n) {
    int64_t b = (n + kRowThreads - 1) / kRowThreads;
    const int64_t cap = (int64_t)tsb::num_sms() * 16;
    return (unsigned)(b > cap ? cap : (b < 1 ? 1 : b));
}

}  // namespace

extern "C" int ts_gail_reward_rows(const float* logits, int64_t n, double* rew, ts_stream_t stream) {
    TS_REQUIRE(logits && rew && n >= 0, "ts_gail_reward_rows: bad argument");
    if (n == 0) return 0;
    gail_reward_kernel<<<row_grid(n), kRowThreads, 0, tsb::as_stream(stream)>>>(logits, n, rew);
    return tsb::check_launch("ts_gail_reward_rows");
}

extern "C" int ts_gail_disc_rows(const float* logits, int64_t n_pi, int64_t n_exp, float* dlogits, float* stats_row,
                                 ts_stream_t stream) {
    TS_REQUIRE(logits && dlogits && stats_row && n_pi > 0 && n_exp > 0, "ts_gail_disc_rows: bad argument");
    gail_disc_kernel<<<1, kDiscThreads, 0, tsb::as_stream(stream)>>>(logits, n_pi, n_exp, dlogits, stats_row);
    return tsb::check_launch("ts_gail_disc_rows");
}
