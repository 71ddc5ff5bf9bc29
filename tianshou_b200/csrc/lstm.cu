// The LSTM cell of the recurrent Q-network (algorithm/recurrent.py): one time step forward and one time step backward.  The GEMMs
// around it -- the input projection of a whole layer, the recurrent product of each step, the input gradient of each step and
// the weight gradients over all steps -- are the layered-network launches of net_gemm.cu.
//
// Reference: torch.nn.LSTM as tianshou/utils/net/common.py Recurrent builds it (gate chunks i, f, g, o of 4H rows;
// c_t = f * c_{t-1} + i * g, h_t = o * tanh(c_t); both bias vectors added to the pre-activations).
#include <math.h>

#include "common.cuh"

namespace {

constexpr int kThreads = 256;

inline unsigned grid_for(int64_t items) {
    int64_t b = (items + kThreads - 1) / kThreads;
    const int64_t cap = (int64_t)tsb::num_sms() * 8;
    return (unsigned)(b > cap ? cap : (b < 1 ? 1 : b));
}

__device__ __forceinline__ float sigmoid_full(float x) { return 1.0f / (1.0f + expf(-x)); }

// One thread per (b, j): the four pre-activations of hidden unit j plus b_hh, the activated gates, c_t and h_t.
__global__ void __launch_bounds__(kThreads) lstm_cell_kernel(const float* __restrict__ pre, const float* __restrict__ b_hh,
                                                             const float* __restrict__ c_prev, int64_t B, int H,
                                                             float* __restrict__ gates, float* __restrict__ c,
                                                             float* __restrict__ h) {
    const int64_t H4 = 4 * (int64_t)H;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < B * H; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t b = e / H;
        const int j = (int)(e - b * H);
        const float* p = pre + b * H4 + j;
        float* gt = gates + b * H4 + j;
        const float i = sigmoid_full(p[0] + b_hh[j]);
        const float f = sigmoid_full(p[H] + b_hh[H + j]);
        const float g = tanhf(p[2 * H] + b_hh[2 * H + j]);
        const float o = sigmoid_full(p[3 * H] + b_hh[3 * H + j]);
        gt[0] = i;
        gt[H] = f;
        gt[2 * H] = g;
        gt[3 * H] = o;
        const float ct = c_prev ? f * c_prev[e] + i * g : i * g;
        c[e] = ct;
        h[e] = o * tanhf(ct);
    }
}

// One thread per (b, j).  dc_t and dc_prev may be the same array: each element is read before it is written, by one thread.
__global__ void __launch_bounds__(kThreads) lstm_cell_bwd_kernel(const float* __restrict__ gates, const float* __restrict__ c,
                                                                 const float* __restrict__ c_prev, const float* __restrict__ dh,
                                                                 const float* dc, int64_t B, int H, float* __restrict__ dgates,
                                                                 float* dc_prev) {
    const int64_t H4 = 4 * (int64_t)H;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < B * H; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t b = e / H;
        const int j = (int)(e - b * H);
        const float* gt = gates + b * H4 + j;
        const float i = gt[0], f = gt[H], g = gt[2 * H], o = gt[3 * H];
        const float th = tanhf(c[e]);
        const float dht = dh[e];
        const float dct = (dc ? dc[e] : 0.0f) + dht * o * (1.0f - th * th);
        const float cp = c_prev ? c_prev[e] : 0.0f;
        float* dg = dgates + b * H4 + j;
        dg[0] = dct * g * i * (1.0f - i);
        dg[H] = dct * cp * f * (1.0f - f);
        dg[2 * H] = dct * i * (1.0f - g * g);
        dg[3 * H] = dht * th * o * (1.0f - o);
        if (dc_prev) dc_prev[e] = dct * f;
    }
}

}  // namespace

extern "C" int ts_lstm_cell(const float* pre, const float* b_hh, const float* c_prev, int64_t B, int32_t H, float* gates, float* c,
                            float* h, ts_stream_t stream) {
    TS_REQUIRE(pre && b_hh && gates && c && h && B >= 1 && H >= 1, "ts_lstm_cell: bad argument");
    lstm_cell_kernel<<<grid_for(B * H), kThreads, 0, tsb::as_stream(stream)>>>(pre, b_hh, c_prev, B, H, gates, c, h);
    return tsb::check_launch("ts_lstm_cell");
}

extern "C" int ts_lstm_cell_bwd(const float* gates, const float* c, const float* c_prev, const float* dh, const float* dc, int64_t B,
                                int32_t H, float* dgates, float* dc_prev, ts_stream_t stream) {
    TS_REQUIRE(gates && c && dh && dgates && B >= 1 && H >= 1, "ts_lstm_cell_bwd: bad argument");
    lstm_cell_bwd_kernel<<<grid_for(B * H), kThreads, 0, tsb::as_stream(stream)>>>(gates, c, c_prev, dh, dc, B, H, dgates, dc_prev);
    return tsb::check_launch("ts_lstm_cell_bwd");
}
