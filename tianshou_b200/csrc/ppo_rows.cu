// Per-row PPO / A2C loss arithmetic on the head outputs of a LAYERED actor-critic (networks outside the fused 17-64-64
// kernels' shape envelope run layer by layer on the tensor-core GEMM of net_gemm.cu; this kernel is the loss in between the
// forward and the backward GEMMs).  One thread per minibatch row; outputs are the gradients w.r.t. the head outputs.
//
// Reference: tianshou/algorithm/modelfree/ppo.py:179-216 (surrogate, dual clip, value clip, entropy), a2c.py:262-270,
// reinforce.py:167-192 + utils/net/discrete.py:69-92 (Categorical(probs = softmax(logits))), continuous.py:220-238 +
// torch.distributions.Normal (diagonal Gaussian, state-independent sigma = exp(logstd)).
#include <math.h>

#include "common.cuh"
#include "ppo_math.cuh"

namespace {

constexpr int kMaxA = ppo::kCatMaxA;

// head: [B][A] (mu or logits); value: [B]; act: [B][A] (Gaussian) or [B] (categorical, float-coded index).
// Outputs (all nullable except logp_out): logp_out [B]; dhead [B][A]; dvalue [B]; dlogstd_rows [B][A] (Gaussian: per-row
// d loss / d logstd including the entropy term, summed by ts_net_colsum); loss_rows [B][3] = (surrogate objective, value loss,
// entropy) per row.
__global__ void ppo_rows_kernel(const float* __restrict__ head, const float* __restrict__ value, const float* __restrict__ logstd,
                                const float* __restrict__ act, const float* __restrict__ adv, const float* __restrict__ ret,
                                const float* __restrict__ logp_old, const float* __restrict__ v_s, int64_t B, int A, int categorical,
                                const ts_ppo_hparams hp, int64_t global_rows, const float* __restrict__ adv_moments,
                                float* __restrict__ logp_out, float* __restrict__ dhead, float* __restrict__ dvalue,
                                float* __restrict__ dlogstd_rows, float* __restrict__ loss_rows) {
    const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const bool grads = dhead != nullptr;
    const ppo::Scalars sc = ppo::make_scalars(hp, global_rows, adv_moments);
    float lp = 0.0f, ent = 0.0f, obj = 0.0f, gl = 0.0f;
    if (categorical) {
        float z[kMaxA];
        for (int a = 0; a < A; ++a) z[a] = head[b * A + a];
        const int action = (int)act[b];
        ppo::Cat c;
        ppo::cat_forward(z, A, action, c, lp, ent);
        if (grads) {
            ppo::actor_row(sc, lp, logp_old[b], adv[b], obj, gl);
            float dz[kMaxA];
            ppo::cat_backward(c, A, action, gl, -sc.ent_coef * sc.inv_b, dz);
            for (int a = 0; a < A; ++a) dhead[b * A + a] = dz[a];
        }
    } else {
        for (int a = 0; a < A; ++a) {
            const float sg = expf(logstd[a]);
            lp += ppo::normal_logp_term(act[b * A + a], head[b * A + a], sg);
            ent += ppo::normal_entropy_term(sg);
        }
        if (grads) {
            ppo::actor_row(sc, lp, logp_old[b], adv[b], obj, gl);
            for (int a = 0; a < A; ++a) {
                float dmu, dls;
                ppo::normal_backward(act[b * A + a], head[b * A + a], expf(logstd[a]), gl, dmu, dls);
                dhead[b * A + a] = dmu;
                if (dlogstd_rows) dlogstd_rows[b * A + a] = dls - sc.ent_coef * sc.inv_b;
            }
        }
    }
    logp_out[b] = lp;
    if (grads) {
        float vf_row = 0.0f, dv = 0.0f;
        ppo::critic_row(sc, value[b], ret[b], v_s[b], vf_row, dv);
        dvalue[b] = dv;
        if (loss_rows) { loss_rows[b * 3] = obj; loss_rows[b * 3 + 1] = vf_row; loss_rows[b * 3 + 2] = ent; }
    }
}

// (sum obj, sum vf, sum ent) -> stats row entries 0..3 (ppo::loss_row) and 5 (rows)
__global__ void ppo_stats_kernel(const float* __restrict__ loss_rows, int64_t B, const ts_ppo_hparams hp, float* __restrict__ stats_row) {
    __shared__ float s[3][256];
    float a0 = 0.f, a1 = 0.f, a2 = 0.f;
    for (int64_t i = threadIdx.x; i < B; i += 256) { a0 += loss_rows[i * 3]; a1 += loss_rows[i * 3 + 1]; a2 += loss_rows[i * 3 + 2]; }
    s[0][threadIdx.x] = a0; s[1][threadIdx.x] = a1; s[2][threadIdx.x] = a2;
    __syncthreads();
    for (int off = 128; off > 0; off >>= 1) {
        if ((int)threadIdx.x < off) {
#pragma unroll
            for (int k = 0; k < 3; ++k) s[k][threadIdx.x] += s[k][threadIdx.x + off];
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        const float rows = (float)B;
        ppo::loss_row(s[0][0], s[1][0], s[2][0], rows, hp, stats_row);
        stats_row[5] = rows;
    }
}

}  // namespace

extern "C" int ts_ppo_rows(const float* head, const float* value, const float* logstd, const float* act, const float* adv,
                           const float* ret, const float* logp_old, const float* v_s, int64_t B, int32_t A, int32_t categorical,
                           const ts_ppo_hparams* hp, int64_t global_rows, const float* adv_moments, float* logp_out, float* dhead,
                           float* dvalue, float* dlogstd_rows, float* loss_rows, ts_stream_t stream) {
    TS_REQUIRE(head && act && logp_out && hp && A >= 1 && A <= kMaxA, "ts_ppo_rows: bad argument (act_dim <= %d)", kMaxA);
    TS_REQUIRE(categorical || logstd, "ts_ppo_rows: Gaussian head needs logstd");
    TS_REQUIRE(!dhead || (value && adv && ret && logp_old && v_s && dvalue), "ts_ppo_rows: gradient mode needs the row data");
    if (B <= 0) return 0;
    ppo_rows_kernel<<<(unsigned)((B + 127) / 128), 128, 0, tsb::as_stream(stream)>>>(
        head, value, logstd, act, adv, ret, logp_old, v_s, B, A, categorical, *hp, global_rows, adv_moments, logp_out, dhead, dvalue,
        dlogstd_rows, loss_rows);
    return tsb::check_launch("ts_ppo_rows");
}

extern "C" int ts_ppo_rows_stats(const float* loss_rows, int64_t B, const ts_ppo_hparams* hp, float* stats_row, ts_stream_t stream) {
    TS_REQUIRE(loss_rows && hp && stats_row && B > 0, "ts_ppo_rows_stats: bad argument");
    ppo_stats_kernel<<<1, 256, 0, tsb::as_stream(stream)>>>(loss_rows, B, *hp, stats_row);
    return tsb::check_launch("ts_ppo_rows_stats");
}
