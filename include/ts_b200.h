/*
 * ts_b200.h -- C ABI of the GPU-native (H100, sm_90a) policy-update hot path for Tianshou-style RL.
 *
 * The reference (thu-ml/tianshou 2.0.1) has NO FFI: its hot path is Python + numba @njit +
 * stock torch ops.  This header declares the entry points a maintainer binds (ctypes / cffi,
 * see INTEGRATION.md) in place of those numba kernels and torch loops.  Every function
 *   - takes plain device pointers, sizes and a cudaStream_t (passed as void*),
 *   - is asynchronous on that stream (no host sync, no allocation, no hidden global state),
 *   - returns 0 on success, non-zero on error; ts_last_error() gives the thread-local message.
 * Pointers are DEVICE pointers unless a parameter is documented as "host".  "u8" flags are
 * numpy/torch bool storage (one byte, 0/1).
 *
 * Each declaration cites the reference code it replaces (path:line in thu-ml/tianshou 2.0.1).
 */
#ifndef TS_B200_H_
#define TS_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TS_B200_ABI_VERSION 1

typedef void* ts_stream_t; /* cudaStream_t */

/* dtype tags for the few polymorphic entry points */
enum { TS_F32 = 0, TS_F64 = 1 };

int ts_version(void);
const char* ts_last_error(void);
/* number of kernel launches issued through this library by the calling process (for bench.py's
 * "gpu_launches" claim); ts_reset_launch_count() zeroes it. */
int64_t ts_launch_count(void);
void ts_reset_launch_count(void);

/* ------------------------------------------------------------------------------------------
 * (1) GAE: segmented reverse scan.
 * Replaces numba `_gae` (tianshou/algorithm/algorithm_base.py:1085-1140) together with the
 * value-mask / end-flag / return-scaling arithmetic around it in
 * `Algorithm.compute_episodic_return` (:704-719) and
 * `ActorCriticOnPolicyAlgorithm._add_returns_and_advantages` (modelfree/a2c.py:131-152):
 *
 *   s      = rms_state ? sqrt(rms_state.var + rms_eps) : 1         (return_scaling un-normalise)
 *   vs     = v_s[i] * s ;  vn = v_s_next[i] * s * (terminated ? !terminated[i] : 1)
 *   delta  = rew[i] + vn*gamma - vs
 *   end    = (truncated?truncated[i]:0) | (terminated_ends?terminated[i]:0) | (extra_end?extra_end[i]:0)
 *   adv[i] = delta + (1-end)*gamma*lam * adv[i+1]        (adv[n] = 0; f64 accumulate)
 *   ret[i] = (adv[i] + vs) / s
 * and, if rms_state != NULL, merges mean/var/count of the UN-scaled returns (adv+vs) into
 * rms_state with Chan's formula exactly as `RunningMeanStd.update`
 * (tianshou/utils/statistics.py:99-114) -- after every block has read the old var.
 *
 * v_s / v_s_next: n values of v_dtype (TS_F32|TS_F64).  rew: n f64 (the buffer stores float64,
 * data/buffer/manager.py:183).  terminated / truncated / extra_end: n u8, each nullable.
 * terminated_ends: if non-zero `terminated` also ends a segment (the normal case); the value
 * mask always uses it when non-NULL.  adv_out / ret_out: n values of out_dtype.
 * rms_state: device double[3] = {mean, var, count} (nullable).
 * batch_moments_out: see ts_rms_merge below (nullable).
 * workspace: device scratch of ts_gae_workspace_bytes(n) bytes (contents ignored).
 * ------------------------------------------------------------------------------------------ */
size_t ts_gae_workspace_bytes(int64_t n);
int ts_gae(const void* v_s, const void* v_s_next, int v_dtype, const double* rew,
           const uint8_t* terminated, const uint8_t* truncated, const uint8_t* extra_end,
           int terminated_ends, int64_t n, double gamma, double lam, double* rms_state,
           double rms_eps, double* batch_moments_out, void* adv_out, void* ret_out, int out_dtype,
           void* workspace, ts_stream_t stream);
/* Multi-GPU return scaling: when batch_moments_out (device double[3] = {count, mean, M2} of this
 * call's un-scaled returns) is non-NULL, ts_gae writes it and leaves rms_state untouched; the
 * caller all-gathers the triples and folds them in rank order with ts_rms_merge so that every
 * replica holds the same RunningMeanStd (SURVEY 8e). */
int ts_rms_merge(double* rms_state, const double* moments /* parts x 3 */, int32_t parts,
                 ts_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * (2) n-step return: windowed gather-reduce.
 * Replaces numba `_nstep_return` (algorithm_base.py:1160-1222) and the whole-buffer
 * `end_flag_B = done.copy(); end_flag_B[unfinished] = True` preparation (:799-800).
 *   rew: B f64 (whole buffer), end_flag: B u8, target_q: I*A f32 (already value-masked),
 *   stacked_idx: n_step rows of I int64 (row k = next^k(indices)), out: I*A of out_dtype.
 * Arithmetic is f64 in the reference's operation order (no FMA contraction) => bit-exact f64.
 * ------------------------------------------------------------------------------------------ */
int ts_nstep_return(const double* rew, const uint8_t* end_flag, const float* target_q,
                    const int64_t* stacked_idx, int64_t I, int64_t A, int32_t n_step,
                    double gamma, void* out, int out_dtype, ts_stream_t stream);

/* end_flag[i] = done[i] | (i is the last written slot of a non-empty sub-buffer); B = offset[E].
 * Replaces algorithm_base.py:799-800 + manager.py:85-91 without the host copy. */
int ts_buffer_end_flags(const uint8_t* done, const int64_t* offset, const int64_t* last_index,
                        const int64_t* lengths, int64_t E, uint8_t* end_flag_out,
                        ts_stream_t stream);

/* target_q[i, :] *= !terminated[idx[i]]  (Algorithm.value_mask, algorithm_base.py:633-651,798) */
int ts_value_mask_rows(float* target_q, const uint8_t* terminated, const int64_t* idx, int64_t I,
                       int64_t A, ts_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * (3) Replay-buffer index kernels (bit-exact int64).
 * Sub-buffer e owns slots [offset[e], offset[e+1]); lengths[e] = current size; last_index[e] =
 * absolute last-written slot.  A plain ReplayBuffer is the E=1 case.
 * Replace numba `_next_index` / `_prev_index` (tianshou/data/buffer/manager.py:339-363,
 * :311-336) and ReplayBuffer.next/prev (buffer_base.py:319-334).
 * ------------------------------------------------------------------------------------------ */
int ts_next_index(const int64_t* index, int64_t n, const int64_t* offset, int64_t E,
                  const uint8_t* done, const int64_t* last_index, const int64_t* lengths,
                  int64_t* out, ts_stream_t stream);
int ts_prev_index(const int64_t* index, int64_t n, const int64_t* offset, int64_t E,
                  const uint8_t* done, const int64_t* last_index, const int64_t* lengths,
                  int64_t* out, ts_stream_t stream);
/* out[k*n + i] = next^k(index[i]) for k = 0..n_step-1 (algorithm_base.py:775-779). */
int ts_stack_next_indices(const int64_t* index, int64_t n, int32_t n_step, const int64_t* offset,
                          int64_t E, const uint8_t* done, const int64_t* last_index,
                          const int64_t* lengths, int64_t* out, ts_stream_t stream);
/* ReplayBufferManager.unfinished_index (manager.py:85-91; buffer_base.py:314-317): ordered list
 * of the slots before each sub-buffer's insertion index whose `done` is false.  insertion_idx: device
 * int64[E] relative to the sub-buffer start (nullable: last_index is used, which is the same slot for buffers
 * filled by add() alone).  out: capacity E; count_out: device int64[1]. */
int ts_unfinished_index(const int64_t* offset, int64_t E, const uint8_t* done,
                        const int64_t* last_index, const int64_t* lengths, const int64_t* insertion_idx,
                        int64_t* out, int64_t* count_out, ts_stream_t stream);
/* sample_indices(0): all valid slots, sub-buffer-major, chronological inside each sub-buffer
 * (manager.py:217-234, buffer_base.py:519-525).  insertion_idx: device int64[E], every sub-buffer's
 * `_insertion_idx` relative to its own start (nullable: derived as last_index + 1, which is only right for
 * buffers filled by add() alone -- from_data() / dropnull() move it independently).  seg_start: device
 * int64[E+1] scratch that receives the exclusive prefix sum of lengths; out capacity >= sum(lengths);
 * total_out int64[1]. */
int ts_sample_all_indices(const int64_t* offset, int64_t E, const int64_t* last_index,
                          const int64_t* lengths, const int64_t* insertion_idx, int64_t* seg_start,
                          int64_t* out, int64_t out_capacity, int64_t* total_out, ts_stream_t stream);
/* mark[p] = 1 if idx[p] is in `members` (np.isin, algorithm_base.py:715).  table: device u8
 * scratch of table_size >= max slot + 1, left zeroed on return. */
int ts_mark_members(const int64_t* idx, int64_t n, const int64_t* members,
                    const int64_t* member_count /* device int64[1] */, int64_t member_capacity,
                    uint8_t* table, int64_t table_size, uint8_t* mark_out, ts_stream_t stream);
/* dst[p, :] = src[idx[p], :] for rows of row_bytes (multiple of 4) -- ReplayBuffer.__getitem__
 * (buffer_base.py:605-649) / Batch.__getitem__ (data/batch.py:714-738) for array leaves. */
int ts_gather_rows(const void* src, int64_t row_bytes, const int64_t* idx, int64_t n, void* dst,
                   ts_stream_t stream);

/* dst[idx[p]] = src[p] for p < n, rows of row_bytes bytes: the device side of the asynchronous buffer mirror --
 * ReplayBuffer.add (buffer_base.py:420-501, manager.py:131-198) writes one row per env at scattered slots; the
 * rows arrive contiguously from pinned staging.  idx entries must be distinct. */
int ts_scatter_rows(const void* src, int64_t row_bytes, const int64_t* idx, int64_t n, void* dst,
                    ts_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * (4) Sum tree for prioritized replay (f64 tree, bit-exact indices).
 * tree: double[2*bound], root at 1, leaves at [bound, bound+size) (data/utils/segtree.py:19-26).
 * Replace numba `_setitem` (:95-101), `_reduce` (:104-116), `_get_prefix_sum_idx` (:119-134).
 * ------------------------------------------------------------------------------------------ */
/* tree[bound+index[k]] = value[k] (duplicates: last wins), then parents re-summed bottom-up. */
int ts_segtree_setitem(double* tree, int64_t bound, const int64_t* index, const void* value,
                       int value_dtype, int64_t n, ts_stream_t stream);
/* out[0] = sum(leaves[start:end]) using the reference's bottom-up walk (same addition order). */
int ts_segtree_reduce(const double* tree, int64_t bound, int64_t start, int64_t end, double* out,
                      ts_stream_t stream);
/* out[k] = min i such that value[k] <= sum(leaves[0..i]) (ties go left).  value: n f64. */
int ts_segtree_prefix_sum_idx(const double* tree, int64_t bound, const double* value, int64_t n,
                              int64_t* out, ts_stream_t stream);
/* value[k] = u[k] * tree[1] then descent -- fuses `np.random.rand(bs) * weight.reduce()`
 * (data/buffer/prio.py:65-66); u stays a host-drawn numpy stream uploaded by the caller. */
int ts_segtree_sample(const double* tree, int64_t bound, const double* u, int64_t n, int64_t* out,
                      ts_stream_t stream);
/* PrioritizedReplayBuffer.update_weight (prio.py:81-90): w = |td|+eps; tree[idx] = w^alpha;
 * prio_minmax (device double[2] = {max_prio, min_prio}) updated with max/min of every w, duplicates
 * included (the tree keeps the last duplicate's w^alpha).  The arithmetic follows numpy's dtypes:
 * TS_F32 td: w = fl32(|td| + fl32(eps)), leaf = (double)powf(w, (float)alpha), minmax with (double)w;
 * TS_F64 td: w, w^alpha and minmax in double.  Device powf / pow are not correctly rounded (CUDA
 * documents 4 / 2 ulp), so leaves can differ from numpy's in the last bits and so can sampled
 * indices: for bit-exact indices compute w^alpha with the host pow (as data/buffer/prio.py does)
 * and write it with ts_segtree_setitem. */
int ts_prio_update_weight(double* tree, int64_t bound, const int64_t* index, const void* td,
                          int td_dtype, int64_t n, double alpha, double eps, double* prio_minmax,
                          ts_stream_t stream);
/* PrioritizedReplayBuffer.get_weight (+ batch-max normalisation, prio.py:69-79,104-106):
 * out[k] = (tree[bound+idx[k]] / min_prio)^(-beta), divided by the batch max if weight_norm. */
int ts_prio_get_weight(const double* tree, int64_t bound, const int64_t* index, int64_t n,
                       const double* prio_minmax, double beta, int weight_norm, double* out,
                       ts_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * (5) Actor-critic MLP (two tanh hidden layers of width `hidden`, separate actor and critic
 * trunks, Gaussian policy head with state-independent log-sigma) -- the network of
 * examples/mujoco/mujoco_ppo.py:90-120 built from tianshou/utils/net/common.py:172-179,343-369
 * and continuous.py:144-169,220-238.
 * All parameters live in ONE flat f32 buffer in torch layout ([out][in] row-major weights);
 * offsets are in floats.  The same offsets index the flat gradient / Adam-moment buffers.
 *
 * Variants selected by `flags` (the reference's discrete PPO test net, test/discrete/test_ppo_discrete.py:90-100:
 * ONE Net(obs -> 64 -> 64, ReLU) shared by DiscreteActor(softmax_output=True) and DiscreteCritic,
 * utils/net/discrete.py:29-123, policy distribution torch.distributions.Categorical(probs)):
 *   TS_AC_RELU         hidden activation max(x, 0) instead of tanh (Net's default, common.py MLP);
 *   TS_AC_CATEGORICAL  head = act_dim logits -> softmax -> Categorical; a_logstd is unused (-1); the
 *                      action array holds ONE index per row, stored as f32 (ppo.py:156 casts it so).
 * A SHARED trunk is expressed by aliased offsets (c_w1 == a_w1, c_b1 == a_b1, c_w2 == a_w2, c_b2 == a_b2): the
 * shared parameters are counted once in n_params and both losses' gradients add into the same slots.
 * Variants with flags != 0 or a shared trunk run the fp32 SIMT kernels.
 * ------------------------------------------------------------------------------------------ */
#define TS_AC_RELU 1
#define TS_AC_CATEGORICAL 2
typedef struct ts_actor_critic_desc {
    int32_t obs_dim;  /* <= 64 */
    int32_t act_dim;  /* <= 16 */
    int32_t hidden;   /* 64 */
    int32_t flags;           /* TS_AC_* bits; 0 = tanh trunks + diagonal-Gaussian head */
    int64_t a_w1, a_b1, a_w2, a_b2, a_w3, a_b3, a_logstd; /* actor: W1[h][obs] .. W3[act][h], logstd[act] */
    int64_t c_w1, c_b1, c_w2, c_b2, c_w3, c_b3;           /* critic: .. W3[1][h], b3[1] */
    int64_t n_params;
} ts_actor_critic_desc;

/* v_out[r] = critic(obs[r, :]) for r < n.  Up to two (obs, out) pairs in one launch (v_s and
 * v_s_ of a2c.py:123-126); pass obs1 = NULL for a single pass.  obs rows are obs_dim f32, dense. */
int ts_critic_forward(const float* params, const ts_actor_critic_desc* desc /* host */,
                      const float* obs0, float* v_out0, const float* obs1, float* v_out1,
                      int64_t n, ts_stream_t stream);
/* Which rows of obs_next repeat the following row of obs (a rollout: all but the episode / segment ends), so that the
 * critic need not be evaluated on them.  alias[i] (n bytes) = 1 iff i + 1 < n and the obs_dim 32-bit words of obs_next[i]
 * equal those of obs[i + 1] (bitwise: -0.0 vs 0.0 or two NaN payloads count as different); extra[0 .. *n_extra) (capacity n,
 * ascending) lists the rows with alias == 0; n_extra: device int32[1].  Deterministic (no atomics), no host sync.
 * workspace: ts_next_alias_workspace_bytes(n) bytes of scratch.  n < 2^31. */
int64_t ts_next_alias_workspace_bytes(int64_t n);
int ts_next_alias_map(const float* obs, const float* obs_next, int64_t n, int32_t obs_dim, uint8_t* alias,
                      int32_t* extra, int32_t* n_extra, void* workspace, ts_stream_t stream);
/* ts_critic_forward(obs, v_s, obs_next, v_next) with one critic evaluation per distinct row, given the map of
 * ts_next_alias_map(obs, obs_next): v_s[j] = critic(obs[j]); v_next[i] = v_s[i + 1] where alias[i];
 * v_next[extra[k]] = critic(obs_next[extra[k]]) for k < *n_extra.  A row's value does not depend on where it sits in a
 * tile, so v_s and v_next are bit for bit those of ts_critic_forward.  The tensor-core path does this in one launch whose
 * tile count follows *n_extra on the device; networks outside its envelope evaluate both inputs in full. */
int ts_critic_forward_dedup(const float* params, const ts_actor_critic_desc* desc /* host */, const float* obs,
                            const float* obs_next, const uint8_t* alias, const int32_t* extra,
                            const int32_t* n_extra, float* v_s, float* v_next, int64_t n, ts_stream_t stream);
/* logp_out[r] = Independent(Normal(mu(obs[r]), exp(logstd)), 1).log_prob(act[r])
 * (ppo.py:157-161 with reinforce.py:167-192).  mu_out (n*act_dim, nullable) receives mu.
 * TS_AC_CATEGORICAL: logp_out[r] = Categorical(probs = softmax(logits(obs[r]))).log_prob(act[r]) with act one f32
 * index per row; mu_out receives the probabilities (the actor's output). */
int ts_actor_logp(const float* params, const ts_actor_critic_desc* desc /* host */,
                  const float* obs, const float* act, int64_t n, float* logp_out, float* mu_out,
                  ts_stream_t stream);

typedef struct ts_ppo_hparams {
    /* all hyper-parameters are doubles (Python floats in the reference); the kernels narrow to
     * f32 at the point where torch would (scalar operand of an f32 tensor op) */
    double eps_clip;
    double dual_clip;     /* <= 0: disabled */
    double vf_coef;
    double ent_coef;
    double max_grad_norm; /* <= 0: no clipping */
    double adv_eps;       /* 1e-8 in the reference (self._eps) */
    /* Adam (torch.optim.Adam semantics, algorithm/optim.py:89-110) */
    double lr, beta1, beta2, adam_eps, weight_decay;
    int32_t value_clip;
    int32_t advantage_normalization;
    int32_t loss_kind;    /* TS_LOSS_PPO (0): clipped surrogate, ppo.py:184-196; TS_LOSS_A2C (1): actor loss
                           * -mean(log_prob * adv) (a2c.py:262-266), eps_clip / dual_clip / logp_old / v_s unused */
    int32_t optimizer;    /* TS_OPT_ADAM (0) or TS_OPT_RMSPROP (1): torch.optim.RMSprop's single-tensor step without
                           * momentum or centering (examples/mujoco/mujoco_a2c.py:117-121).  RMSprop reads lr, beta2 as its
                           * smoothing constant alpha, adam_eps as its eps and weight_decay; beta1 is unused.  square_avg
                           * lives in exp_avg_sq, exp_avg is untouched.  (The field fills the struct's tail padding: the
                           * layout and size are those of the Adam-only struct.) */
} ts_ppo_hparams;
#define TS_LOSS_PPO 0
#define TS_LOSS_A2C 1
#define TS_OPT_ADAM 0
#define TS_OPT_RMSPROP 1

/* Per-optimiser-step device statistics: {loss, clip_loss, vf_loss, ent_loss, grad_norm, n_rows,
 * 0, 0} -- 8 floats per step (ppo.py:213-216 without the 4 host syncs). */
#define TS_PPO_STATS_STRIDE 8
/* grad buffer layout: n_params floats + TS_PPO_GRAD_EXTRA scalar slots {sum_clip, sum_vf,
 * sum_ent, n_rows} so that ONE allreduce carries gradients and loss sums (SURVEY 8e). */
#define TS_PPO_GRAD_EXTRA 4

/* One minibatch forward/backward (ppo.py:179-211 + loss.backward of algorithm_base.py:497):
 * rows are perm[lo..hi) of the rollout tensors.  Every CTA writes ITS OWN partial sum of
 * d(loss)/d(params) (already scaled by 1/global_rows) and of the four loss sums into row
 * blockIdx.x of `partials` ([ts_ppo_partial_rows()][n_params + TS_PPO_GRAD_EXTRA] floats) -- no
 * cross-CTA atomics, deterministic.  *n_partials_out (host) receives the number of rows written;
 * they are folded by ts_grad_reduce / ts_clip_adam_step.  `global_rows` is the minibatch size
 * over all ranks (the mean's denominator); adv_moments: device float[2] = {mean, std} when
 * advantage_normalization, else NULL.  perm may be NULL (identity). */
int32_t ts_ppo_partial_rows(void);

/* Bytes of the optional `weight_image` scratch of ts_ppo_update: a 128-byte control block (grid-barrier state of
 * the persistent kernel: must be ZERO when first used and is left zero by every launch; one scratch per model, never
 * shared by two updates in flight) followed by both networks' weights pre-split into the bf16x3 tensor-core operand
 * layout, so that a CTA stages a network with one bulk copy.  0 when the network
 * shape is not covered by the tensor-core kernels (pass NULL then). */
int64_t ts_ppo_weight_image_bytes(const ts_actor_critic_desc* desc);
int ts_ppo_grad(const float* params, const ts_actor_critic_desc* desc, const ts_ppo_hparams* hp,
                const float* obs, const float* act, const float* adv, const float* ret,
                const float* logp_old, const float* v_s, const int32_t* perm, int64_t lo,
                int64_t hi, int64_t global_rows, const float* adv_moments, float* partials,
                int32_t* n_partials_out /* host */, ts_stream_t stream);
/* grad[i] = sum_p partials[p][i] (fixed order) for i < n_params + TS_PPO_GRAD_EXTRA: the flat
 * gradient + loss sums a multi-GPU caller all-reduces before ts_clip_adam_step. */
int ts_grad_reduce(const float* partials, int32_t n_partials, const ts_actor_critic_desc* desc,
                   float* grad, ts_stream_t stream);
/* mean and unbiased std of adv[perm[lo..hi)] (ppo.py:184-186) -> out[0..1]: ts_minibatch_adv_sums
 * WRITES (sum, sum of squares) of the rows to sums (device double[2]; fixed summation order, the same
 * as ts_epoch_adv_sums) so a multi-GPU caller can allreduce them; ts_adv_moments_finalize turns
 * (sum, sumsq, count=global_rows) into {mean, std} and leaves sums as they are.  A single row gives
 * std 0 (torch: NaN). */
int ts_minibatch_adv_sums(const float* adv, const int32_t* perm, int64_t lo, int64_t hi,
                          double* sums, ts_stream_t stream);
int ts_adv_moments_finalize(const double* sums, int64_t global_rows, float* out,
                            ts_stream_t stream);
/* clip_grad_norm_ + Adam.step (algorithm_base.py:496-500; torch/optim/adam.py single-tensor
 * path; RMSprop.step when hp->optimizer == TS_OPT_RMSPROP) on the flat buffers, and one row of per-step statistics.  If partials != NULL the
 * gradient is first folded from the n_partials rows (single-GPU fast path: reduce + norm + clip
 * + Adam in ONE launch); otherwise `grad` must already hold the (all-reduced) gradient.
 * grad: n_params + TS_PPO_GRAD_EXTRA floats (scratch / input).  step_count: device int64[1],
 * incremented.  stats_row: device float[TS_PPO_STATS_STRIDE]. */
int ts_clip_adam_step(float* params, float* grad, const float* partials, int32_t n_partials,
                      float* exp_avg, float* exp_avg_sq, int64_t* step_count,
                      const ts_actor_critic_desc* desc, const ts_ppo_hparams* hp, float* stats_row,
                      ts_stream_t stream);

/* The whole single-GPU `PPO._update_with_batch` loop (ppo.py:164-224) on one stream:
 * for r in repeat: [recompute v_s/returns/adv (a2c.py:115-153)] ; for each minibatch of
 * perm[r] (Batch.split bounds, batch.py:1199-1215): grad + clip + Adam.  No host sync.
 * perm: repeat*N int32 (row r = the permutation of repeat r).  bounds: host int64[2*n_mb].
 * rollout tensors (all N rows, device): obs, obs_next, act f32; rew f64; terminated,
 * truncated, extra_end u8; v_s, returns, adv, logp_old f32 (in/out: must be valid on entry,
 * rewritten when recompute_adv).  stats: repeat*n_mb rows.  rms_state as in ts_gae (nullable
 * when return_scaling is off).  v_next_tmp: N f32 scratch.  gae_ws: ts_gae_workspace_bytes(N).
 * grad: n_params + TS_PPO_GRAD_EXTRA floats scratch; partials: ts_ppo_partial_rows() rows of the
 * same width.  adv_tmp: 32 + 8 * n_minibatch bytes of scratch (double[2] sums, float[2] moments,
 * then one (mean, std) float pair per minibatch).  weight_image: ts_ppo_weight_image_bytes(desc) bytes of scratch
 * (nullable: the kernels then gather + split the weights themselves every step); rebuilt from `params` on entry.
 * row_feed: NULL, or a feed from ts_host_perm_feed_start whose dev_rows == perm: pass r then waits (on `stream`, not on the
 * host) until row r of the host permutation job has arrived in `perm`.
 */
int ts_ppo_update(float* params, float* grad, float* partials, float* exp_avg, float* exp_avg_sq,
                  int64_t* step_count, const ts_actor_critic_desc* desc, const ts_ppo_hparams* hp,
                  const float* obs, const float* obs_next, const float* act, const double* rew,
                  const uint8_t* terminated, const uint8_t* truncated, const uint8_t* extra_end,
                  float* v_s, float* returns, float* adv, const float* logp_old,
                  float* v_next_tmp, int64_t N, const int32_t* perm, int32_t repeat,
                  const int64_t* bounds /* host */, int32_t n_minibatch, int32_t recompute_adv,
                  double gamma, double lam, double* rms_state, double rms_eps, void* gae_ws,
                  void* adv_tmp, void* weight_image, float* stats, void* row_feed, ts_stream_t stream);
/* ts_ppo_update whose value recompute evaluates the critic once per distinct observation: next_alias / next_extra /
 * n_next_extra are the map of ts_next_alias_map(obs, obs_next) (see ts_critic_forward_dedup; same results).  All three
 * NULL: exactly ts_ppo_update. */
int ts_ppo_update_dedup(float* params, float* grad, float* partials, float* exp_avg, float* exp_avg_sq,
                        int64_t* step_count, const ts_actor_critic_desc* desc, const ts_ppo_hparams* hp,
                        const float* obs, const float* obs_next, const float* act, const double* rew,
                        const uint8_t* terminated, const uint8_t* truncated, const uint8_t* extra_end,
                        float* v_s, float* returns, float* adv, const float* logp_old,
                        float* v_next_tmp, int64_t N, const int32_t* perm, int32_t repeat,
                        const int64_t* bounds /* host */, int32_t n_minibatch, int32_t recompute_adv,
                        double gamma, double lam, double* rms_state, double rms_eps, void* gae_ws,
                        void* adv_tmp, void* weight_image, float* stats, void* row_feed,
                        const uint8_t* next_alias, const int32_t* next_extra, const int32_t* n_next_extra,
                        ts_stream_t stream);

/* ---- multi-GPU fused update: gradient all-reduce INSIDE the epoch kernel over NVLink peer memory -------------
 * Replaces, for one process per GPU (data-parallel replicas, each rank owns its own rollout shard), the
 * reference's single-process optimiser step (ppo.py:215-218) x world ranks: the loss is the mean over the
 * union of the ranks' local minibatches, the summed gradient / global-norm clip / Adam step are bit-identical
 * on every rank.  No NCCL call on the data path: after the local fold every CTA pushes its slice of the
 * gradient as (fp32 value, sequence number) 8-byte packets straight into every peer's exchange buffer and
 * gathers the peers' packets from its own.
 *
 * Plumbing: ts_peer_alloc cudaMalloc's + zeroes a buffer and returns its CUDA IPC handle (TS_PEER_HANDLE_BYTES
 * opaque bytes the host exchanges, e.g. with torch.distributed.all_gather); ts_peer_open maps a peer's buffer
 * into this process; ts_peer_close / ts_peer_free undo them.  Buffer size: ts_ppo_peer_buffer_bytes(desc, world)
 * (world <= 8).  The buffers carry a sequence number across launches: allocate once, zero-initialised, and use
 * them for every update of the same replicas. */
#define TS_PEER_HANDLE_BYTES 64
int ts_peer_alloc(int64_t bytes, void** ptr_out, uint8_t* handle_out /* TS_PEER_HANDLE_BYTES */);
int ts_peer_open(const uint8_t* handle, void** ptr_out);
int ts_peer_close(void* ptr);
int ts_peer_free(void* ptr);
int64_t ts_ppo_peer_buffer_bytes(const ts_actor_critic_desc* desc, int32_t world);

/* Per-minibatch advantage moments of one pass across ranks (ppo.py:181-183 on the global minibatch):
 * ts_epoch_adv_sums writes (sum, sum of squares) in f64 per minibatch of THIS rank's shard; the host all-reduces
 * the 2 * n_minibatch doubles; ts_epoch_adv_finalize turns them into (mean, unbiased std) float pairs for
 * minibatches of world * (hi - lo) rows. */
int ts_epoch_adv_sums(const float* adv, const int32_t* perm, int64_t lo0, int64_t mb_size, int64_t end,
                      int32_t n_minibatch, double* sums, ts_stream_t stream);
int ts_epoch_adv_finalize(const double* sums, int64_t lo0, int64_t mb_size, int64_t end, int32_t n_minibatch,
                          int32_t world, float* out, ts_stream_t stream);

/* ONE pass over the minibatches [lo0 + m * mb_size, ...) (last one ends at `end`; Batch.split bounds,
 * batch.py:1199-1215) of this rank's shard, every optimiser step of the pass in one persistent launch, gradients
 * summed over the `world` ranks in-kernel.  Arguments as ts_ppo_update (perm: this pass's N int32 or NULL;
 * stats: n_minibatch rows, global losses).  adv_moments: n_minibatch (mean, std) pairs from
 * ts_epoch_adv_finalize, required iff hp->advantage_normalization.  peer_buffers: host array of `world` device
 * pointers (index = rank; own buffer from ts_peer_alloc, the others from ts_peer_open); world == 1: may be NULL.
 * Every rank must call with the same shapes and the same number of minibatches.  A peer that does not show
 * up within 20 s traps the kernel (CUDA error at the next synchronisation) instead of hanging the GPU. */
int ts_ppo_epoch_multi(float* params, float* grad, float* partials, float* exp_avg, float* exp_avg_sq,
                       int64_t* step_count, const ts_actor_critic_desc* desc, const ts_ppo_hparams* hp,
                       const float* obs, const float* act, const float* adv, const float* returns,
                       const float* logp_old, const float* v_s, const int32_t* perm, int64_t lo0,
                       int64_t mb_size, int64_t end, int32_t n_minibatch, const float* adv_moments,
                       void* weight_image, float* stats, int32_t rank, int32_t world,
                       void* const* peer_buffers /* host */, ts_stream_t stream);

/* HOST function (no device work): out[0..n) = np.random.permutation(n) for numpy's legacy MT19937 RandomState whose
 * state is (key[624], *pos) -- the draw Batch.split makes once per pass (batch.py:1209).  Bit-identical to numpy
 * (MT19937 + random_interval masked rejection + backward Fisher-Yates of RandomState.shuffle); key / *pos are
 * advanced exactly as numpy would, so writing them back with np.random.set_state keeps the global stream in step.
 * Writes int32 directly (e.g. into the pinned upload buffer). */
int ts_host_mt19937_permutation(uint32_t* key /* in/out */, int32_t* pos /* in/out */, int64_t n, int32_t* out);

/* HOST, asynchronous: all `repeat` permutations of one update() (rows of out[repeat][n], int32, typically pinned),
 * identical to `repeat` consecutive np.random.permutation(n) draws from the state (key, pos).  A producer thread walks the
 * MT19937 stream, n_workers threads apply the swaps of different passes concurrently; ts_host_perm_job_wait(job, r)
 * blocks until row r is complete (rows complete in order of r up to worker interleaving); ts_host_perm_job_finish joins
 * the threads, returns the advanced generator state (write it back with np.random.set_state) and frees the job.
 * `out` must stay valid until finish.  Valid because nothing else consumes numpy's global stream inside
 * Algorithm.update() (batch.py:1209 is its only draw). */
int ts_host_perm_job_start(const uint32_t* key, int32_t pos, int64_t n, int32_t repeat, int32_t* out, int32_t n_workers,
                           void** job_out);
int ts_host_perm_job_wait(void* job, int32_t r);
int ts_host_perm_job_finish(void* job, uint32_t* key_out, int32_t* pos_out);

/* Asynchronous feed of a job's rows to the device -- the hand-over of `Batch.split`'s per-pass index array
 * (tianshou/data/batch.py:1209-1215: `indices = np.random.permutation(length)`, then one slice per minibatch) to the update
 * kernels; replaces the per-pass `perm.to(device)` of a host-driven loop: for
 * r in [0, repeat) a host function on an internal copy stream blocks that stream until row r is complete, then
 * host_rows[r] (pinned, the job's `out`) is copied to dev_rows[r] and an event is recorded.  ts_host_perm_feed_wait_row
 * makes `stream` wait for row r (ts_ppo_update does it before pass r when given the feed), so one asynchronous call enqueues
 * every pass of an update.  ts_host_perm_feed_finish: after the consumer's work has completed and BEFORE
 * ts_host_perm_job_finish (the host functions use the job). */
int ts_host_perm_feed_start(void* job, const int32_t* host_rows, int32_t* dev_rows, int64_t n, int32_t repeat, void** feed_out);
int ts_host_perm_feed_wait_row(void* feed, int32_t r, ts_stream_t stream);
int ts_host_perm_feed_finish(void* feed);

/* Device-side minibatch order (opt-in alternative to np.random.permutation, batch.py:1209):
 * out[r*n + i] = pi_r(i), pi_r a keyed bijection of [0,n) (cycle-walking Feistel/Philox). */
int ts_make_permutation(uint64_t seed, int32_t first_epoch, int32_t n_epochs, int64_t n,
                        int32_t* out, ts_stream_t stream);
/* int64 -> int32 narrowing of a host-drawn permutation already uploaded to the device. */
int ts_narrow_i64_i32(const int64_t* src, int64_t n, int32_t* dst, ts_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * (9) Layered networks of the off-policy algorithms (SURVEY.md 8(f) ranks 2-3): every nn.Linear / nn.Conv2d
 * forward and autograd backward inside SAC._update_with_batch (modelfree/sac.py:304-336),
 * _minimize_critic_squared_loss (modelfree/ddpg.py:267-285), DQN._update_with_batch (modelfree/dqn.py:382-404)
 * and DQNet (env/atari/atari_network.py:60-122) is ONE call of ts_net_gemm (wgmma, fp32-faithful bf16x3):
 *
 *     C[M,N] (+)= act'(act_grad_src) * act( A[M,K] * B[N,K]^T + bias[N] )
 *
 * A / B are fp32 arrays; x_mn_major = 0: element (mn, k) at p[mn * ld + k] (k contiguous), 1: at p[k * ld + mn].
 *   forward      Y  = act(X W^T + b)   : A = X  (lda = in),  B = W  [out][in]            (0, 0)
 *   input grad   dX = (dY W) * mask    : A = dY (lda = out), B = W  as [k = out][n = in] (0, 1)
 *   weight grad  dW = dY^T X           : A = dY as [k = row][m = out] (1), B = X as [k = row][n = in] (1)
 * act_grad_src (nullable): OUTPUT y of the layer whose activation derivative multiplies the result --
 * act_grad_kind TS_ACT_RELU: * (y[m * ld_mask + n] > 0), TS_ACT_TANH: * (1 - y^2)  (back-propagation through the
 * activation of the layer that produced this GEMM's output operand).  workspace (nullable): ts_net_gemm_workspace_floats(M, N, K) floats enable split-K
 * for long reductions with few output tiles (weight gradients); partial sums are added in a fixed order. */
enum { TS_ACT_NONE = 0, TS_ACT_RELU = 1, TS_ACT_TANH = 2 };
int ts_net_gemm(const float* a, int64_t lda, int32_t a_mn_major, const float* b, int64_t ldb, int32_t b_mn_major,
                float* c, int64_t ldc, int32_t M, int32_t N, int32_t K, const float* bias, int32_t act,
                const float* act_grad_src, int64_t ld_mask, int32_t act_grad_kind, int32_t accumulate, float* workspace,
                int64_t workspace_floats, ts_stream_t stream);
int64_t ts_net_gemm_workspace_floats(int32_t M, int32_t N, int32_t K);
/* out[n] (+)= sum_m x[m * ld + n]  (bias gradients) */
int ts_net_colsum(const float* x, int64_t ld, int32_t M, int32_t N, float* out, int32_t accumulate, ts_stream_t stream);
/* `batch` GEMMs of ts_net_gemm's contract in one launch (the members of an EnsembleLinear layer, utils/net/common.py:518-550):
 * member e reads a + e * stride_a, b + e * stride_b, bias + e * stride_bias, act_grad_src + e * stride_mask and writes
 * c + e * stride_c (element strides; 0 = the operand is shared by every member).  Split-K counts the output tiles of all
 * members; workspace: ts_net_gemm_batched_workspace_floats(batch, M, N, K) floats ([members][splits][M][N]).  With one member
 * the result is bitwise ts_net_gemm's (ts_net_gemm is that case).  With W_e[k * out + n] ([E][in][out]):
 *   forward      Y_e  = act(X W_e + b_e) : A = X  (lda = in, 0),  B = W_e (ldb = out, 1)
 *   input grad   dX_e = dZ_e W_e^T       : A = dZ_e (lda = out, 0), B = W_e (ldb = out, 0)
 *   weight grad  dW_e = X^T dZ_e         : A = X (lda = in, 1), B = dZ_e (ldb = out, 1), C [in][out] */
int ts_net_gemm_batched(int32_t batch, const float* a, int64_t lda, int32_t a_mn_major, int64_t stride_a, const float* b,
                        int64_t ldb, int32_t b_mn_major, int64_t stride_b, float* c, int64_t ldc, int64_t stride_c, int32_t M,
                        int32_t N, int32_t K, const float* bias, int64_t stride_bias, int32_t act, const float* act_grad_src,
                        int64_t ld_mask, int64_t stride_mask, int32_t act_grad_kind, int32_t accumulate, float* workspace,
                        int64_t workspace_floats, ts_stream_t stream);
int64_t ts_net_gemm_batched_workspace_floats(int32_t batch, int32_t M, int32_t N, int32_t K);
/* out[e * stride_out + n] (+)= sum_m x[e * stride_x + m * ld + n] for e < batch (per-member bias gradients) */
int ts_net_colsum_batched(int32_t batch, const float* x, int64_t ld, int64_t stride_x, int32_t M, int32_t N, float* out,
                          int64_t stride_out, int32_t accumulate, ts_stream_t stream);
/* out[i] (+)= sum_{e < batch} x[e * stride + i], i < n, members added in index order (no atomics) */
int ts_net_member_sum(const float* x, int32_t batch, int64_t stride, int64_t n, float* out, int32_t accumulate,
                      ts_stream_t stream);

/* PPO / A2C loss rows between the forward and backward GEMMs of a layered actor-critic (ppo.py:179-216, a2c.py:262-270):
 * head [B][A] = mu (Gaussian, sigma = exp(logstd[A])) or logits (categorical: Categorical(probs = softmax(logits)),
 * utils/net/discrete.py:69-92), value [B].  logp_out [B] always; with dhead != NULL also dhead [B][A], dvalue [B],
 * dlogstd_rows [B][A] (Gaussian, nullable), loss_rows [B][3] = (surrogate objective, value loss, entropy).
 * act: [B][A] (Gaussian) or [B] float-coded indices (categorical). */
int ts_ppo_rows(const float* head, const float* value, const float* logstd, const float* act, const float* adv,
                const float* ret, const float* logp_old, const float* v_s, int64_t B, int32_t A, int32_t categorical,
                const ts_ppo_hparams* hp, int64_t global_rows, const float* adv_moments, float* logp_out, float* dhead,
                float* dvalue, float* dlogstd_rows, float* loss_rows, ts_stream_t stream);
/* stats row (loss, actor loss, vf loss, entropy, -, rows) from loss_rows */
int ts_ppo_rows_stats(const float* loss_rows, int64_t B, const ts_ppo_hparams* hp, float* stats_row, ts_stream_t stream);

/* NPG / TRPO on a layered actor (modelfree/npg.py:123-224, modelfree/trpo.py:132-191).  head [B][A] = mu (Gaussian,
 * sigma = exp(logstd[A])) or logits (categorical, Categorical(probs = softmax(logits))); act as in ts_ppo_rows.
 *
 * Fisher-vector product rows (npg.py:195-200 without the damping term): the Gauss-Newton product J^T H J of the actor, H the
 * Hessian of the row's KL(old || new) w.r.t. the head outputs at old = new.  tangent [B][A] = J v on the head; out [B][A] =
 * (H tangent) / B feeds the backward GEMMs; Gaussian: out_logstd[A] = 2 * tangent_logstd (the whole log-std part, not rows). */
int ts_npg_fvp_rows(const float* head, const float* tangent, const float* logstd, const float* tangent_logstd, int64_t B,
                    int32_t A, int32_t categorical, float* out, float* out_logstd, ts_stream_t stream);
/* surrogate rows: loss_rows[B] = -logp * adv (npg.py:155-156) or, ratio_surrogate, -exp(logp - logp_old) * adv
 * (trpo.py:135-138); with dhead != NULL d(mean loss)/d head [B][A] and, Gaussian, per-row d / d logstd [B][A] */
int ts_npg_rows(const float* head, const float* logstd, const float* act, const float* adv, const float* logp_old, int64_t B,
                int32_t A, int32_t categorical, int32_t ratio_surrogate, float* loss_rows, float* dhead, float* dlogstd_rows,
                ts_stream_t stream);
/* kl_rows[B] = KL(old || new) per row with torch's kl_divergence formulas (npg.py:172-174, trpo.py:177), categorical: inf
 * where a new probability is exactly 0 */
int ts_npg_kl_rows(const float* head_old, const float* logstd_old, const float* head_new, const float* logstd_new, int64_t B,
                   int32_t A, int32_t categorical, float* kl_rows, ts_stream_t stream);
/* *out = mean of rows[B], fixed summation order */
int ts_npg_mean_rows(const float* rows, int64_t B, float* out, ts_stream_t stream);
/* conjugate gradient (npg.py:202-224) with its scalars in device memory: state[3] doubles = (r.r, done flag, iterations).
 * ts_cg_init: x = 0, r = p = g.  ts_cg_step: z = F p on entry (damping added here: z += damping p), then alpha, x, r, the new
 * r.r in fp64, the residual test (done: this and every later step is a no-op) and p.  iters_out (nullable) <- iterations. */
int ts_cg_init(const float* g, float* x, float* r, float* p, int64_t n, double* state, ts_stream_t stream);
int ts_cg_step(float* x, float* r, float* p, float* z, int64_t n, double damping, double residual_tol, double* state,
               float* iters_out, ts_stream_t stream);
/* trpo.py:152-159: z = F s on entry; *step = sqrt(2 max_kl / (s . (z + damping s))); stats_row[2] = 0 (kl), [3] = *step,
 * [5] = -1 (accepted candidate), [6] = 0 (line search failed) */
int ts_trpo_step_size(const float* s, const float* z, int64_t n, double damping, double max_kl, float* step, float* stats_row,
                      ts_stream_t stream);
/* out = theta + coef * (scale ? *scale : 1) * dir  (npg.py:168-170 natural step, trpo.py:165 line-search candidate) */
int ts_npg_axpy(float* out, const float* theta, const float* dir, double coef, const float* scale, int64_t n, ts_stream_t stream);
/* trpo.py:170-186 for candidate i < max_backtracks: mean new loss / kl from the rows, stats_row[2] = kl; accepted when
 * kl < max_kl and new loss < stats_row[0] (*flag = 1, stats_row[3] = *step, [5] = i); else *step *= backtrack_coeff
 * (*flag = 0) or, at the last candidate, stats_row[3] = 0, [6] = 1 (*flag = 2) */
int ts_trpo_decide(const float* loss_rows, const float* kl_rows, int64_t B, int32_t i, int32_t max_backtracks, double max_kl,
                   double backtrack_coeff, float* step, float* stats_row, int32_t* flag, ts_stream_t stream);
/* npg.py:136-137: adv = (adv - mean) / std over the whole batch, unbiased std, no epsilon */
int ts_npg_normalize_adv(float* adv, int64_t n, ts_stream_t stream);

/* Frame stacking on the device (ReplayBuffer.get, data/buffer/buffer_base.py:557-603): out[i][s] for s = 0..S-1 is
 * the slot of the s-th oldest frame of the stacked observation of index[i] (out[i][S-1] = index[i], each earlier
 * one = prev() of the next, manager.py:311-336). */
int ts_stack_prev_indices(const int64_t* index, int64_t n, int32_t stack_num, const int64_t* offset, int64_t E,
                          const uint8_t* done, const int64_t* last_index, const int64_t* lengths, int64_t* out,
                          ts_stream_t stream);
/* im2col rows for nn.Conv2d(k, stride s, no padding) in torch's weight order (column = c*k*k + kh*k + kw):
 * col[(b, ho, wo)][:].  _u8: source = single uint8 frames [slot][H][W] (save_only_last_obs buffers), channel c of
 * sample b is frame stack_idx[b*C + c], values = fl32(v / denom) with the division in f64 (ScaledObsInputActionReprNet
 * divides the uint8 array by 255.0 in numpy, env/atari/atari_network.py:26-55; denom = 1 for raw values).
 * _f32: source = fp32 NHWC activations [B][H][W][C]. */
int ts_im2col_u8(const uint8_t* frames, const int64_t* stack_idx, int32_t B, int32_t C, int32_t H, int32_t W, int32_t k,
                 int32_t s, double denom, float* col, ts_stream_t stream);
int ts_im2col_f32(const float* x_nhwc, int32_t B, int32_t C, int32_t H, int32_t W, int32_t k, int32_t s, float* col,
                  ts_stream_t stream);
/* inverse of ts_im2col_f32 for gradients (gather form, deterministic); relu_src (nullable, NHWC like dx): zero
 * where relu_src <= 0 */
int ts_col2im_f32(const float* dcol, int32_t B, int32_t C, int32_t H, int32_t W, int32_t k, int32_t s,
                  const float* relu_src, float* dx_nhwc, ts_stream_t stream);
/* nn.Flatten of NCHW from NHWC activations and its backward */
int ts_nhwc_to_nchw_flat(const float* x, int32_t B, int32_t HW, int32_t C, float* y, ts_stream_t stream);
int ts_nchw_flat_to_nhwc(const float* dy, int32_t B, int32_t HW, int32_t C, const float* relu_src, float* dx, ts_stream_t stream);
/* out = concat([a, b], dim=1)  (critic input obs ++ act, utils/net/continuous.py:160-166) */
int ts_concat2(const float* a, int32_t wa, const float* b, int32_t wb, int64_t rows, float* out, ts_stream_t stream);

/* SACPolicy.forward (modelfree/sac.py:108-131) on the actor head rows head[b] = (mu[0..A) | raw log-sigma[0..A)), row
 * stride ld: sigma = exp(clamp(raw, sig_min, sig_max)), x = mu + sigma*noise, act = tanh(x), log_prob = Normal log-prob
 * summed over actions - sum log(1 - act^2 + eps) (:25-39). */
int ts_squashed_gaussian(const float* head, int64_t ld, const float* noise, int64_t B, int32_t A, float sig_min,
                         float sig_max, float eps, float* act, float* logp, float* sigma_out, ts_stream_t stream);
/* backward of mean(alpha*logp - min(q1,q2)) through the head: dact = d loss / d act from the critics (already / B);
 * dhead has the layout of head */
int ts_squashed_gaussian_bwd(const float* head, int64_t ld, const float* noise, const float* act, const float* sigma,
                             const float* dact, int64_t B, int32_t A, float sig_min, float sig_max, float eps,
                             float alpha_over_b, float* dhead, ts_stream_t stream);
/* td = q - target; loss rows td^2*w; dq = 2 td w / B   (modelfree/ddpg.py:279-284) */
int ts_critic_mse(const float* q, const float* target, const float* weight, int64_t B, float* td, float* dq, float* loss_rows,
                  ts_stream_t stream);
/* DQN loss (modelfree/dqn.py:384-399): td = returns - q[b][act[b]]; weighted MSE or Huber(delta > 0) */
int ts_dqn_loss(const float* q, const int64_t* act, const float* returns, const float* weight, int64_t B, int32_t A,
                float huber_delta, float* td, float* dq, float* loss_rows, ts_stream_t stream);
/* DQN._target_q (dqn.py:365-380): double -> q_target[b][argmax_a q_online[b][a]], else max_a q_target[b][a] */
int ts_dqn_target(const float* q_online, const float* q_target, int64_t B, int32_t A, int32_t is_double, float* out,
                  ts_stream_t stream);
/* min(q1, q2) - alpha * logp   (td3.py:94-102, sac.py:298-302) */
int ts_sac_target(const float* q1, const float* q2, const float* logp, float alpha, int64_t B, float* out, ts_stream_t stream);
/* rows of alpha*logp - min(q1,q2) and d(-min)/dq / B with torch.minimum's tie rule (sac.py:315-321) */
int ts_sac_actor_q_grad(const float* q1, const float* q2, const float* logp, float alpha, int64_t B, float* dq1, float* dq2,
                        float* loss_rows, ts_stream_t stream);
int ts_mean(const float* x, int64_t n, float* out, ts_stream_t stream);
/* clip_grad_norm_ (optional) + torch.optim.Adam step on a flat parameter vector (algorithm_base.py:496-500, optim.py:89-110);
 * `step` = the 1-based step number of this call */
int ts_adam_step(float* params, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t n, int64_t step, double lr,
                 double beta1, double beta2, double eps, double weight_decay, double max_grad_norm, double* norm_scratch,
                 ts_stream_t stream);
/* the same step with the step counter in DEVICE memory (*step_dev = steps taken so far; incremented by the call): no host-side
 * state in the launch, so a captured CUDA graph containing it can be replayed update after update */
int ts_adam_step_dev(float* params, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t n, int64_t* step_dev, double lr,
                     double beta1, double beta2, double eps, double weight_decay, double max_grad_norm, double* norm_scratch,
                     ts_stream_t stream);
/* clip_grad_norm_ (optional) + torch.optim.RMSprop step without momentum or centering on a flat parameter vector
 * (algorithm_base.py:496-500, optim.py RMSpropOptimizerFactory; torch/optim/rmsprop.py _single_tensor_rmsprop):
 *   g = clipped grad (+ weight_decay * p);  square_avg = square_avg * alpha + (1 - alpha) * g * g;
 *   p -= lr * g / (sqrt(square_avg) + eps)
 * No bias correction, so the step count is the caller's (torch's `step` state). */
int ts_rmsprop_step(float* params, const float* grad, float* square_avg, int64_t n, double lr, double alpha, double eps,
                    double weight_decay, double max_grad_norm, double* norm_scratch, ts_stream_t stream);
/* target = tau * source + (1 - tau) * target   (utils/lagged_network.py:8-18) */
int ts_polyak_update(float* target, const float* source, int64_t n, double tau, ts_stream_t stream);

/* GAIL discriminator rows (imitation/gail.py).  Rewards (gail.py:193-206): rew[n] = -log_sigmoid(-logits[n]) evaluated in fp32
 * as torch does (min(0, z) - log1p(exp(-|z|)), z = -logit), widened to f64 for GAE; grid-stride over any n. */
int ts_gail_reward_rows(const float* logits, int64_t n, double* rew, ts_stream_t stream);
/* one discriminator step (gail.py:226-235): logits [n_pi + n_exp] = [policy rows | expert rows];
 * dlogits = d loss / d logit with loss = -log_sigmoid(-logits_pi).mean() + -log_sigmoid(logits_exp).mean()
 * (sigmoid(x) / n_pi, -sigmoid(-x) / n_exp); stats_row[4] = (loss, (logits_pi < 0).mean(), (logits_exp > 0).mean(), n_pi).
 * Fixed-order reduction, no atomics: two calls on the same input are bit-identical. */
int ts_gail_disc_rows(const float* logits, int64_t n_pi, int64_t n_exp, float* dlogits, float* stats_row, ts_stream_t stream);

/* ---- discrete SAC (discrete_sac.cu) ---- */
/* The categorical rows of discrete SAC (discrete_sac.py:147-155 target value, :176-184 actor loss), in torch's fp32
 * Categorical(logits=...) formulation: per row b with p = softmax(logits[b]), log p = logits[b] - logsumexp(logits[b]),
 * m = min(q1[b], q2[b]): probs[b] = p; entropy[b] = H = -sum clamp(log p, finfo.min) * p; v[b] = sum p * m + alpha * H;
 * dlogits[b] (nullable: the target needs none) = dlogit_scale * d(-v[b]) / dlogits[b]
 *                                              = dlogit_scale * (alpha p (log p + H) - p (m - sum p * m)).
 * [B, A] row-major, any A >= 1, any B (warps stride over the rows).  Fixed-order reductions, no atomics: two calls on the
 * same input are bit-identical. */
int ts_discrete_sac_rows(const float* logits, const float* q1, const float* q2, float alpha, int64_t B, int32_t A, float* v,
                         float* entropy, float* probs, float* dlogits, float dlogit_scale, ts_stream_t stream);

/* ---- CQL (cql.cu) ---- */
/* Per-row pieces of CQL's critic step (imitation/cql.py:295-365; CalQL calibration :331-346).  q1 / q2: each critic's outputs
 * on one forward over B + 3N rows, N = B * R, ordered [data B | random N | current-pi N | next-pi N].  target [B]: the one-step
 * target.  Block row i (observation i / R) has the values v_j = q_j - c_j with c = (rand_logp, logp_cur[i], logp_next[i]);
 * cal_ret (nullable: uncalibrated) [B]: v_j = max(v_j, cal_ret[i / R]).  With x_j = v_j / T and the multiplier
 * scale = log_alpha ? clamp(exp(*log_alpha), alpha_min, alpha_max) : 1 (device scalar):
 *   sq_rows [2][B]   (q - target)^2 of the data rows;  lse_rows [2][N]   logsumexp over the THREE values x_j of the row (the
 *                    reference concatenates three (N, 1) blocks along dim 1)
 *   dq1 / dq2 [B+3N] d critic loss / d q: data rows 2 (q - target) / B - scale w / B; block rows
 *                    (scale T w / N) exp(x_j - lse) / T times 1, 1/2 or 0 as v_j is above, equal to or below cal_ret (torch.maximum).
 * Any R >= 1, any B (grid-stride). */
int ts_cql_rows(const float* q1, const float* q2, const float* target, int64_t B, int32_t R, const float* logp_cur,
                const float* logp_next, float rand_logp, const float* cal_ret, float temperature, float cql_weight,
                const float* log_alpha, float alpha_min, float alpha_max, float* dq1, float* dq2, float* sq_rows,
                float* lse_rows, ts_stream_t stream);
/* The losses of ts_cql_rows' rows (cql.py:353-384), one block, fixed-order sums (bit-identical from run to run):
 * penalty_k = mean(lse_k) w T - mean(q_k data) w; with log_alpha (Lagrange): a = clamp(exp(*log_alpha)), c_k = a (penalty_k -
 * threshold), out[2] = a, out[3] = cql_alpha_loss = -(c1 + c2) 0.5, *grad_log_alpha = its derivative (clamp passes the gradient
 * inside [alpha_min, alpha_max]); out[0], out[1] = mean (q_k - target)^2 + (c_k or penalty_k). */
int ts_cql_losses(const float* q1, const float* q2, const float* sq_rows, const float* lse_rows, int64_t B, int64_t N,
                  float temperature, float cql_weight, const float* log_alpha, float alpha_min, float alpha_max,
                  float threshold, float* grad_log_alpha, float* out, ts_stream_t stream);
/* One-step target of CQL (cql.py:282-292): out = rew + logical_not(done) * gamma * (min(q1, q2) - alpha * logp) in fp32, in
 * the reference's operation order; rew / done are fp32 rows (to_torch(batch, dtype=torch.float)). */
int ts_cql_target(const float* q1, const float* q2, const float* logp, float alpha, const float* rew, const float* done,
                  float gamma, int64_t B, float* out, ts_stream_t stream);

/* ---- TD3 / TD3+BC (td3.cu) ---- */
/* The deterministic actor's action rows written straight into a critic input x [B][O + A] = [obs | a]
 * (utils/net/continuous.py:84, modelfree/td3.py:190-202): a = max_action * tanh(z) from the actor's last-layer output z [B][A];
 * with noise [B][A] (nullable: the actor step) a += clamp(noise * policy_noise, -noise_clip, noise_clip), the clamp skipped when
 * noise_clip <= 0 and the sum NOT clipped back to the action bounds.  Any B (grid-stride). */
int ts_td3_act_rows(const float* z, const float* noise, int64_t B, int32_t A, float max_action, float policy_noise,
                    float noise_clip, const float* obs, int32_t O, float* x, ts_stream_t stream);
/* out = torch.min(q1, q2) of the two lagged critics (modelfree/td3.py:94-102); NaN propagates.  Any B (grid-stride). */
int ts_td3_target_min(const float* q1, const float* q2, int64_t B, float* out, ts_stream_t stream);
/* The actor loss on q = Q1(s, pi(s)) [B] (modelfree/td3.py:214-219, imitation/td3_bc.py:113-120), one block, fixed-order sums
 * (bit-identical from run to run).  act (nullable) [B][A]: the batch actions of TD3+BC, with pi = max_action * tanh(z):
 *   act == NULL : *loss = -mean(q);                                              dq[b] = -1 / B
 *   act != NULL : lmbda = alpha / mean|q| (detached); *loss = -lmbda mean(q) + mean((pi - act)^2);  dq[b] = -lmbda / B
 * Every row of dq [B] is written. */
int ts_td3_actor_rows(const float* q, const float* z, const float* act, int64_t B, int32_t A, float max_action, float alpha,
                      float* dq, float* loss, ts_stream_t stream);
/* Backward of pi = max_action * tanh(z) (and of TD3+BC's F.mse_loss(pi, act) when act is given):
 * dz = (dact + [act] 2 (pi - act) / (B A)) * max_action * (1 - tanh(z)^2); dact [B][A] = d loss / d pi through critic 1.
 * Any B (grid-stride). */
int ts_td3_actor_head_bwd(const float* z, const float* dact, const float* act, int64_t B, int32_t A, float max_action, float* dz,
                          ts_stream_t stream);

/* ---- REDQ (redq.cu) ---- */
/* The target of REDQ (modelfree/redq.py:254-269) from the lagged ensemble's q [E][B] on (s', a'): over the members whose bit is
 * set in `subset` (at most 64 members), target_mode TS_REDQ_MIN: min (NaN propagates), TS_REDQ_MEAN: their sum in member order
 * / count; out[b] = that - alpha * logp[b].  Any B (grid-stride). */
#define TS_REDQ_MIN 0
#define TS_REDQ_MEAN 1
int ts_redq_target(const float* q, int32_t E, int64_t B, uint64_t subset, int32_t target_mode, float alpha, const float* logp,
                   float* out, ts_stream_t stream);
/* The ensemble's critic loss (redq.py:273-279) on q [E][B], target [B] and weight [B] (nullable: 1): td [E][B] = q - target,
 * dq [E][B] = 2 w td / (E B), row_mean [B] = mean_e td (signed: the prioritised buffer's batch.weight), rows [B] = sum_e td^2 w
 * (scratch) and *loss = mean(td^2 w) over E * B, summed in a fixed order (bit-identical from run to run). */
int ts_redq_critic_rows(const float* q, const float* target, const float* weight, int32_t E, int64_t B, float* td, float* dq,
                        float* row_mean, float* rows, float* loss, ts_stream_t stream);
/* The actor loss (redq.py:285-289) on q [E][B] = Q_e(s, pi(s)) and logp [B]: rows [B] = alpha logp - mean_e q (scratch),
 * *loss = mean(rows) in a fixed order, dq [E][B] = -1 / (E B).  The loss's gradient at logp is alpha / B at every row: the
 * alpha_over_b of ts_squashed_gaussian_bwd. */
int ts_redq_actor_rows(const float* q, const float* logp, int32_t E, int64_t B, float alpha, float* dq, float* rows, float* loss,
                       ts_stream_t stream);

/* ---- BDQN (bdqn.cu) ---- */
/* The 1-step target of BDQN (modelfree/bdqn.py:126-175) from a branching network's value output v [B][1] and branch scores
 * s [nb][B][A] (Q = v + (s - mean_a s)) on s': per branch the first arg-max a*_k of the selecting network's Q (v_sel, s_sel: the
 * online network when double, else the lagged one) read from the evaluating network's Q (v_val, s_val);
 * y[b] = fp32(rew[i] + fp32(gamma * m) * (1 - end[i])), i = idx[b], m = the fp32 mean over branches summed in numpy's order
 * (pairwise over blocks of 8, exact for up to 128 branches), rew the buffer's float64 column, end its end flags (done, or an
 * unfinished episode's last slot).  y_branch [B][nb] (nullable): the per-branch targets fp32(rew + fp32(gamma * Q'_k) (1 - end)).
 * Any B (grid-stride). */
int ts_bdqn_target(const float* v_sel, const float* s_sel, const float* v_val, const float* s_val, int64_t B, int32_t nb,
                   int32_t A, float gamma, const double* rew, const uint8_t* end, const int64_t* idx, float* y, float* y_branch,
                   ts_stream_t stream);
/* BDQN's loss (bdqn.py:177-196) on v [B][1], s [nb][B][A], act [B][nb] (each in [0, A)), y [B] and weight [B] (nullable: 1):
 * td [B][nb] = y - Q at the chosen action of each branch, rows [B] = w mean_k td^2 (scratch), td_sum [B] = sum_k td (signed: the
 * prioritised buffer's batch.weight), *loss = mean(rows) in a fixed order, and the gradients of the dueling combine:
 * ds [nb][B][A] = g - mean_a g and dv [B] = sum_k g, g = -2 w td / (nb B) at the chosen action.  y_branch (B = 1 only, nullable):
 * adds the population variance of the per-branch targets to *loss, as the reference's [nb, nb, A] broadcast does. */
int ts_bdqn_rows(const float* v, const float* s, const int64_t* act, const float* y, const float* weight, const float* y_branch,
                 int64_t B, int32_t nb, int32_t A, float* td, float* rows, float* td_sum, float* ds, float* dv, float* loss,
                 ts_stream_t stream);

/* ---- BCQ (bcq.cu) ---- */
/* The VAE's reparameterisation (utils/net/continuous.py:464-470): from head = [mean | log_std_raw] [B][2L] and eps [B][L],
 * std = exp(clamp(log_std_raw, -4, 15)) into std_out [B][L] and z = mean + std * eps straight into the decoder input
 * x [B][O + L] = [s | z].  Any B (grid-stride). */
int ts_bcq_vae_reparam(const float* head, const float* eps, int64_t B, int32_t L, const float* s, int32_t O, float* std_out,
                       float* x, ts_stream_t stream);
/* The VAE loss (imitation/bcq.py:202-206) on the decoder output y [B][A], one block, fixed-order sums (bit-identical from run to
 * run): *loss = mean((act - recon)^2) + mean(-log std + (std^2 + mean^2 - 1) / 2) / 2 with recon = max_action * tanh(y);
 * dy [B][A] = d loss / d y (the KL term does not reach y). */
int ts_bcq_vae_loss(const float* y, const float* act, const float* head, const float* std_in, int64_t B, int32_t A, int32_t L,
                    float max_action, float* dy, float* loss, ts_stream_t stream);
/* The backward of the VAE head: from dz [B][L] (the decoder's input gradient over the z columns) and the KL term,
 * dhead [B][2L] = d loss / d [mean | log_std_raw]; the log_std clamp passes the gradient at its bounds (torch's clamp).  Any B. */
int ts_bcq_vae_head_bwd(const float* head, const float* std_in, const float* eps, const float* dz, int64_t B, int32_t L,
                        float* dhead, ts_stream_t stream);
/* The decoder input of VAE.decode with a drawn latent (continuous.py:481-490, bcq.py:213-217): x [B N][O + L] =
 * [s[r / N] | clamp(z[r], -clip, clip)], the repeat_interleave of s fused in.  Any B. */
int ts_bcq_decode_input(const float* s, int64_t B, int32_t N, int32_t O, const float* z, int32_t L, float clip, float* x,
                        ts_stream_t stream);
/* Decoded actions beside their states: x [rows][O + A] = [s[r step] | max_action * tanh(y[r step])], s with row stride lds,
 * y [.][A] the decoder output.  step > 1 picks one row per group of step rows.  Any rows. */
int ts_bcq_act_rows(const float* s, int64_t lds, const float* y, int64_t step, int64_t rows, int32_t O, int32_t A,
                    float max_action, float* x, ts_stream_t stream);
/* Perturbation.forward (continuous.py:407-412) into a critic input x [rows][O + A] = [s[r] | clamp(a + phi_m tanh(logits[r / S]),
 * -max_action, max_action)] with the decoded action a = vae_max * tanh(y[r]), phi_m = phi * max_action and max_action the
 * perturbation's; S = 1 gives every row its own logits (a Net preprocess), S = the group size broadcasts one logits row over
 * the group (an MLP preprocess's row 0).  Any rows. */
int ts_bcq_perturb(const float* logits, int64_t S, const float* y, int64_t rows, int32_t A, float vae_max, float max_action,
                   float phi_m, const float* s, int64_t lds, int32_t O, float* x, ts_stream_t stream);
/* Backward of ts_bcq_perturb to dlogits [G][A] from dact [G S][A] = d loss / d perturbed action: per group a fixed-order sum of
 * dact where the clamp passed (inclusive bounds), times phi_m * (1 - tanh(logits)^2).  Any G. */
int ts_bcq_perturb_bwd(const float* logits, int64_t S, int64_t G, const float* y, const float* dact, int32_t A, float vae_max,
                       float max_action, float phi_m, float* dlogits, ts_stream_t stream);
/* BCQ's one-step target (bcq.py:222-237): out[b] = rew[b] + logical_not(done[b]) * gamma * max over the N rows of group b of
 * lmbda * min(q1, q2) + one_minus_lmbda * max(q1, q2), fp32 in torch's order; NaN propagates.  rew / done fp32 [B]. */
int ts_bcq_target(const float* q1, const float* q2, int64_t B, int32_t N, float lmbda, float one_minus_lmbda, const float* rew,
                  const float* done, float gamma, float* out, ts_stream_t stream);
/* BCQPolicy's choice (bcq.py:111-114): per group g of S rows of q, the first index of the maximum (a NaN is the maximum, as in
 * torch.argmax); act [G][A] = that row's columns col0 .. col0 + A of x (row stride ldx), idx [G] (nullable) = the index. */
int ts_bcq_select(const float* q, int64_t G, int64_t S, const float* x, int64_t ldx, int32_t col0, int32_t A, float* act,
                  int64_t* idx, ts_stream_t stream);

/* ---- discrete BCQ (discrete_bcq.cu) ---- */
/* Discrete BCQ's bootstrap value (imitation/discrete_bcq.py:115-118 the policy's masked arg-max, :228-234 the target):
 * per row b, mask_a = (logits[b][a] - max_a logits[b]) < log_tau (log_tau = -inf masks nothing),
 * a* = argmax_a (q_online[b][a] - FLT_MAX * mask_a) evaluated in fp32 with torch.argmax's rule (lowest index among ties, a NaN
 * is the maximum), out[b] = q_old[b][a*]; act_out [B] (nullable) = a*.  [B, A] row-major, one warp per row, any A >= 1, any B. */
int ts_discrete_bcq_target(const float* q_online, const float* logits, const float* q_old, float log_tau, int64_t B, int32_t A,
                           float* out, int64_t* act_out, ts_stream_t stream);
/* Discrete BCQ's loss (discrete_bcq.py:244-252) on the Q head's q [B][A] and the imitator head's logits [B][A]:
 * losses[4] = (loss, q_loss, i_loss, reg_loss) with q_loss = smooth_l1_loss(q[b][act[b]], returns[b]) (beta 1, mean),
 * i_loss = nll_loss(log_softmax(logits), act) (mean), reg_loss = mean(logits^2) over B * A, loss = q_loss + i_loss +
 * penalty * reg_loss; dq, dlogits [B][A] = d loss / d q, d loss / d logits (every element written).  act must lie in [0, A):
 * the caller checks it.  rows [3][B] is scratch (the per-row terms).  One warp per row, then one block summing the rows in a
 * fixed order: two calls on the same input are bit-identical.  Any A >= 1, any B >= 1. */
int ts_discrete_bcq_rows(const float* q, const float* logits, const int64_t* act, const float* returns, int64_t B, int32_t A,
                         float penalty, float* dq, float* dlogits, float* rows, float* losses, ts_stream_t stream);

/* ---- discrete CRR (discrete_crr.cu) ---- */
enum { TS_CRR_EXP = 0, TS_CRR_BINARY = 1, TS_CRR_ALL = 2 };
/* Discrete CRR's loss (imitation/discrete_crr.py:131-158) on the critic head's q [B][A] and the actor head's logits [B][A]
 * at s, and the lagged heads' q_old, logits_old [B][A] at s' (the same pointers as q / logits are allowed).  Per row, with
 * p = softmax(logits), qa = q[b][act[b]]: target = rew + gamma * (done > 0 ? 0 : sum_a softmax(logits_old)_a q_old_a);
 * adv = qa - sum_a p_a q_a; coef = clamp(exp(adv / beta), 0, ratio_upper_bound) | 1[adv > 0] | 1 by mode;
 * losses[4] = (loss, actor_loss, critic_loss, cql_loss): critic_loss = mean_b 0.5 (qa - target)^2, cql_loss = mean_b
 * (logsumexp(q[b]) - qa), and actor_loss = mean_b(-log p[act]) * mean_b(coef): the reference multiplies -log_prob [B] by the
 * coefficient [B, 1] (discrete_crr.py:155), which broadcasts to [B, B], so its mean is the product of the two means, not the mean
 * of the per-row products.  loss = actor_loss + critic_loss + min_q_weight * cql_loss.
 * dq, dlogits [B][A] = d loss / d q, d loss / d logits as the reference's autograd takes it: the advantage is not detached, so
 * in TS_CRR_EXP mode the coefficient carries gradient into q (through qa and sum p q) and into the logits (through p) wherever
 * the clamp passes; the other modes carry none through the coefficient.  rew, done fp32 [B]; act in [0, A), checked by the
 * caller; rows [4 B + 2] scratch (the per-row terms and the two means).  Three launches (rows, their sums in one block, the
 * gradient, which needs the two batch means), fixed-order sums, bit-identical from run to run.  Any A >= 1, any B >= 1. */
int ts_discrete_crr_rows(const float* q, const float* logits, const int64_t* act, const float* q_old, const float* logits_old,
                         const float* rew, const float* done, int64_t B, int32_t A, float gamma, int32_t mode, float beta,
                         float ratio_upper_bound, float min_q_weight, float* dq, float* dlogits, float* rows, float* losses,
                         ts_stream_t stream);

/* ---- QR-DQN and discrete CQL (qrdqn.cu) ---- */
/* QR-DQN's target distribution (modelfree/qrdqn.py:94-106 with compute_q_value = logits.mean(2), :18-20): q_online, q_next
 * [B][A][N] at s_{t+n} (q_next the lagged network's output, or q_online itself); per row b, m_a = mean_k q_online[b][a][k] in
 * fp32, a* = argmax_a m_a with torch.argmax's rule (lowest index among ties, a NaN is the maximum), out [B][N] = q_next[b][a*];
 * act_out [B] (nullable) = a*.  The arg-max always comes from q_online (the reference has no is_double switch).  One warp per
 * row, any A >= 1, N >= 1, B. */
int ts_qrdqn_target(const float* q_online, const float* q_next, int64_t B, int32_t A, int32_t N, float* out, int64_t* act_out,
                    ts_stream_t stream);
/* The quantile-Huber loss of QR-DQN (qrdqn.py:108-131) and, with min_q_weight > 0, discrete CQL (imitation/discrete_cql.py:80-113)
 * on q [B][A][N] at s, the n-step returns [B][N], tau_hat [N] (the reference's midpoints, built by the caller) and the importance
 * weight [B] (nullable: 1).  With c_i = q[b][act[b]][i], u_ij = returns[b][j] - c_i, h_ij = smooth_l1(u_ij) (beta 1):
 * qr_b = (1/N) sum_i sum_j h_ij |tau_i - 1[u_ij <= 0]|, prio [B] = (1/N) sum_i sum_j h_ij;
 * losses[4] = (loss, qr_loss, cql_loss, mean_b prio) with qr_loss = mean_b(weight_b qr_b), cql_loss = mean_b(logsumexp_a m_a -
 * m_act) over the quantile means m_a = mean_k q[b][a][k] (0 when min_q_weight == 0), loss = qr_loss + min_q_weight * cql_loss.
 * dq [B][A][N] = d loss / d q, every element written: the indicator is detached, as in the reference, and the weight scales the
 * quantile term only.  act must lie in [0, A): the caller checks it.  rows [3][B] is scratch.  One block per row (threads over
 * the current quantiles, the row's targets and taus in shared memory), then one block summing the rows in a fixed order: two
 * calls on the same input are bit-identical.  Any B >= 1, A >= 1, N >= 2 with 2 N (+ A when min_q_weight > 0) <= 12288;
 * larger shapes are refused. */
int ts_qrdqn_rows(const float* q, const int64_t* act, const float* returns, const float* tau_hat, const float* weight, int64_t B,
                  int32_t A, int32_t N, float min_q_weight, float* dq, float* prio, float* rows, float* losses, ts_stream_t stream);

/* ---- C51 (c51.cu) ---- */
/* C51's target distribution (modelfree/c51.py:113-124 with compute_q_value = (p * support).sum(2), :62-63): logits_online,
 * logits_next [B][A][N] are the network's raw last-layer outputs at s_{t+n} (logits_next the lagged network's, or logits_online
 * itself); per row b, p_a = softmax over the N atoms of logits_online[b][a], Q_a = sum_k p_ak support[k] in fp32,
 * a* = argmax_a Q_a with torch.argmax's rule (lowest index among ties, a NaN is the maximum), next_dist [B][N] =
 * softmax(logits_next[b][a*]); act_out [B] (nullable) = a*.  One warp per row, grid-stride; any A >= 1, N >= 2, B >= 0 (B == 0
 * launches nothing). */
int ts_c51_target(const float* logits_online, const float* logits_next, const float* support, int64_t B, int32_t A, int32_t N,
                  float* next_dist, int64_t* act_out, ts_stream_t stream);
/* The categorical cross-entropy of C51 (c51.py:125-160) on logits [B][A][N] at s (raw: the softmax is taken here), the n-step
 * returns [B][N] (r + gamma^n support * mask), support [N], next_dist [B][N] from ts_c51_target and the importance weight [B]
 * (nullable: 1).  With t_k = clamp(returns[b][k], v_min, v_max), target_j = sum_k clamp(1 - |t_k - support_j| / delta_z, 0, 1)
 * next_dist[b][k] (the reference's dense projection, k summed in order), p = softmax(logits[b][act[b]]):
 * CE_b = -sum_j target_j log(p_j + 1e-8), prio [B] = CE_b (unweighted); losses[4] = (loss, loss, mean_b CE_b, 0) with
 * loss = mean_b(weight_b CE_b).  dlogits [B][A][N] = d loss / d logits, every element written: with
 * g_j = -(weight_b / B) target_j / (p_j + 1e-8), the taken block gets p_k (g_k - sum_j p_j g_j), every other block 0; the target
 * carries no gradient.  act must lie in [0, A): the caller checks it.  rows [3][B] is scratch.  One block per row (threads over
 * the atoms, four arrays of N floats in shared memory), grid-stride, then one block summing the rows in a fixed order, no
 * atomics: two calls on the same input are bit-identical.  Any B >= 1, A >= 1, 2 <= N <= 3072, delta_z > 0, v_min <= v_max;
 * anything else is refused. */
int ts_c51_rows(const float* logits, const int64_t* act, const float* returns, const float* support, float v_min, float v_max,
                float delta_z, const float* next_dist, const float* weight, int64_t B, int32_t A, int32_t N, float* dlogits,
                float* prio, float* rows, float* losses, ts_stream_t stream);

/* ---- Rainbow (rainbow.cu) ---- */
/* The train-mode weight of a noisy layer (utils/net/discrete.py NoisyLinear): mu_w, sigma_w [out][in], mu_b, sigma_b [out], the
 * factorised noise eps_p [in], eps_q [out]; w_eff [out][in] = mu_w + sigma_w * (eps_q[o] * eps_p[i]), b_eff [out] = mu_b +
 * sigma_b * eps_q[o], each product and sum rounded on its own: bit for bit torch's ger, then *, then +.  Any out, in >= 1. */
int ts_noisy_weight(const float* mu_w, const float* sigma_w, const float* mu_b, const float* sigma_b, const float* eps_p,
                    const float* eps_q, int32_t out, int32_t in, float* w_eff, float* b_eff, ts_stream_t stream);
/* The gradient of a noisy layer's four trainable tensors from dw [out][in] and db [out], the gradients at its effective weight and
 * bias: g_mu_w = dw, g_sigma_w = dw * (eps_q[o] * eps_p[i]), g_mu_b = db, g_sigma_b = db * eps_q[o], each product rounded on its
 * own.  Any out, in >= 1. */
int ts_noisy_grad(const float* dw, const float* db, const float* eps_p, const float* eps_q, int32_t out, int32_t in, float* g_mu_w,
                  float* g_sigma_w, float* g_mu_b, float* g_sigma_b, ts_stream_t stream);
/* The dueling combine of the categorical heads (common.py:355-364, atari_network.py:196-206): q [B][A][N] (the Q head's A * N
 * outputs), v [B][N]; logits [B][A][N] = (q - m) + v with m [B][N] = (sum_a q in index order) / A.  Any B >= 0 (B == 0 launches
 * nothing), A, N >= 1. */
int ts_dueling_atoms(const float* q, const float* v, int64_t B, int32_t A, int32_t N, float* logits, ts_stream_t stream);
/* Its backward from dlogits [B][A][N]: dv [B][N] = s = sum_a dlogits (index order), dq [B][A][N] = dlogits - s / A.  No atomics:
 * two calls on the same input are bit-identical.  Any B >= 0, A, N >= 1. */
int ts_dueling_atoms_bwd(const float* dlogits, int64_t B, int32_t A, int32_t N, float* dq, float* dv, ts_stream_t stream);

/* ---- DRQN (lstm.cu) ---- */
/* One time step of the LSTM of utils/net/common.py Recurrent (torch.nn.LSTM, gate chunks i, f, g, o).  pre [B][4H] holds
 * x W_ih^T + b_ih + h_{t-1} W_hh^T (ts_net_gemm launches); the kernel adds b_hh [4H].  c_prev [B][H] is nullable (zero: t = 0).
 * gates [B][4H] = sigmoid / sigmoid / tanh / sigmoid of the pre-activations (saved for the backward), c [B][H] = f c_prev + i g,
 * h [B][H] = o tanh(c), with full-accuracy expf / tanhf and no atomics.  Any B, H >= 1; rows past B are not touched. */
int ts_lstm_cell(const float* pre, const float* b_hh, const float* c_prev, int64_t B, int32_t H, float* gates, float* c, float* h,
                 ts_stream_t stream);
/* Its backward from the saved gates, c [B][H] (= c_t), c_prev (nullable: zero), the incoming dh [B][H] and the carried dc [B][H]
 * (nullable: zero, the last step): dgates [B][4H], the gradient at the four pre-activations, and dc_prev [B][H] = dc_t f
 * (nullable: not written).  dc and dc_prev may be the same array.  No atomics: two calls on the same input are bit-identical.
 * Any B, H >= 1. */
int ts_lstm_cell_bwd(const float* gates, const float* c, const float* c_prev, const float* dh, const float* dc, int64_t B, int32_t H,
                     float* dgates, float* dc_prev, ts_stream_t stream);

/* ---- IQN (iqn.cu) ---- */
/* The network of IQN (utils/net/discrete.py:163-216) is a trunk on B rows (feat [B][D]), the cosine embedding of S fractions per
 * row and a head on the B * S rows h[b * S + s] = feat[b] * e[b * S + s], sample-major, so the head's output is q [B][S][A].  The
 * GEMMs (the embedding's Linear(C, D) + ReLU included) are ts_net_gemm launches; these are the pieces between them.
 * ts_iqn_cos: out [R][C] = cos(taus[r] * (fl32(pi) * (c + 1))) with both products rounded in fp32, bit for bit the argument the
 * reference's CosineEmbeddingNetwork forms (discrete.py:144-160: np.pi times an fp32 arange, times the fractions), and cosf at
 * full accuracy.  Any R >= 0, C >= 1. */
int ts_iqn_cos(const float* taus, int64_t R, int32_t C, float* out, ts_stream_t stream);
/* ts_iqn_mix: h [B * S][D] = feat [B][D] (row b repeated over its S samples) * e [B * S][D]   (discrete.py:211-214). */
int ts_iqn_mix(const float* feat, const float* e, int64_t B, int32_t S, int32_t D, float* h, ts_stream_t stream);
/* ts_iqn_mix_backward: from dh [B * S][D] = d loss / d h, dfeat [B][D] = (sum_s dh[b * S + s] * e[b * S + s], s in order) times the
 * derivative of the trunk's last activation trunk_act (TS_ACT_NONE / RELU / TANH, at its output trunk_out [B][D], the rule of
 * ts_net_gemm's mask; nullable with TS_ACT_NONE), and de_pre [B * S][D] = dh * feat[b] * 1[e > 0], the gradient at the embedding's
 * pre-activation (e is its ReLU output).  Bit-identical from run to run. */
int ts_iqn_mix_backward(const float* dh, const float* feat, const float* e, int64_t B, int32_t S, int32_t D, int32_t trunk_act,
                        const float* trunk_out, float* dfeat, float* de_pre, ts_stream_t stream);
/* IQN's target distribution (modelfree/qrdqn.py:94-106 through IQNPolicy, iqn.py:72-100): q_online [B][S_on][A] and q_next
 * [B][S_next][A] at s_{t+n} (q_next the lagged network's output on its own fractions, or q_online itself); per row b,
 * m_a = mean_s q_online[b][s][a] in fp32, a* = argmax_a m_a with torch.argmax's rule (lowest index among ties, a NaN is the
 * maximum), out [B][S_next] = q_next[b][.][a*]; act_out [B] (nullable) = a*.  One warp per row, any A, S_on, S_next >= 1, B. */
int ts_iqn_target(const float* q_online, const float* q_next, int64_t B, int32_t A, int32_t S_on, int32_t S_next, float* out,
                  int64_t* act_out, ts_stream_t stream);
/* The quantile-Huber loss of IQN (iqn.py:156-183) on q [B][S_on][A] at s, the fractions taus [B][S_on] of that forward, the n-step
 * returns [B][S_t] and the importance weight [B] (nullable: 1).  With c_i = q[b][i][act[b]], u_ij = returns[b][j] - c_i,
 * h_ij = smooth_l1(u_ij) (beta 1): qr_b = (1/S_on) sum_i sum_j h_ij |taus[b][i] - 1[u_ij <= 0]|, prio [B] = (1/S_on) sum_i sum_j
 * h_ij; losses[4] = (loss, loss, 0, mean_b prio) with loss = mean_b(weight_b qr_b).  dq [B][S_on][A] = d loss / d q, every element
 * written (the indicator detached, as in the reference).  act must lie in [0, A): the caller checks it.  rows [3][B] is scratch.
 * One block per row (threads over the current quantiles, the row's targets in shared memory), then one block summing the rows in
 * a fixed order: two calls on the same input are bit-identical.  Any B, A, S_on >= 1 and S_t <= 12288; larger S_t is refused. */
int ts_iqn_rows(const float* q, const int64_t* act, const float* returns, const float* taus, const float* weight, int64_t B,
                int32_t A, int32_t S_on, int32_t S_t, float* dq, float* prio, float* rows, float* losses, ts_stream_t stream);

/* ---- FQF (fqf.cu) ---- */
/* FQF's network is IQN's, evaluated at fractions that a one-layer fraction net proposes from the trunk's features; the quantile
 * passes are the IQN launches above, the quantile loss is ts_iqn_rows with tau_hats as the per-row fractions.
 * ts_fqf_fractions: the fraction proposal (utils/net/discrete.py:219-252) from the fraction net's output z [B][N]: per row,
 * p [B][N] = softmax(z), logp [B][N] = max(z - logsumexp(z), -FLT_MAX) (Categorical's normalised logits with its entropy's clamp),
 * H [B] = -sum_j logp * p, taus [B][N + 1] = (0, cumsum p) with the cumsum in order in double, rounded to fp32 at each step (as
 * torch's CPU cumsum), tau_hats [B][N] = (taus[:, :-1] + taus[:, 1:]) / 2 and inner [B][N - 1] = taus[:, 1:-1], contiguous, to
 * feed ts_iqn_cos.  One block per row.  Any B >= 0, 2 <= N <= 12288; larger N is refused. */
int ts_fqf_fractions(const float* z, int64_t B, int32_t N, float* taus, float* tau_hats, float* inner, float* p, float* logp,
                     float* H, ts_stream_t stream);
/* FQF's target distribution (fqf.py:94-98, :178-193): q_online [B][N][A] at s_{t+n} on its tau_hats, its fractions taus [B][N + 1],
 * q_next [B][N][A] (the lagged network on the online tau_hats, or q_online itself).  Per row, m_a = sum_n (taus[n + 1] - taus[n]) *
 * q_online[b][n][a] with the widths and products rounded in fp32, a* = argmax_a m_a with torch.argmax's rule (lowest index among
 * ties, a NaN is the maximum), out [B][N] = q_next[b][.][a*]; act_out [B] (nullable) = a*.  One warp per row, any A, N >= 1, B. */
int ts_fqf_target(const float* q_online, const float* taus, const float* q_next, int64_t B, int32_t A, int32_t N, float* out,
                  int64_t* act_out, ts_stream_t stream);
/* FQF's fraction loss (fqf.py:221-247) and its gradient at the fraction net's output.  q_hat [B][N][A] are the quantiles at
 * tau_hats, q_tau [B][N - 1][A] those at taus[:, 1:-1]; taus, p, logp, H are ts_fqf_fractions' outputs.  With the chosen action's
 * quantiles, g_i (i = 1 .. N - 1) is the reference's gradient_of_taus with its strict > / < sign tests; per row
 * fraction_b = sum_i g_i taus[b][i].  dz [B][N] = (1/B) p_j ((G_j - sum_k p_k G_k) + ent_coef (logp_j + H_b)), G_j = sum_{i > j} g_i
 * (0 where p_j is 0): the gradient of fraction_loss - ent_coef * mean_b H.  losses[4] = (fraction_loss - ent_coef * entropy_loss,
 * fraction_loss, entropy_loss, 0) with fraction_loss = mean_b fraction_b and entropy_loss = mean_b H_b; placed after ts_iqn_rows'
 * four, one read returns all of an update's statistics.  act must lie in [0, A): the caller checks it.  rows [3][B] is scratch.
 * One block per row, then one block summing the rows in a fixed order: two calls on the same input are bit-identical.  Any
 * B, A >= 1, 2 <= N <= 12288 and finite ent_coef; anything else is refused. */
int ts_fqf_fraction_rows(const float* q_hat, const float* q_tau, const int64_t* act, const float* taus, const float* p,
                         const float* logp, const float* H, int64_t B, int32_t A, int32_t N, float ent_coef, float* dz, float* rows,
                         float* losses, ts_stream_t stream);

/* ---- imitation learning (imitation.cu) ---- */
/* The regression loss of imitation_base.py:115-118 on a ContinuousActorDeterministic (utils/net/continuous.py: max_action *
 * tanh(last(...))): with z [B][A] the last Linear's output and act [B][A] the buffer's actions (any values, also outside
 * +-max_action), loss[0] = F.mse_loss(max_action * tanh(z), act), the mean over B * A elements, and dz [B][A] = 2 (pi - act) / (B A)
 * * max_action * (1 - tanh(z)^2) in torch's operation order.  dz grid-stride, then one block summing in a fixed order, no
 * atomics: two calls on the same input are bit-identical.  Any B, A >= 1. */
int ts_imitation_mse_rows(const float* z, const float* act, int64_t B, int32_t A, float max_action, float* dz, float* loss,
                          ts_stream_t stream);
/* The classification loss of imitation_base.py:119-122, F.nll_loss(F.log_softmax(y), act), the mean over B.  out [B][A] is the
 * last Linear's output z.  softmax_output = 0: y = z, dz = (softmax(z) - onehot(act)) / B.  softmax_output = 1 (DiscreteActor's
 * default, utils/net/discrete.py:87): y = softmax(z), log_softmax is taken of those probabilities as the reference codes it, and
 * dz = p (g - sum_k p_k g_k) with p = softmax(z), g = (softmax(p) - onehot(act)) / B.  rows [B] receives each row's loss.  One
 * warp per row (lanes stride A, any A), max-shifted log-sum-exps with full-accuracy expf / logf, then one block summing the rows
 * in a fixed order, no atomics: two calls on the same input are bit-identical.  act must lie in [0, A): the caller checks it.
 * Any B, A >= 1. */
int ts_imitation_nll_rows(const float* out, const int64_t* act, int64_t B, int32_t A, int32_t softmax_output, float* dz, float* rows,
                          float* loss, ts_stream_t stream);

/* ---- intrinsic curiosity module (icm.cu) ---- */
/* The inputs of IntrinsicCuriosityModule's two models (utils/net/discrete.py:418-427) from the feature rows phi [2B][F] =
 * [phi1 ; phi2] (one feature-net pass over [obs ; obs_next]): fwd_in [B][F + A] = [phi1 | one_hot(act, A)], inv_in [B][2F] =
 * [phi1 | phi2].  act [B] is int64 (act_f32 = 0) or float32 holding integers (act_f32 = 1); it must lie in [0, A): the caller
 * checks it.  One grid-stride launch; any B, F, A >= 1. */
int ts_icm_inputs(const float* phi, const void* act, int32_t act_f32, int64_t B, int32_t F, int32_t A, float* fwd_in, float* inv_in,
                  ts_stream_t stream);
/* The ICM losses (modelbased/icm.py:77-109) from phi [2B][F], the forward model's output phi2_hat [B][F] and the inverse model's
 * act_hat [B][A], with w = forward_loss_weight:
 *   rows [2][B]    mse[b] = 0.5 sum_j (phi2_hat - phi2)^2, then ce[b] = logsumexp(act_hat[b]) - act_hat[b][act[b]] (max-shifted);
 *   losses [3]     (((1 - w) mean(ce) + w mean(mse)) lr_scale, mean(mse), mean(ce)): a fixed-order one-block sum;
 *   dphi2_hat      lr_scale w / B (phi2_hat - phi2);   dact_hat  lr_scale (1 - w) / B (softmax(act_hat) - onehot(act));
 *   dphi [B:2B][F] -dphi2_hat, the direct term of phi2 (its rows [0:B] are not touched);
 *   rew_out [B]    (nullable) rew_in[b] + (double)(fp32 mse[b] * reward_scale), the intrinsic reward added to the float64 reward;
 *                  an array of its own (the reward column it reads may be a replay buffer's).
 * One warp per row (any F, A), then the one-block sum; no atomics, so two calls on the same input are bit-identical. */
int ts_icm_rows(const float* phi, const float* phi2_hat, const float* act_hat, const void* act, int32_t act_f32, int64_t B, int32_t F,
                int32_t A, float lr_scale, float forward_loss_weight, const double* rew_in, float reward_scale, double* rew_out,
                float* dphi, float* dphi2_hat, float* dact_hat, float* rows, float* losses, ts_stream_t stream);
/* The gradient at the feature net's output, in place in dphi [2B][F] (rows [B:2B] hold ts_icm_rows' direct term): rows b < B
 * become dinv[b][0:F] + dfwd[b], rows B + b add dinv[b][F:2F]; dinv [B][2F] is the inverse model's input gradient, dfwd [B][F]
 * the forward model's over its phi1 columns.  Then times the derivative of the feature net's last activation act (TS_ACT_*) at
 * its output phi [2B][F] (nullable for TS_ACT_NONE).  Grid-stride; any B, F >= 1. */
int ts_icm_feature_grad(float* dphi, const float* dinv, const float* dfwd, const float* phi, int32_t act, int64_t B, int32_t F,
                        ts_stream_t stream);

/* ---- PSRL (algorithm/modelbased/psrl.py) -------------------------------------------------------------------------------------
 * Bytes of the workspace of ts_psrl_update for n rows of an n_state x n_action model.  Its first part (counts of the model's
 * size) must be zero when first used and is left zero by every update; that part's layout does not depend on n, so a workspace
 * sized for one n serves any smaller n. */
int64_t ts_psrl_update_workspace_bytes(int64_t n, int32_t n_state, int32_t n_action);
/* PSRL._update_with_batch + PSRLModel.observe (psrl.py:65-98, :245-276) over n rows, taken in the order perm [n] (int64, a
 * permutation of [0, n): np.random.permutation's order of batch.split(size=1)).  obs / act / obs_next [n] are int64 indices
 * (idx_f32 = 0) or float32 holding them (idx_f32 = 1); rew [n] is float32 or float64 (rew_dtype TS_F32 / TS_F64), squared in
 * float32 when sq_f32 (the buffer's rewards are float32) and in float64 otherwise; done [n] (uint8, nullable unless
 * add_done_loop) adds the self-loops of obs_next: trans_count[s', :, s'] += 1, rew_count[s', :] += 1.
 * The batch sums of each (s, a) run in float64 in the permuted order; the counts are exact.  Then, per element, with
 * explicitly rounded operations: trans_count += counts; sum_count = rew_count + counts; rew_mean = (rew_mean rew_count +
 * rew_sum) / sum_count; rew_square_sum += square sums; rew_std = sqrt(1 / (sum_count / (rew_square_sum / sum_count - rew_mean^2
 * + eps32) + 1 / rew_std_prior^2)); rew_count = sum_count.  The five state arrays are float64 [n_state][n_action](, [n_state]).
 * An index outside its range (negative, not an integer, or >= n_state / n_action) sets result[0] = 1 and changes nothing.
 * result [3] (float64): the error flag, mean(rew_mean), mean(rew_std) (fixed-order sums): one device-to-host copy.
 * The caller checks that every column holds n entries: the kernels read each of them at every row. */
int ts_psrl_update(const void* obs, const void* act, const void* obs_next, int32_t idx_f32, const void* rew, int32_t rew_dtype,
                   int32_t sq_f32, const uint8_t* done, int32_t add_done_loop, const int64_t* perm, int64_t n, int32_t n_state,
                   int32_t n_action, double* trans_count, double* rew_mean, double* rew_std, double* rew_square_sum,
                   double* rew_count, const double* rew_std_prior, void* workspace, int64_t workspace_bytes, double* result,
                   ts_stream_t stream);
/* PSRLModel.observe (psrl.py:65-98) with the batch's dense float64 arrays: trans_count_batch [n_state][n_action][n_state],
 * rew_sum, rew_square_sum_batch, rew_count_batch [n_state][n_action]; the same per-element update as ts_psrl_update.  flag: one
 * int of device scratch.  result [3]: 0, mean(rew_mean), mean(rew_std). */
int ts_psrl_observe(const double* trans_count_batch, const double* rew_sum, const double* rew_square_sum_batch,
                    const double* rew_count_batch, int32_t n_state, int32_t n_action, double* trans_count, double* rew_mean,
                    double* rew_std, double* rew_square_sum, double* rew_count, const double* rew_std_prior, int* flag,
                    double* result, ts_stream_t stream);
/* The most states ts_psrl_value_iteration takes on this device: V [n_state] float64 must fit in one CTA's shared memory. */
int32_t ts_psrl_max_states(void);
/* Bytes of the scratch of ts_psrl_value_iteration (contents ignored). */
int64_t ts_psrl_value_iteration_scratch_bytes(int32_t n_state, int32_t n_action);
/* PSRLModel.value_iteration (psrl.py:116-150) in one cooperative launch of at most one CTA per SM.  trans_prob [n_state]
 * [n_action][n_state], rew and noise [n_state][n_action], value [n_state]: all float64.  Sweeps Q = rew + gamma (P . V),
 * V' = max_a Q, from V = value, while any state has |V' - V| > 1e-8 + eps |V| (np.allclose; NaN is never close), at most
 * max_iterations sweeps.  Converged: value = V' and out[s] = the first argmax_a (Q + eps noise).  Not converged: value and
 * out[0:n_state] are left as they were.  out [n_state + 3] (int64): the policy, the sweep count, 1 if converged, and the bits of
 * max |V' - V| over the last sweep when it was the max_iterations-th.  Each sweep's dot products use one fixed order: reruns are
 * bit-identical.  The caller checks the shapes: the kernel reads and writes every element those shapes name. */
int ts_psrl_value_iteration(const double* trans_prob, const double* rew, const double* noise, int32_t n_state, int32_t n_action,
                            double gamma, double eps, int64_t max_iterations, double* value, void* scratch, int64_t* out,
                            ts_stream_t stream);

#ifdef TS_B200_DIAGNOSTICS
/* Diagnostics build only (libts_b200_diag.so, `python -m tianshou_b200.csrc.build --diag`): not part of the product library. */
/* Hardware self-test of the wgmma building blocks (csrc/wgmma.cuh), one CTA:
 * D[M,N] = a[M,K] * b[N,K]^T with dtype 1 = 3-way bf16 split (the only one; other values are rejected),
 * M in {64,128}, N <= 128, K <= 128 (multiples of 16); a_mn / b_mn place the operand MN-major instead of K-major in
 * shared memory; swap exchanges LBO/SBO (diagnostic).  d receives D row-major [M][N]. */
int ts_umma_selftest(const float* a, const float* b, float* d, int32_t M, int32_t N, int32_t K,
                     int32_t dtype, int32_t a_mn, int32_t b_mn, int32_t swap, ts_stream_t stream);

/* Diagnostics: enable / read the phase timeline (32 x %globaltimer ns) that CTA 0 of the tensor-core
 * PPO step kernel records (csrc/mlp_tc.cu). */
int ts_tc_timeline(int32_t enable, uint64_t* out32 /* host, nullable */);
#endif /* TS_B200_DIAGNOSTICS */


#ifdef __cplusplus
}
#endif
#endif /* TS_B200_H_ */
