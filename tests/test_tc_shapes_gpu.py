"""The tensor-core actor-critic kernels (csrc/mlp_tc.cu) over the network shapes they accept (obs_dim 1..32, act_dim
1..16), against float64 references, with parameters that expose indexing bugs (ts_testutil.perturb_params).

The shape grid reaches the branches the (17, 6) tests never take: obs_dim <= 16 (a single K = 16 layer-1 MMA, the
24-column [X | 1] operand of the dW1 GEMM, two 8-column chunks per staged row), act_dim > 8 (head columns 8..15 on
warpgroups 2-3, action groups a = cq + 4 u beyond 8) and the weight image of every obs_dim."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import oracle_np as onp
from ts_testutil import (build_ppo, named_params, param_offsets, perturb_params, ppo_reference_fp64, record_parity,
                         synth_rollout)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

# (obs_dim, act_dim): every MuJoCo config of the envelope and the edges of both dimensions
# Swimmer 8/2, Hopper 11/3, HalfCheetah / Walker2d 17/6, Ant 27/8; obs 16 / act 8 are the branch boundaries
SHAPES = [(1, 1), (4, 1), (8, 2), (11, 3), (16, 16), (17, 6), (17, 9), (24, 8), (27, 8), (31, 13), (32, 16)]
SHAPE_IDS = [f"obs{o}-act{a}" for o, a in SHAPES]


def _build(obs_dim, act_dim, algo_cls="ppo", **kw):
    """A perturbed PPO / A2C model on the tensor-core path."""
    if algo_cls == "a2c":
        from tianshou_b200.algorithm import A2C, AdamOptimizerFactory, ProbabilisticActorPolicy
        from ts_testutil import Box, build_actor_critic, gaussian_dist
        actor, critic = build_actor_critic(obs_dim, act_dim, DEV)
        policy = ProbabilisticActorPolicy(actor=actor, dist_fn=gaussian_dist, action_scaling=True, action_bound_method="clip",
                                          action_space=Box(act_dim))
        algo = A2C(policy=policy, critic=critic, optim=AdamOptimizerFactory(lr=3e-4), **kw)
    else:
        algo, actor, critic = build_ppo(obs_dim, act_dim, DEV, **kw)
    perturb_params(actor, critic, seed=obs_dim * 100 + act_dim)
    assert algo._flat.weight_image is not None, "this shape must run the tensor-core kernels"
    return algo, actor, critic


def _torch_fp32_forward(actor, critic, obs):
    """torch's own fp32 evaluation of the same layers (CPU), the yardstick for what fp32 can achieve."""
    import copy
    a, c = copy.deepcopy(actor).cpu(), copy.deepcopy(critic).cpu()
    x = torch.from_numpy(obs)
    with torch.no_grad():
        return (c.last.model(c.preprocess.model.model(x)).flatten().numpy(),
                a.mu.model(a.preprocess.model.model(x)).numpy())


# --------------------------------------------------------------------------------------------- forward kernels
@pytest.mark.parametrize("obs_dim,act_dim", SHAPES, ids=SHAPE_IDS)
def test_forward_kernels_vs_fp64(obs_dim, act_dim):
    """ts_critic_forward with two inputs (the second input's tiles) and ts_actor_logp with mu_out, at one row, just below
    and above one tile, and more tiles than two per SM."""
    from tianshou_b200 import ops
    algo, actor, critic = _build(obs_dim, act_dim)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    rng = np.random.default_rng(obs_dim * 31 + act_dim)
    sigma = np.exp(named_params(actor, critic)["a_logstd"].detach().cpu().numpy().reshape(-1))
    for n in (1, 127, 129, 2 * sms * 128 + 5):
        obs = rng.standard_normal((n, obs_dim)).astype(np.float32)
        obs2 = rng.standard_normal((n, obs_dim)).astype(np.float32)
        zeros = np.zeros(n)
        mb = dict(obs=obs, act=np.zeros((n, act_dim)), adv=zeros, returns=zeros, logp_old=zeros, v_s=zeros)
        hp0 = dict(eps_clip=0.2, vf_coef=0.5, ent_coef=0.0, advantage_normalization=False)
        ref = ppo_reference_fp64(actor, critic, mb, hp0)
        act = (ref["mu"] + sigma * rng.standard_normal((n, act_dim))).astype(np.float32)    # actions from the policy
        ref = ppo_reference_fp64(actor, critic, dict(mb, act=act), hp0)
        ref2 = ppo_reference_fp64(actor, critic, dict(mb, obs=obs2), hp0)
        v1, v2 = ops.critic_forward(algo._flat.flat, algo._desc, torch.from_numpy(obs).to(DEV), torch.from_numpy(obs2).to(DEV))
        lp, mu = ops.actor_logp(algo._flat.flat, algo._desc, torch.from_numpy(obs).to(DEV), torch.from_numpy(act).to(DEV),
                                want_mu=True)
        v32, mu32 = _torch_fp32_forward(actor, critic, obs)
        v32b, _ = _torch_fp32_forward(actor, critic, obs2)
        lp32 = torch.distributions.Normal(torch.from_numpy(mu32), torch.from_numpy(sigma.astype(np.float32))).log_prob(
            torch.from_numpy(act)).sum(-1).numpy()
        tag = f"tc_fwd/{obs_dim}x{act_dim}/n{n}"
        for name, got, want, f32 in (("v", v1, ref["v"], v32), ("v_second", v2, ref2["v"], v32b), ("mu", mu, ref["mu"], mu32),
                                     ("logp", lp, ref["logp"], lp32)):
            got = got.cpu().numpy()
            scale = float(np.abs(want).max())
            err_torch = float(np.abs(f32.astype(np.float64) - want).max())
            # bf16x3 products are fp32-faithful: as close to fp64 as torch's own fp32 forward (8x its error), plus a floor of
            # 2e-6 of max |ref| for the MUFU tanh (~1e-7 absolute per activation) where torch's error happens to be tiny
            record_parity(f"{tag}/{name}", got, want, rtol=0.0, atol=8.0 * err_torch + 2e-6 * scale)


# ------------------------------------------------------------------------------------------- ts_ppo_grad
HP_SETS = {
    "vclip_advnorm_ent": dict(algo="ppo", eps_clip=0.2, dual_clip=None, value_clip=True, advantage_normalization=True,
                              vf_coef=0.5, ent_coef=0.01),
    "dual_clip": dict(algo="ppo", eps_clip=0.2, dual_clip=2.0, value_clip=False, advantage_normalization=False,
                      vf_coef=0.25, ent_coef=0.003),
    "a2c": dict(algo="a2c", vf_coef=0.5, ent_coef=0.01),
}


def _guarded_inputs(rng, actor, critic, obs_dim, act_dim, n, hp):
    """Random minibatch inputs around the current policy.  Branch guard: a row whose fp64 ratio lies within 1e-4 of
    1 +- eps_clip (or of dual_clip) gets a new logp_old, a row whose value delta lies within 1e-4 of +-eps_clip (or whose
    two clipped value errors are within 1e-4 of each other) a new v_s -- so the fp32 kernel and the fp64 reference take
    the same side of every clip / min / max, and the comparison measures rounding, not which branch a tie fell on."""
    sigma = np.exp(named_params(actor, critic)["a_logstd"].detach().cpu().numpy().reshape(-1))
    obs = rng.standard_normal((n, obs_dim)).astype(np.float32)
    adv = rng.standard_normal(n).astype(np.float32)
    ret = rng.standard_normal(n).astype(np.float32)
    zeros = np.zeros(n)
    mb = dict(obs=obs, act=np.zeros((n, act_dim)), adv=adv, returns=ret, logp_old=zeros, v_s=zeros)
    ref = ppo_reference_fp64(actor, critic, mb, hp)
    mb["act"] = (ref["mu"] + sigma * rng.standard_normal((n, act_dim))).astype(np.float32)
    ref = ppo_reference_fp64(actor, critic, mb, hp)
    logp, v = ref["logp"], ref["v"]
    lpo = (logp + 0.5 * rng.standard_normal(n)).astype(np.float32)
    v_s = (v + 0.3 * rng.standard_normal(n)).astype(np.float32)
    eps, dual = hp.get("eps_clip", 0.0), hp.get("dual_clip") or 0.0
    for _ in range(100):
        ratio = np.exp(logp - lpo.astype(np.float64))
        bad = (np.abs(ratio - (1 - eps)) < 1e-4) | (np.abs(ratio - (1 + eps)) < 1e-4) | (np.abs(ratio - dual) < 1e-4)
        if not bad.any():
            break
        lpo[bad] = (logp[bad] + 0.5 * rng.standard_normal(int(bad.sum()))).astype(np.float32)
    for _ in range(100):
        dlt = v - v_s.astype(np.float64)
        v_clip = v_s + np.clip(dlt, -eps, eps)
        tie = (np.abs(dlt) > eps) & (np.abs(np.abs(ret - v) - np.abs(ret - v_clip)) < 1e-4)
        bad = (np.abs(np.abs(dlt) - eps) < 1e-4) | tie
        if not bad.any():
            break
        v_s[bad] = (v[bad] + 0.3 * rng.standard_normal(int(bad.sum()))).astype(np.float32)
    mb.update(logp_old=lpo, v_s=v_s)
    return mb


@pytest.mark.parametrize("hp_name", list(HP_SETS))
@pytest.mark.parametrize("obs_dim,act_dim", SHAPES, ids=SHAPE_IDS)
def test_ppo_grad_kernel_vs_fp64(obs_dim, act_dim, hp_name):
    """ts_ppo_grad (ppo_tc_kernel<false>, weights staged by the CTA) on 300 permuted rows -- three tiles, the last one
    partial: every parameter gradient and the four loss sums against torch autograd in float64."""
    from tianshou_b200._cabi import call, ptr, stream_ptr
    cfg = dict(HP_SETS[hp_name])
    kind = cfg.pop("algo")
    if kind == "a2c":
        algo, actor, critic = _build(obs_dim, act_dim, "a2c", **cfg)
        hpr = dict(loss_kind="a2c", vf_coef=cfg["vf_coef"], ent_coef=cfg["ent_coef"], advantage_normalization=False)
    else:
        algo, actor, critic = _build(obs_dim, act_dim, **cfg)
        hpr = dict(cfg, adv_eps=1e-8)
    hp = algo._loss_hparams()
    rng = np.random.default_rng(obs_dim * 7 + act_dim)
    n, lo, hi = 700, 37, 337
    full = _guarded_inputs(rng, actor, critic, obs_dim, act_dim, n, hpr)
    perm = rng.permutation(n).astype(np.int32)
    idx = perm[lo:hi]
    ref = ppo_reference_fp64(actor, critic, {k: v[idx] for k, v in full.items()}, hpr)

    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    f = algo._flat
    d = {k: t(full[k]) for k in ("obs", "act", "adv", "returns", "logp_old", "v_s")}
    d_perm = t(perm)
    adv_mom = None
    if hp.advantage_normalization:
        sums = torch.zeros(2, dtype=torch.float64, device=DEV)
        adv_mom = torch.zeros(2, dtype=torch.float32, device=DEV)
        call("ts_minibatch_adv_sums", ptr(d["adv"]), ptr(d_perm), lo, hi, ptr(sums), stream_ptr())
        call("ts_adv_moments_finalize", ptr(sums), hi - lo, ptr(adv_mom), stream_ptr())
    f.grad.zero_()
    n_part = C.c_int32(0)
    call("ts_ppo_grad", ptr(f.flat), C.byref(algo._desc), C.byref(hp), ptr(d["obs"]), ptr(d["act"]), ptr(d["adv"]),
         ptr(d["returns"]), ptr(d["logp_old"]), ptr(d["v_s"]), ptr(d_perm), lo, hi, hi - lo, ptr(adv_mom), ptr(f.partials),
         C.byref(n_part), stream_ptr())
    assert n_part.value == 3
    call("ts_grad_reduce", ptr(f.partials), n_part.value, C.byref(algo._desc), ptr(f.grad), stream_ptr())
    got = f.grad.cpu().numpy()
    f.grad.zero_()
    tag = f"tc_grad/{hp_name}/{obs_dim}x{act_dim}"
    # the gradients are read at the offsets where the modules' own parameters live (checks the descriptor's mapping)
    for k, off in param_offsets(f.flat, actor, critic).items():
        want = ref["grads"][k]
        gk = got[off:off + want.size].reshape(want.shape)
        # Head bias and log-std gradients are fp32 column sums: the bar of test_ppo_grad_kernel_vs_oracle.  Every other
        # gradient leaves a weight-gradient MMA in the three-product bf16 scheme (kWgradFull = false: a0 b0 + a0 b1 + a1 b0,
        # up to ~3 * 2^-16 = 4.6e-5 relative per product); with non-zero biases and a full-scale head they are sums of
        # cancelling per-row terms, so the absolute term is 1e-4 of max |ref| (observed up to 4.3e-5 at obs 1 / act 1)
        gemm = k[2] in "wb" and k[2:] != "b3"
        atol = (1e-4 if gemm else 2e-5) * max(1e-6, float(np.abs(want).max())) + 1e-7
        record_parity(f"{tag}/{k}", gk, want, rtol=2e-4, atol=atol)
    ex = got[f.n:f.n + 4]
    B = hi - lo
    assert ex[3] == B
    record_parity(f"{tag}/clip_loss", -ex[0] / B, ref["clip"], rtol=1e-4, atol=1e-6)
    record_parity(f"{tag}/vf_loss", ex[1] / B, ref["vf"], rtol=1e-4, atol=1e-6)
    record_parity(f"{tag}/ent_loss", ex[2] / B, ref["ent"], rtol=1e-5, atol=1e-6)


# ---------------------------------------------------------------------------------- epoch kernel via PPO.update
EPOCH_KW = dict(gamma=0.99, gae_lambda=0.95, max_grad_norm=0.5, vf_coef=0.25, ent_coef=0.01, return_scaling=True,
                eps_clip=0.2, value_clip=True, dual_clip=None, advantage_normalization=True, recompute_advantage=True)
EPOCH_HP = dict(eps_clip=0.2, dual_clip=None, vf_coef=0.25, ent_coef=0.01, max_grad_norm=0.5, adv_eps=1e-8, value_clip=True,
                advantage_normalization=True, lr=3e-4, beta1=0.9, beta2=0.999, adam_eps=1e-8, weight_decay=0.0)


def _rollout(obs_dim, act_dim, E, T, seed):
    from tianshou_b200.data import Batch, VectorReplayBuffer
    buf = VectorReplayBuffer(E * T, E, device=DEV)
    for s in synth_rollout(np.random.default_rng(seed), E, T, obs_dim, act_dim, p_term=0.03, trunc_len=15):
        buf.add(Batch(**s), buffer_ids=np.arange(E))
    N = E * T
    last = np.arange(E) * T + T - 1
    unf = np.zeros(N, dtype=bool)
    unf[last] = ~buf.done[last]
    roll = dict(obs=buf.obs.copy(), obs_next=buf.obs_next.copy(), act=buf.act.copy(), rew=buf.rew.copy(),
                terminated=buf.terminated.copy(), truncated=buf.truncated.copy(), unfinished=unf)
    return buf, roll


def _epoch_vs_oracle(obs_dim, act_dim, E, T, bs, repeat, tag):
    from tianshou_b200.utils import policy_within_training_step
    algo, actor, critic = _build(obs_dim, act_dim, **EPOCH_KW)
    p = {k: v.detach().cpu().numpy().copy() for k, v in named_params(actor, critic).items()}
    buf, roll = _rollout(obs_dim, act_dim, E, T, seed=obs_dim + 1000 * act_dim)
    N = E * T
    np.random.seed(4)
    perms = np.stack([np.random.permutation(N) for _ in range(repeat)])
    m = {k: np.zeros_like(v) for k, v in p.items()}
    v = {k: np.zeros_like(x) for k, x in p.items()}
    rms = onp.RunningMeanStd()
    res = onp.ppo_update(p, m, v, 0, roll, perms, bs, repeat, EPOCH_HP, rms, 0.99, 0.95, True)
    np.random.seed(4)
    with policy_within_training_step(algo.policy):
        stats = algo.update(buffer=buf, batch_size=bs, repeat=repeat)
    bounds = onp.minibatch_bounds(N, bs)
    assert stats.gradient_steps == repeat * len(bounds) == res["losses"].shape[0]
    table = algo.last_loss_table
    # Row 0 is computed from identical parameters: the bar of test_ppo_update_matches_reference.  The absolute term is in
    # units of max |column|, except the actor loss: with normalised advantages and ratio ~1 it is a cancelling mean of O(1)
    # per-row terms (~1e-8 at row 0), so its unit is 1.  Later rows follow two Adam trajectories: an element whose gradient
    # is a rounding-level cancellation gets a step of up to +-lr whose sign rounding decides (the reason for the
    # parameters' 0.1 lr floor); with a full-scale head and sigma down to 0.3 that moves later losses by up to 1e-3 (observed
    # at obs 16 / act 16, batch 64, 32 steps): 3e-3 of the unit there
    for col, name in enumerate(["loss", "actor_loss", "vf_loss", "ent_loss", "grad_norm"]):
        # column 4: the total gradient norm of each step before clipping (the kernel's fp64 sum of squares of the folded
        # gradient vs clip_grad_norm_'s)
        ref = res["grad_norms"] if col == 4 else res["losses"][:, col]
        unit = max(1e-3, float(np.abs(ref).max()), 1.0 if name == "actor_loss" else 0.0)
        record_parity(f"{tag}/step0_{name}", table[:1, col], ref[:1], rtol=2e-4, atol=2e-5 * unit)
        record_parity(f"{tag}/per_step_{name}", table[:, col], ref, rtol=1e-3, atol=3e-3 * unit)
    assert np.array_equal(table[:, 5], np.tile([hi - lo for lo, hi in bounds], repeat))
    steps = res["losses"].shape[0]
    for k, pv in named_params(actor, critic).items():
        # test_ppo_update_matches_reference's bar (1e-3 relative + 0.1 lr) per optimiser step: the rounding-decided Adam
        # steps above accumulate over the update (observed 1.3 lr after the 32 steps of obs 24 / act 8, batch 64)
        record_parity(f"{tag}/param_{k}", pv.detach().cpu().numpy(), p[k], rtol=1e-3, atol=0.1 * 3e-4 * steps)


@pytest.mark.parametrize("bs", [300, 64])      # 300: merged last minibatch (widest > mb_size); 64: below one tile
@pytest.mark.parametrize("obs_dim,act_dim", SHAPES, ids=SHAPE_IDS)
def test_epoch_kernel_update_vs_oracle(obs_dim, act_dim, bs):
    """PPO.update (persistent epoch kernel, weight image) on a 1000-row rollout, repeat 2, against the numpy oracle: the
    loss table row by row including the gradient norm, and the parameters after the update."""
    _epoch_vs_oracle(obs_dim, act_dim, 20, 50, bs, 2, f"tc_epoch/{obs_dim}x{act_dim}/bs{bs}")


def test_epoch_kernel_multi_tile_per_cta_vs_oracle():
    """Hopper-shaped network, 65536 rows in minibatches of 32768 = 256 tiles: every CTA handles several tiles per step."""
    _epoch_vs_oracle(11, 3, 512, 128, 32768, 2, "tc_epoch/11x3/bs32768")


@pytest.mark.parametrize("obs_dim,act_dim", SHAPES, ids=SHAPE_IDS)
def test_epoch_kernel_weight_image_matches_staged_weights(obs_dim, act_dim):
    """The epoch kernel gets the weights into shared memory either by one bulk copy of the pre-split weight image or, with
    no image, by gathering and splitting them in the CTA (stage_weights).  Both stage the same bf16 pieces and the same
    Gaussian constants, so two identical models updated on the same data must agree bit for bit."""
    from tianshou_b200.utils import policy_within_training_step
    runs = []
    for use_image in (True, False):
        algo, actor, critic = _build(obs_dim, act_dim, **EPOCH_KW)
        if not use_image:
            algo._flat.weight_image = None
        buf, _ = _rollout(obs_dim, act_dim, 20, 50, seed=7)
        np.random.seed(9)
        with policy_within_training_step(algo.policy):
            algo.update(buffer=buf, batch_size=300, repeat=2)
        f = algo._flat
        runs.append(dict(params=f.flat.cpu().numpy().copy(), exp_avg=f.exp_avg.cpu().numpy().copy(),
                         exp_avg_sq=f.exp_avg_sq.cpu().numpy().copy(), table=algo.last_loss_table.copy()))
    for k in runs[0]:
        a, b = runs[0][k], runs[1][k]
        assert np.array_equal(a, b), f"{k}: image and staged weights differ, max |diff| {np.abs(a - b).max():.3e}"
