"""PPO update parity on the GPU: kernels vs the numpy oracle, and the public
``PPO.update(buffer, batch_size, repeat)`` vs the outputs of the imported reference
(tests/golden/ppo_ref_*.npz: same initial weights, same buffer contents, same numpy seed)."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import oracle_np as onp
from ts_testutil import PARAM_ORDER, build_ppo, load_golden, named_params, record_parity, restore_vector_buffer, synth_rollout

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _opt(g, k):
    v = float(g["kw_" + k])
    return None if np.isnan(v) else v


def ppo_kwargs(g):
    return dict(gamma=float(g["kw_gamma"]), gae_lambda=float(g["kw_gae_lambda"]), max_grad_norm=_opt(g, "max_grad_norm"),
                vf_coef=float(g["kw_vf_coef"]), ent_coef=float(g["kw_ent_coef"]),
                return_scaling=bool(g["kw_return_scaling"]), eps_clip=float(g["kw_eps_clip"]),
                value_clip=bool(g["kw_value_clip"]), dual_clip=_opt(g, "dual_clip"),
                advantage_normalization=bool(g["kw_advantage_normalization"]),
                recompute_advantage=bool(g["kw_recompute_advantage"]))


def flat_dict(actor, critic):
    return {k: v.detach().cpu().numpy().copy() for k, v in named_params(actor, critic).items()}


# ------------------------------------------------------------------------------ forward kernels
def test_critic_and_logp_kernels_vs_oracle():
    from tianshou_b200 import ops
    g = load_golden("ppo_ref_A.npz")
    algo, actor, critic = build_ppo(17, 6, DEV, params={k: g["p0_" + k] for k in PARAM_ORDER}, **ppo_kwargs(g))
    p = flat_dict(actor, critic)
    rng = np.random.default_rng(0)
    for n in (1, 127, 128, 129, 1000, 20_000):
        obs = rng.standard_normal((n, 17)).astype(np.float32)
        obs2 = rng.standard_normal((n, 17)).astype(np.float32)
        act = rng.standard_normal((n, 6)).astype(np.float32)
        v1, v2 = ops.critic_forward(algo._flat.flat, algo._desc, torch.from_numpy(obs).to(DEV), torch.from_numpy(obs2).to(DEV))
        np.testing.assert_allclose(v1.cpu().numpy(), onp.critic_forward(p, obs), rtol=1e-5, atol=2e-6)
        np.testing.assert_allclose(v2.cpu().numpy(), onp.critic_forward(p, obs2), rtol=1e-5, atol=2e-6)
        lp, mu = ops.actor_logp(algo._flat.flat, algo._desc, torch.from_numpy(obs).to(DEV), torch.from_numpy(act).to(DEV),
                                want_mu=True)
        mu_ref, sigma, _, _ = onp.actor_forward(p, obs)
        np.testing.assert_allclose(mu.cpu().numpy(), mu_ref, rtol=1e-5, atol=2e-6)
        np.testing.assert_allclose(lp.cpu().numpy(), onp.normal_logp(act, mu_ref, sigma), rtol=1e-5, atol=1e-5)
        # and against the torch modules that share the same storage
        with torch.no_grad():
            v_t = critic(torch.from_numpy(obs).to(DEV)).flatten()
        np.testing.assert_allclose(v1.cpu().numpy(), v_t.cpu().numpy(), rtol=1e-5, atol=2e-6)


@pytest.mark.parametrize("variant", ["A", "B"])
def test_ppo_grad_kernel_vs_oracle(variant):
    """One minibatch: gradients and loss sums of ts_ppo_grad vs the manual-backward oracle."""
    from tianshou_b200._cabi import call, ptr, stream_ptr
    g = load_golden(f"ppo_ref_{variant}.npz")
    algo, actor, critic = build_ppo(17, 6, DEV, params={k: g["p0_" + k] for k in PARAM_ORDER}, **ppo_kwargs(g))
    p = flat_dict(actor, critic)
    rng = np.random.default_rng(1)
    n = 700
    obs = rng.standard_normal((n, 17)).astype(np.float32)
    act = (rng.standard_normal((n, 6)) * 0.7).astype(np.float32)
    adv = rng.standard_normal(n).astype(np.float32)
    ret = rng.standard_normal(n).astype(np.float32)
    v_s = (ret + 0.3 * rng.standard_normal(n)).astype(np.float32)
    mu, sigma, _, _ = onp.actor_forward(p, obs)
    logp_old = (onp.normal_logp(act, mu, sigma) + 0.3 * rng.standard_normal(n)).astype(np.float32)
    perm = rng.permutation(n).astype(np.int32)
    lo, hi = 37, 37 + 300
    hp = algo._ppo_hparams()
    hpd = dict(eps_clip=hp.eps_clip, dual_clip=hp.dual_clip or None, vf_coef=hp.vf_coef, ent_coef=hp.ent_coef,
               adv_eps=1e-8, value_clip=bool(hp.value_clip), advantage_normalization=bool(hp.advantage_normalization))
    idx = perm[lo:hi]
    mb = dict(obs=obs[idx], act=act[idx], adv=adv[idx], returns=ret[idx], logp_old=logp_old[idx], v_s=v_s[idx])
    grads, (loss, clip, vf, ent) = onp.ppo_minibatch_grad(p, mb, hpd)

    t = lambda a: torch.from_numpy(a).to(DEV)
    f = algo._flat
    f.grad.zero_()
    adv_mom = None
    d_obs, d_act, d_adv, d_ret, d_lpo, d_vs, d_perm = t(obs), t(act), t(adv), t(ret), t(logp_old), t(v_s), t(perm)
    if hp.advantage_normalization:
        sums = torch.zeros(2, dtype=torch.float64, device=DEV)
        adv_mom = torch.zeros(2, dtype=torch.float32, device=DEV)
        call("ts_minibatch_adv_sums", ptr(d_adv), ptr(d_perm), lo, hi, ptr(sums), stream_ptr())
        call("ts_adv_moments_finalize", ptr(sums), hi - lo, ptr(adv_mom), stream_ptr())
        np.testing.assert_allclose(adv_mom.cpu().numpy(), [adv[idx].mean(), adv[idx].std(ddof=1)], rtol=1e-5)
    n_part = C.c_int32(0)
    call("ts_ppo_grad", ptr(f.flat), C.byref(algo._desc), C.byref(hp), ptr(d_obs), ptr(d_act), ptr(d_adv), ptr(d_ret),
         ptr(d_lpo), ptr(d_vs), ptr(d_perm), lo, hi, hi - lo, ptr(adv_mom), ptr(f.partials), C.byref(n_part), stream_ptr())
    assert n_part.value == 3          # 300 rows -> three 128-row tiles, one partial row each
    call("ts_grad_reduce", ptr(f.partials), n_part.value, C.byref(algo._desc), ptr(f.grad), stream_ptr())
    got = f.grad.cpu().numpy()
    off = 0
    for k in PARAM_ORDER:
        sz = p[k].size
        gk = got[off:off + sz].reshape(p[k].shape)
        scale = max(1e-6, float(np.abs(grads[k]).max()))
        np.testing.assert_allclose(gk, grads[k], rtol=2e-4, atol=2e-5 * scale + 1e-7, err_msg=k)
        off += sz
    B = hi - lo
    np.testing.assert_allclose(-got[off] / B, clip, rtol=1e-4, atol=1e-6)
    np.testing.assert_allclose(got[off + 1] / B, vf, rtol=1e-4, atol=1e-6)
    np.testing.assert_allclose(got[off + 2] / B, ent, rtol=1e-5)
    assert got[off + 3] == B
    f.grad.zero_()


# ------------------------------------------------------------------------- public update() path
@pytest.mark.parametrize("variant", ["A", "B", "C", "D"])
def test_ppo_update_matches_reference(variant):
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden(f"ppo_ref_{variant}.npz")
    E, cap = int(g["cfg_E"]), int(g["cfg_cap"])
    bs = int(g["cfg_bs"])
    bs = None if bs < 0 else bs
    repeat = int(g["cfg_repeat"])
    kw = ppo_kwargs(g)
    lr = float(g["kw_lr"]) if "kw_lr" in g.files else 3e-4
    algo, actor, critic = build_ppo(17, 6, DEV, lr=lr, params={k: g["p0_" + k] for k in PARAM_ORDER}, **kw)
    captured = {}
    orig = algo._preprocess_batch

    def hook(batch, buffer, indices):
        b = orig(batch, buffer, indices)
        captured["pre"] = {k: b[k].detach().cpu().numpy().copy() for k in ("v_s", "returns", "adv", "logp_old")}
        captured["indices"] = indices.cpu().numpy().copy()
        return b

    algo._preprocess_batch = hook
    for u in range(2):
        o = f"u{u}_"
        buf = restore_vector_buffer(g, o, E, cap, device=DEV)
        np.random.seed(1000 + u)
        with policy_within_training_step(algo.policy):
            stats = algo.update(buffer=buf, batch_size=bs, repeat=repeat)
        assert np.array_equal(captured["indices"], g[o + "indices"])                  # sample(0) order, bit-exact
        pre = captured["pre"]
        # North star: returns / advantages within 1e-5 relative of the reference's fp32 results.  Tolerance used here:
        # |err| <= 1e-5 * |ref| + 1e-5 * max|ref|  (elementwise relative + an absolute floor scaled to the column, because
        # advantages cross zero); observed errors are recorded in gpurun_out/parity_report.json.
        tag = f"ppo_{variant}_u{u}"
        for k in ("v_s", "returns", "adv", "logp_old"):
            ref = g[o + k]
            record_parity(f"{tag}/{k}", pre[k], ref, rtol=1e-5, atol=1e-5 * float(np.abs(ref).max()))
        assert stats.gradient_steps == int(g[o + "gradient_steps"])
        ref_losses = g[o + "losses"]                       # [steps, 4]: what ppo.py:213-216 appended per optimiser step
        table = algo.last_loss_table
        assert table.shape[0] == ref_losses.shape[0]
        for col, name in enumerate(["loss", "actor_loss", "vf_loss", "ent_loss"]):
            # per-minibatch, row by row (not only mean / min / max)
            record_parity(f"{tag}/per_step_{name}", table[:, col], ref_losses[:, col], rtol=2e-4,
                          atol=2e-5 * max(1e-3, float(np.abs(ref_losses[:, col]).max())))
            s = getattr(stats, name)
            np.testing.assert_allclose(s.mean, ref_losses[:, col].mean(), rtol=2e-4, atol=2e-5, err_msg=name)
        for k, pv in named_params(actor, critic).items():
            # Adam divides by sqrt(v): at step t a gradient difference of relative size e moves the parameter by up to
            # ~lr * e / (1 - beta1) -- the absolute term is stated in units of one Adam step (lr)
            record_parity(f"{tag}/param_{k}", pv.detach().cpu().numpy(), g[o + "p_" + k], rtol=1e-3, atol=0.1 * lr)
        if kw["return_scaling"]:
            np.testing.assert_allclose([algo.ret_rms.mean, algo.ret_rms.var, algo.ret_rms.count], g[o + "rms"], rtol=1e-5)
        assert stats.train_time > 0


def test_update_outside_training_step_raises():
    g = load_golden("ppo_ref_D.npz")
    algo, _, _ = build_ppo(17, 6, DEV, **ppo_kwargs(g))
    buf = restore_vector_buffer(g, "u0_", int(g["cfg_E"]), int(g["cfg_cap"]), device=DEV)
    with pytest.raises(RuntimeError):
        algo.update(buffer=buf, batch_size=64, repeat=1)


def test_state_dict_round_trip_and_module_views():
    """Parameters stay ordinary nn.Parameters (views of the flat buffer); optimizer state exports
    in torch.optim.Adam format and reloads (SURVEY 5: checkpoint / resume)."""
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden("ppo_ref_A.npz")
    kw = ppo_kwargs(g)
    algo, actor, critic = build_ppo(17, 6, DEV, params={k: g["p0_" + k] for k in PARAM_ORDER}, **kw)
    buf = restore_vector_buffer(g, "u0_", int(g["cfg_E"]), int(g["cfg_cap"]), device=DEV)
    np.random.seed(1000)
    with policy_within_training_step(algo.policy):
        algo.update(buffer=buf, batch_size=128, repeat=1)
    sd = algo.state_dict()
    assert "_optimizers" in sd and len(sd["_optimizers"][0]["state"]) == 13
    assert float(sd["_optimizers"][0]["state"][0]["step"]) == 4.0
    algo2, actor2, critic2 = build_ppo(17, 6, DEV, **kw)
    algo2.load_state_dict(sd)
    for (k, a), (_, b) in zip(named_params(actor, critic).items(), named_params(actor2, critic2).items(), strict=True):
        assert torch.equal(a, b), k
    assert torch.equal(algo._flat.exp_avg, algo2._flat.exp_avg) and torch.equal(algo._flat.exp_avg_sq, algo2._flat.exp_avg_sq)
    assert int(algo2._flat.step.item()) == 4
    # both continue identically (the running return statistics are a plain attribute, not part of the
    # state_dict -- in the reference too, a2c.py:112)
    import copy
    algo2.ret_rms = copy.deepcopy(algo.ret_rms)
    for a in (algo, algo2):
        np.random.seed(7)
        with policy_within_training_step(a.policy):
            a.update(buffer=buf, batch_size=128, repeat=1)
    for (k, a), (_, b) in zip(named_params(actor, critic).items(), named_params(actor2, critic2).items(), strict=True):
        np.testing.assert_allclose(a.detach().cpu().numpy(), b.detach().cpu().numpy(), rtol=1e-5, atol=1e-7, err_msg=k)


def test_device_shuffle_is_a_permutation_and_trains():
    from tianshou_b200 import ops
    from tianshou_b200.utils import policy_within_training_step
    for n in (1, 2, 5, 1000, 4096 * 128):
        perms = ops.make_permutation(123, 0, 3, n, torch.device(DEV)).cpu().numpy()
        for r in range(3):
            assert np.array_equal(np.sort(perms[r]), np.arange(n))
        if n > 100:
            assert not np.array_equal(perms[0], perms[1])
            assert not np.array_equal(perms[0], np.arange(n))
    g = load_golden("ppo_ref_A.npz")
    algo, actor, critic = build_ppo(17, 6, DEV, params={k: g["p0_" + k] for k in PARAM_ORDER},
                                    minibatch_shuffle="device", **ppo_kwargs(g))
    buf = restore_vector_buffer(g, "u0_", int(g["cfg_E"]), int(g["cfg_cap"]), device=DEV)
    with policy_within_training_step(algo.policy):
        stats = algo.update(buffer=buf, batch_size=128, repeat=3)
    assert stats.gradient_steps == 12
    # same data, same hyper-parameters, different minibatch composition: close to the reference run
    np.testing.assert_allclose(stats.vf_loss.mean, g["u0_losses"][:, 2].mean(), rtol=0.05)


@pytest.mark.parametrize("bs", [16384, 32768, None])   # 128 tiles (one per CTA), 256 and 512 tiles (several per CTA)
def test_large_rollout_update_vs_oracle(bs):
    """Config-2-shaped slice (512 envs x 128 steps) through the public API vs the numpy oracle; the larger
    minibatches exercise the multi-tile-per-CTA path of the persistent kernel (gradient rows accumulated, not stored)."""
    from tianshou_b200.data import Batch, VectorReplayBuffer
    from tianshou_b200.utils import policy_within_training_step
    E, T = 512, 128
    kw = dict(gamma=0.99, gae_lambda=0.95, max_grad_norm=0.5, vf_coef=0.25, ent_coef=0.0, return_scaling=True,
              eps_clip=0.2, value_clip=True, dual_clip=None, advantage_normalization=False, recompute_advantage=True)
    algo, actor, critic = build_ppo(17, 6, DEV, **kw)
    p = {k: v.detach().cpu().numpy().copy() for k, v in named_params(actor, critic).items()}
    buf = VectorReplayBuffer(E * T, E, device=DEV)
    rng = np.random.default_rng(0)
    for s in synth_rollout(rng, E, T, 17, 6):
        buf.add(Batch(**s), buffer_ids=np.arange(E))
    N = E * T
    idx = np.arange(N)
    unf = np.zeros(N, dtype=bool)
    unf[np.arange(E) * T + T - 1] = ~buf.done[np.arange(E) * T + T - 1]
    roll = dict(obs=buf.obs[idx], obs_next=buf.obs_next[idx], act=buf.act[idx], rew=buf.rew[idx],
                terminated=buf.terminated[idx].copy(), truncated=buf.truncated[idx], unfinished=unf)
    np.random.seed(0)
    perms = np.stack([np.random.permutation(N) for _ in range(2)])
    m = {k: np.zeros_like(v) for k, v in p.items()}
    v = {k: np.zeros_like(vv) for k, vv in p.items()}
    hp = dict(eps_clip=0.2, dual_clip=None, vf_coef=0.25, ent_coef=0.0, max_grad_norm=0.5, adv_eps=1e-8, value_clip=True,
              advantage_normalization=False, lr=3e-4, beta1=0.9, beta2=0.999, adam_eps=1e-8, weight_decay=0.0)
    rms = onp.RunningMeanStd()
    res = onp.ppo_update(p, m, v, 0, roll, perms, bs, 2, hp, rms, 0.99, 0.95, True)
    np.random.seed(0)
    with policy_within_training_step(algo.policy):
        stats = algo.update(buffer=buf, batch_size=bs, repeat=2)
    assert stats.gradient_steps == 2 * (N // bs if bs else 1)
    np.testing.assert_allclose(stats.loss.mean, res["losses"][:, 0].mean(), rtol=1e-3, atol=1e-5)
    np.testing.assert_allclose(stats.vf_loss.mean, res["losses"][:, 2].mean(), rtol=1e-3, atol=1e-5)
    for k, pv in named_params(actor, critic).items():
        np.testing.assert_allclose(pv.detach().cpu().numpy(), p[k], rtol=2e-3, atol=3e-5, err_msg=k)
    np.testing.assert_allclose([algo.ret_rms.mean, algo.ret_rms.var, algo.ret_rms.count],
                               [rms.mean, rms.var, rms.count], rtol=1e-5)


@pytest.mark.parametrize("name,E,T,bs,repeat", [("C2_full", 4096, 128, 16384, 1), ("C5_slice", 1024, 256, 32768, 1)])
def test_full_size_update_vs_oracle(name, E, T, bs, repeat):
    """BASELINE configs[1] at FULL size (4096 envs x 128 steps, minibatch 16384) and a configs[4]-shaped slice (256-step
    rollouts, minibatch N/8) through the public ``update()``: v_s / returns / adv / logp_old at the north star's 1e-5,
    the per-minibatch loss table row by row, and the post-update parameters, against the numpy oracle."""
    from oracle import oracle_c
    from tianshou_b200.data import VectorReplayBuffer
    from tianshou_b200.synthetic import fill_vector_buffer
    from tianshou_b200.utils import policy_within_training_step
    kw = dict(gamma=0.99, gae_lambda=0.95, max_grad_norm=0.5, vf_coef=0.25, ent_coef=0.0, return_scaling=True,
              eps_clip=0.2, value_clip=True, dual_clip=None, advantage_normalization=False, recompute_advantage=True)
    algo, actor, critic = build_ppo(17, 6, DEV, **kw)
    p = {k: v.detach().cpu().numpy().copy() for k, v in named_params(actor, critic).items()}
    buf = VectorReplayBuffer(E * T, E, device=DEV)
    fill_vector_buffer(buf, np.random.default_rng(5), E, T, 17, 6)
    N = E * T
    last = np.arange(E) * T + T - 1
    unf = np.zeros(N, dtype=bool)
    unf[last] = ~buf.done[last]
    roll = dict(obs=buf.obs.copy(), obs_next=buf.obs_next.copy(), act=buf.act.copy(), rew=buf.rew.copy(),
                terminated=buf.terminated.copy(), truncated=buf.truncated.copy(), unfinished=unf)
    np.random.seed(11)
    perms = np.stack([np.random.permutation(N) for _ in range(repeat)])
    m = {k: np.zeros_like(v) for k, v in p.items()}
    v = {k: np.zeros_like(vv) for k, vv in p.items()}
    hp = dict(eps_clip=0.2, dual_clip=None, vf_coef=0.25, ent_coef=0.0, max_grad_norm=0.5, adv_eps=1e-8, value_clip=True,
              advantage_normalization=False, lr=3e-4, beta1=0.9, beta2=0.999, adam_eps=1e-8, weight_decay=0.0)
    rms = onp.RunningMeanStd()
    gae_py = onp.gae
    onp.gae = lambda v_s, v_s_, rew, end, gamma, lam: oracle_c.gae(v_s, v_s_, rew, end, gamma, lam)   # the C loop (numba in the reference)
    try:
        res = onp.ppo_update(p, m, v, 0, roll, perms, bs, repeat, hp, rms, 0.99, 0.95, True)
    finally:
        onp.gae = gae_py
    captured = {}
    orig = algo._preprocess_batch

    def hook(batch, buffer, indices):
        b = orig(batch, buffer, indices)
        captured.update({k: b[k].detach().cpu().numpy().copy() for k in ("v_s", "returns", "adv", "logp_old")})
        return b

    algo._preprocess_batch = hook
    np.random.seed(11)
    with policy_within_training_step(algo.policy):
        stats = algo.update(buffer=buf, batch_size=bs, repeat=repeat)
    assert stats.gradient_steps == repeat * (N // bs)
    for k in ("v_s", "returns", "adv", "logp_old"):
        ref = res["first"][k]
        record_parity(f"{name}/{k}", captured[k], ref, rtol=1e-5, atol=1e-5 * float(np.abs(ref).max()))
    table = algo.last_loss_table
    for col, nm in enumerate(["loss", "actor_loss", "vf_loss", "ent_loss"]):
        ref = res["losses"][:, col]
        record_parity(f"{name}/per_step_{nm}", table[:, col], ref, rtol=2e-4, atol=2e-5 * max(1e-3, float(np.abs(ref).max())))
    for k, pv in named_params(actor, critic).items():
        record_parity(f"{name}/param_{k}", pv.detach().cpu().numpy(), p[k], rtol=1e-3, atol=0.1 * 3e-4)
    np.testing.assert_allclose([algo.ret_rms.mean, algo.ret_rms.var, algo.ret_rms.count], [rms.mean, rms.var, rms.count], rtol=1e-5)


def test_policy_forward_fused_inference_matches_torch_modules():
    """Collector-side ``policy(batch)`` (reinforce.py:167-192): under no_grad the actor output comes from the fused
    forward kernel; it must agree with the torch module forward, keep the Batch structure, and leave autograd alone."""
    from tianshou_b200.data import Batch
    g = load_golden("ppo_ref_A.npz")
    algo, actor, critic = build_ppo(17, 6, DEV, params={k: g["p0_" + k] for k in PARAM_ORDER}, **ppo_kwargs(g))
    pol = algo.policy
    assert pol._fused_inference is not None
    obs = np.random.default_rng(0).standard_normal((300, 17)).astype(np.float32)
    with torch.no_grad():
        torch.manual_seed(0)
        fused = pol(Batch(obs=obs, info=Batch()))
        pol.use_fused_inference = False
        torch.manual_seed(0)
        ref = pol(Batch(obs=obs, info=Batch()))
        pol.use_fused_inference = True
    (mu_f, sig_f), (mu_r, sig_r) = fused.logits, ref.logits
    np.testing.assert_allclose(mu_f.cpu().numpy(), mu_r.cpu().numpy(), rtol=2e-5, atol=2e-6)
    assert torch.equal(sig_f, sig_r) and fused.act.shape == ref.act.shape == (300, 6)
    np.testing.assert_allclose(fused.act.cpu().numpy(), ref.act.cpu().numpy(), rtol=1e-4, atol=1e-5)   # same torch RNG draw
    assert fused.state is None and isinstance(fused.dist, torch.distributions.Independent)
    out = pol(Batch(obs=obs, info=Batch()))              # grad enabled: the torch modules run (autograd graph intact)
    assert out.logits[0].requires_grad


def test_wide_observation_runs_simt_kernels_vs_oracle():
    """obs_dim = 40 is outside the tensor-core kernels' envelope (<= 32): value / log-prob passes and the whole update run
    the fp32 SIMT kernels (per-step ts_ppo_grad -> ts_clip_adam_step); same parity bar against the numpy oracle."""
    _simt_update_vs_oracle(40, 5)


@pytest.mark.parametrize("OBS,ACT", [(33, 1), (60, 16), (64, 4)])
def test_simt_envelope_edges_vs_oracle(OBS, ACT):
    """The same SIMT update at the edges of its envelope: 33 is the first width past the tensor-core kernels; (60, 16) and
    (64, 4) are the widest shapes whose training tile fits in the H100's 227 KB of shared memory per block."""
    _simt_update_vs_oracle(OBS, ACT)


def _simt_update_vs_oracle(OBS, ACT):
    from tianshou_b200.data import Batch, VectorReplayBuffer
    from tianshou_b200.utils import policy_within_training_step
    E, T = 24, 20
    kw = dict(gamma=0.99, gae_lambda=0.95, max_grad_norm=0.5, vf_coef=0.25, ent_coef=0.01, return_scaling=True,
              eps_clip=0.2, value_clip=True, dual_clip=None, advantage_normalization=True, recompute_advantage=True)
    algo, actor, critic = build_ppo(OBS, ACT, DEV, **kw)
    assert algo._flat.weight_image is None            # no tensor-core path for this shape
    p = {k: v.detach().cpu().numpy().copy() for k, v in named_params(actor, critic).items()}
    buf = VectorReplayBuffer(E * T, E, device=DEV)
    for s in synth_rollout(np.random.default_rng(3), E, T, OBS, ACT, p_term=0.03, trunc_len=15):
        buf.add(Batch(**s), buffer_ids=np.arange(E))
    N = E * T
    unf = np.zeros(N, dtype=bool)
    last = np.arange(E) * T + T - 1
    unf[last] = ~buf.done[last]
    roll = dict(obs=buf.obs.copy(), obs_next=buf.obs_next.copy(), act=buf.act.copy(), rew=buf.rew.copy(),
                terminated=buf.terminated.copy(), truncated=buf.truncated.copy(), unfinished=unf)
    np.random.seed(4)
    perms = np.stack([np.random.permutation(N) for _ in range(2)])
    m = {k: np.zeros_like(v) for k, v in p.items()}
    v = {k: np.zeros_like(vv) for k, vv in p.items()}
    hp = dict(eps_clip=0.2, dual_clip=None, vf_coef=0.25, ent_coef=0.01, max_grad_norm=0.5, adv_eps=1e-8, value_clip=True,
              advantage_normalization=True, lr=3e-4, beta1=0.9, beta2=0.999, adam_eps=1e-8, weight_decay=0.0)
    rms = onp.RunningMeanStd()
    res = onp.ppo_update(p, m, v, 0, roll, perms, 100, 2, hp, rms, 0.99, 0.95, True)
    np.random.seed(4)
    with policy_within_training_step(algo.policy):
        stats = algo.update(buffer=buf, batch_size=100, repeat=2)
    assert stats.gradient_steps == res["losses"].shape[0]
    for col, name in enumerate(["loss", "actor_loss", "vf_loss", "ent_loss"]):
        np.testing.assert_allclose(getattr(stats, name).mean, res["losses"][:, col].mean(), rtol=1e-3, atol=2e-5, err_msg=name)
    for k, pv in named_params(actor, critic).items():
        np.testing.assert_allclose(pv.detach().cpu().numpy(), p[k], rtol=2e-3, atol=3e-5, err_msg=k)


def test_simt_shape_past_shared_memory_is_refused():
    """obs 64 / act 16 passes the descriptor check but its SIMT training tile needs 235 KB of shared memory: the update
    must fail with a message naming the size, not an opaque launch-configuration error."""
    from tianshou_b200.data import Batch, VectorReplayBuffer
    from tianshou_b200.utils import policy_within_training_step
    algo, _, _ = build_ppo(64, 16, DEV, gamma=0.99, gae_lambda=0.95, max_grad_norm=0.5, vf_coef=0.25, ent_coef=0.0,
                           eps_clip=0.2, value_clip=False, advantage_normalization=False)
    buf = VectorReplayBuffer(4 * 8, 4, device=DEV)
    for s in synth_rollout(np.random.default_rng(0), 4, 8, 64, 16):
        buf.add(Batch(**s), buffer_ids=np.arange(4))
    with pytest.raises(RuntimeError, match="bytes of shared memory per block"):
        with policy_within_training_step(algo.policy):
            algo.update(buffer=buf, batch_size=16, repeat=1)


def test_a2c_update_matches_reference():
    """A2C through the same persistent kernel (TS_LOSS_A2C) vs the imported reference's A2C run (tests/golden/a2c_ref.npz)."""
    from tianshou_b200.algorithm import A2C, AdamOptimizerFactory, ProbabilisticActorPolicy
    from tianshou_b200.algorithm.modelfree.a2c import A2C as A2C_via_ref_path
    from tianshou_b200.utils import policy_within_training_step
    from ts_testutil import Box, build_actor_critic, gaussian_dist, load_params
    assert A2C_via_ref_path is A2C
    g = load_golden("a2c_ref.npz")
    actor, critic = build_actor_critic(17, 6, DEV)
    load_params(actor, critic, {k: g["p0_" + k] for k in PARAM_ORDER})
    policy = ProbabilisticActorPolicy(actor=actor, dist_fn=gaussian_dist, action_scaling=True, action_bound_method="clip",
                                      action_space=Box(6))
    algo = A2C(policy=policy, critic=critic, optim=AdamOptimizerFactory(lr=3e-4), gamma=float(g["kw_gamma"]),
               gae_lambda=float(g["kw_gae_lambda"]), max_grad_norm=float(g["kw_max_grad_norm"]),
               vf_coef=float(g["kw_vf_coef"]), ent_coef=float(g["kw_ent_coef"]), return_scaling=bool(g["kw_return_scaling"]))
    E, cap = int(g["cfg_E"]), int(g["cfg_cap"])
    for u in range(2):
        o = f"u{u}_"
        buf = restore_vector_buffer(g, o, E, cap, device=DEV)
        np.random.seed(1000 + u)
        with policy_within_training_step(algo.policy):
            stats = algo.update(buffer=buf, batch_size=int(g["cfg_bs"]), repeat=int(g["cfg_repeat"]))
        assert stats.gradient_steps == int(g[o + "gradient_steps"])
        ref_losses = g[o + "losses"]
        for col, name in enumerate(["loss", "actor_loss", "vf_loss", "ent_loss"]):
            np.testing.assert_allclose(getattr(stats, name).mean, ref_losses[:, col].mean(), rtol=5e-4, atol=2e-5, err_msg=name)
        for k, pv in named_params(actor, critic).items():
            np.testing.assert_allclose(pv.detach().cpu().numpy(), g[o + "p_" + k], rtol=2e-3, atol=3e-5, err_msg=f"a2c u{u} {k}")
        np.testing.assert_allclose([algo.ret_rms.mean, algo.ret_rms.var, algo.ret_rms.count], g[o + "rms"], rtol=1e-5)
