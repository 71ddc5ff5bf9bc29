"""Layer-wise actor-critic path (algorithm/layered.py: every Linear forward / backward = one wgmma GEMM launch, loss rows
in between) -- the path networks OUTSIDE the fused 17-64-64 kernels' envelope take.  Checked (a) on the reference's own
goldens by forcing the path onto shapes the fused kernels also cover (discrete shared-trunk ReLU net ppo_ref_C1*, MuJoCo
tanh net ppo_ref_A/B), and (b) on shapes only this path accepts (obs 376, MLP[256,256] -- Humanoid / BASELINE configs[3]
width; a three-layer trunk) against the numpy oracle / torch autograd."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import oracle_np as onp
from test_ppo_gpu import ppo_kwargs
from ts_testutil import PARAM_ORDER, build_ppo, load_golden, named_params, record_parity, restore_vector_buffer, synth_rollout

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture
def force_layered(monkeypatch):
    monkeypatch.setenv("TS_B200_FORCE_LAYERED", "1")


def _run_updates(algo, g, tag, params_fn, lr):
    from tianshou_b200.utils import policy_within_training_step
    E, cap = int(g["cfg_E"]), int(g["cfg_cap"])
    bs = int(g["cfg_bs"])
    bs = None if bs < 0 else bs
    captured = {}
    orig = algo._preprocess_batch

    def hook(batch, buffer, indices):
        b = orig(batch, buffer, indices)
        captured.update({k: b[k].detach().cpu().numpy().copy() for k in ("v_s", "returns", "adv", "logp_old")})
        return b

    algo._preprocess_batch = hook
    for u in range(2):
        o = f"u{u}_"
        buf = restore_vector_buffer(g, o, E, cap, device=DEV)
        np.random.seed(1000 + u)
        with policy_within_training_step(algo.policy):
            stats = algo.update(buffer=buf, batch_size=bs, repeat=int(g["cfg_repeat"]))
        for k in ("v_s", "returns", "adv", "logp_old"):
            ref = g[o + k]
            record_parity(f"{tag}_u{u}/{k}", captured[k], ref, rtol=1e-5, atol=1e-5 * max(1e-3, float(np.abs(ref).max())))
        ref_losses = g[o + "losses"]
        assert stats.gradient_steps == ref_losses.shape[0]
        for col, name in enumerate(["loss", "actor_loss", "vf_loss", "ent_loss"]):
            # (absolute floor 5e-7: a surrogate loss that averages to ~1e-3 is a mean of O(1) terms)
            record_parity(f"{tag}_u{u}/per_step_{name}", algo.last_loss_table[:, col], ref_losses[:, col], rtol=2e-4,
                          atol=5e-7 + 2e-5 * max(1e-3, float(np.abs(ref_losses[:, col]).max())))
        for k, pv in params_fn().items():
            record_parity(f"{tag}_u{u}/param_{k}", pv.detach().cpu().numpy(), g[o + "p_" + k], rtol=1e-3, atol=0.1 * lr)


@pytest.mark.parametrize("variant", ["C1", "C1b", "C1c"])
def test_layered_discrete_ppo_matches_reference(variant, force_layered):
    from test_ppo_discrete_gpu import build_discrete
    from test_ppo_discrete_gpu import named_params as discrete_params
    g = load_golden(f"ppo_ref_{variant}.npz")
    algo, actor, critic = build_discrete(g, DEV)
    assert algo._layered is not None and algo._desc is None and algo._layered.shared == bool(g["cfg_shared"])
    lr = float(g["kw_lr"]) if "kw_lr" in g.files else 3e-4
    _run_updates(algo, g, f"layered_{variant}", lambda: discrete_params(actor, critic), lr)


@pytest.mark.parametrize("variant", ["A", "B"])
def test_layered_gaussian_ppo_matches_reference(variant, force_layered):
    g = load_golden(f"ppo_ref_{variant}.npz")
    lr = float(g["kw_lr"]) if "kw_lr" in g.files else 3e-4
    algo, actor, critic = build_ppo(17, 6, DEV, lr=lr, params={k: g["p0_" + k] for k in PARAM_ORDER}, **ppo_kwargs(g))
    assert algo._layered is not None and not algo._layered.categorical
    _run_updates(algo, g, f"layered_{variant}", lambda: named_params(actor, critic), lr)


def test_wide_network_runs_the_tensor_core_gemm_path_vs_oracle():
    """obs 376 / MLP[256,256] tanh (outside every fused kernel): one update vs the numpy oracle."""
    from tianshou_b200.algorithm import PPO, AdamOptimizerFactory, ProbabilisticActorPolicy
    from tianshou_b200.data import Batch, VectorReplayBuffer
    from tianshou_b200.utils import policy_within_training_step
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.continuous import ContinuousActorProbabilistic, ContinuousCritic
    from ts_testutil import Box, gaussian_dist
    O, A, H = 376, 17, (256, 256)
    torch.manual_seed(0)
    actor = ContinuousActorProbabilistic(preprocess_net=Net(state_shape=(O,), hidden_sizes=H, activation=torch.nn.Tanh),
                                         action_shape=(A,), unbounded=True).to(DEV)
    critic = ContinuousCritic(preprocess_net=Net(state_shape=(O,), hidden_sizes=H, activation=torch.nn.Tanh)).to(DEV)
    torch.nn.init.constant_(actor.sigma_param, -0.5)
    policy = ProbabilisticActorPolicy(actor=actor, dist_fn=gaussian_dist, action_scaling=True, action_bound_method="clip",
                                      action_space=Box(A))
    kw = dict(gamma=0.99, gae_lambda=0.95, max_grad_norm=0.5, vf_coef=0.25, ent_coef=0.01, return_scaling=True, eps_clip=0.2,
              value_clip=True, dual_clip=None, advantage_normalization=True, recompute_advantage=True)
    algo = PPO(policy=policy, critic=critic, optim=AdamOptimizerFactory(lr=3e-4), **kw)
    assert algo._layered is not None
    p = {k: v.detach().cpu().numpy().copy() for k, v in named_params(actor, critic).items()}
    E, T = 16, 48
    buf = VectorReplayBuffer(E * T, E, device=DEV)
    for s in synth_rollout(np.random.default_rng(2), E, T, O, A, p_term=0.03, trunc_len=30):
        buf.add(Batch(**s), buffer_ids=np.arange(E))
    N = E * T
    last = np.arange(E) * T + T - 1
    unf = np.zeros(N, dtype=bool)
    unf[last] = ~buf.done[last]
    roll = dict(obs=buf.obs.copy(), obs_next=buf.obs_next.copy(), act=buf.act.copy(), rew=buf.rew.copy(),
                terminated=buf.terminated.copy(), truncated=buf.truncated.copy(), unfinished=unf)
    np.random.seed(9)
    perms = np.stack([np.random.permutation(N) for _ in range(2)])
    m = {k: np.zeros_like(v) for k, v in p.items()}
    v = {k: np.zeros_like(vv) for k, vv in p.items()}
    hp = dict(eps_clip=0.2, dual_clip=None, vf_coef=0.25, ent_coef=0.01, max_grad_norm=0.5, adv_eps=1e-8, value_clip=True,
              advantage_normalization=True, lr=3e-4, beta1=0.9, beta2=0.999, adam_eps=1e-8, weight_decay=0.0)
    rms = onp.RunningMeanStd()
    res = onp.ppo_update(p, m, v, 0, roll, perms, 256, 2, hp, rms, 0.99, 0.95, True)
    np.random.seed(9)
    with policy_within_training_step(algo.policy):
        stats = algo.update(buffer=buf, batch_size=256, repeat=2)
    assert stats.gradient_steps == res["losses"].shape[0]
    for col, name in enumerate(["loss", "actor_loss", "vf_loss", "ent_loss"]):
        ref = res["losses"][:, col]
        record_parity(f"layered_wide/per_step_{name}", algo.last_loss_table[:, col], ref, rtol=2e-4, atol=2e-5 * max(1e-3, float(np.abs(ref).max())))
    for k, pv in named_params(actor, critic).items():
        record_parity(f"layered_wide/param_{k}", pv.detach().cpu().numpy(), p[k], rtol=1e-3, atol=0.1 * 3e-4)


def test_three_layer_relu_trunk_gradients_vs_autograd():
    """A deeper trunk (three hidden layers, different widths) per network."""
    _trunk_gradients_vs_fp64_autograd("three-layer")


def test_two_net_wrappers_around_one_trunk_gradients_vs_autograd():
    """Actor and critic hold two different ``Net`` wrappers around ONE (128, 128) MLP: the trunk is shared, and its gradient
    is the sum of both losses' gradients (not the critic's alone)."""
    _trunk_gradients_vs_fp64_autograd("two-wrappers")


def _trunk_gradients_vs_fp64_autograd(trunk):
    """Gradients of one layered minibatch step vs float64 torch autograd of the same PPO loss on copies of the same modules."""
    import copy

    from tianshou_b200.algorithm import PPO, AdamOptimizerFactory, ProbabilisticActorPolicy
    from tianshou_b200.utils.net.common import ActorCritic, Net
    from tianshou_b200.utils.net.continuous import ContinuousActorProbabilistic, ContinuousCritic
    from ts_testutil import Box, gaussian_dist
    O, A, H = (29, 4, (96, 80, 40)) if trunk == "three-layer" else (17, 6, (128, 128))
    torch.manual_seed(1)
    a_net = Net(state_shape=(O,), hidden_sizes=H)
    c_net = Net(state_shape=(O,), hidden_sizes=H)
    if trunk == "two-wrappers":
        c_net.model = a_net.model
    actor = ContinuousActorProbabilistic(preprocess_net=a_net, action_shape=(A,), unbounded=True).to(DEV)
    critic = ContinuousCritic(preprocess_net=c_net).to(DEV)
    policy = ProbabilisticActorPolicy(actor=actor, dist_fn=gaussian_dist, action_scaling=True, action_bound_method="clip",
                                      action_space=Box(A))
    algo = PPO(policy=policy, critic=critic, optim=AdamOptimizerFactory(lr=0.0), eps_clip=0.2, vf_coef=0.5, ent_coef=0.02,
               value_clip=False, advantage_normalization=False, max_grad_norm=None)
    L = algo._layered
    assert L is not None and len(L.a_trunk.layers) == len(H) and L.shared == (trunk == "two-wrappers")
    B = 200
    g = torch.Generator().manual_seed(0)
    obs = torch.randn(B, O, generator=g).to(DEV)
    act = torch.randn(B, A, generator=g).to(DEV)
    adv, ret, vso = (torch.randn(B, generator=g).to(DEV) for _ in range(3))
    with torch.no_grad():
        (mu, sig), _ = actor(obs)
        lpo = gaussian_dist((mu, sig)).log_prob(act) + 0.2 * torch.randn(B, generator=g).to(DEV)

    class _B:
        pass

    batch = _B()
    batch.obs, batch.act, batch.adv, batch.returns, batch.logp_old, batch.v_s = obs, act, adv, ret, lpo.contiguous(), vso
    stats_row = torch.zeros(8, device=DEV)
    L.minibatch_step(batch, torch.arange(B, device=DEV), algo._loss_hparams(), None, algo.optim._optim, None, stats_row)
    # float64 autograd of ppo.py:183-211 on copies of the modules (lr = 0: the step did not move the parameters), through
    # their Sequentials: MLP.forward casts its input to float32
    actor64, critic64 = copy.deepcopy((actor, critic))
    actor64.double()
    critic64.double()
    obs, act, adv, ret, lpo = (t.double() for t in (obs, act, adv, ret, lpo))
    mu = actor64.mu.model(actor64.preprocess.model.model(obs))
    dist = gaussian_dist((mu, (actor64.sigma_param.view(1, -1) + torch.zeros_like(mu)).exp()))
    ratio = (dist.log_prob(act) - lpo).exp()
    surr = torch.min(ratio * adv, ratio.clamp(0.8, 1.2) * adv)
    value = critic64.last.model(critic64.preprocess.model.model(obs)).flatten()
    loss = -surr.mean() + 0.5 * (ret - value).pow(2).mean() - 0.02 * dist.entropy().mean()
    loss.backward()
    tag = f"layered_{trunk}"
    record_parity(f"{tag}/loss", stats_row[:1].cpu().numpy(), np.array([float(loss)]), rtol=2e-5, atol=1e-6)
    params64 = list(ActorCritic(actor64, critic64).parameters())      # the group's order: ActorCritic order, shared once
    for i, (p_, p64) in enumerate(zip(L.group.params, params64, strict=True)):
        got = L.group.view(L.group.grad, p_).view(p_.shape).cpu().numpy()
        ref = p64.grad.cpu().numpy()
        record_parity(f"{tag}/grad{i}", got, ref, rtol=2e-4, atol=2e-5 * float(np.abs(ref).max()) + 1e-9)


# ------------------------------------------------------------------------------------------- ts_ppo_rows per row
ROWS_HP = {
    "vclip_advnorm_ent": dict(loss_kind="ppo", eps_clip=0.2, dual_clip=0.0, value_clip=1, adv_norm=1, vf_coef=0.5, ent_coef=0.01),
    "dual_clip": dict(loss_kind="ppo", eps_clip=0.2, dual_clip=2.0, value_clip=0, adv_norm=0, vf_coef=0.25, ent_coef=0.003),
    "a2c": dict(loss_kind="a2c", eps_clip=0.2, dual_clip=0.0, value_clip=0, adv_norm=0, vf_coef=0.5, ent_coef=0.01),
}
F32_EPS = float(np.finfo(np.float32).eps)


def _rows_reference(z, value, logstd, act, adv, ret, lpo, vs, mom, hp, categorical, dtype):
    """Per-row PPO / A2C loss (ppo.py:179-211, a2c.py:262-270) with torch autograd in ``dtype`` on the CPU.  Categorical
    head: Categorical(probs=softmax(z)) written out as torch.distributions does it (renormalise, clamp to [eps, 1 - eps]
    with the FLOAT32 eps of the reference's dtype, log), so a float64 run keeps the reference's clamp.  Gaussian head:
    Normal(mu, exp(logstd)), the log-std broadcast to one leaf per row so its gradient comes back per row."""
    T = lambda a: torch.as_tensor(np.asarray(a)).to(dtype)
    z = T(z).requires_grad_(True)
    v = T(value).requires_grad_(True)
    B, A = z.shape
    ls_rows = None
    if categorical:
        p = torch.softmax(z, dim=-1)
        pn = p / p.sum(-1, keepdim=True)
        lg = torch.log(pn.clamp(F32_EPS, 1 - F32_EPS))
        logp = lg.gather(1, torch.as_tensor(np.asarray(act)).long().view(-1, 1)).view(-1)
        ent = -(pn * lg).sum(-1)
    else:
        ls_rows = T(logstd).reshape(1, A).expand(B, A).clone().requires_grad_(True)
        dist = torch.distributions.Normal(z, ls_rows.exp())
        logp = dist.log_prob(T(act)).sum(-1)
        ent = dist.entropy().sum(-1)
    Adv = T(adv)
    if hp["loss_kind"] == "a2c":
        obj = logp * Adv
    else:
        if hp["adv_norm"]:
            Adv = (Adv - float(mom[0])) / (float(mom[1]) + 1e-8)
        ratio = (logp - T(lpo)).exp()
        e = hp["eps_clip"]
        obj = torch.min(ratio * Adv, ratio.clamp(1 - e, 1 + e) * Adv)
        if hp["dual_clip"]:
            obj = torch.where(Adv < 0, torch.max(obj, hp["dual_clip"] * Adv), obj)
    R, vso = T(ret), T(vs)
    if hp["value_clip"]:
        v_clip = vso + (v - vso).clamp(-hp["eps_clip"], hp["eps_clip"])
        vf = torch.max((R - v).pow(2), (R - v_clip).pow(2))
    else:
        vf = (R - v).pow(2)
    loss = -obj.mean() + hp["vf_coef"] * vf.mean() - hp["ent_coef"] * ent.mean()
    loss.backward()
    d = lambda t: t.detach().numpy().astype(np.float64)
    return dict(logp=d(logp), dhead=d(z.grad), dvalue=d(v.grad), dlogstd=None if ls_rows is None else d(ls_rows.grad),
                rows=np.stack([d(obj), d(vf), d(ent)], 1))


def _rows_inputs(rng, B, A, categorical, hp):
    """Head rows around a random policy.  Categorical: every fourth row is saturated -- one logit 30 above the rest, so
    every other probability is ~1e-13, far below the clamp -- and the action taken there is a clamped one in half of
    those rows; the other rows are redrawn until no probability lies within 4x of eps or 1 - eps.  Branch guard as in
    test_tc_shapes_gpu: no ratio within 1e-4 of a clip boundary, no value delta within 1e-4 of +-eps_clip, no two clipped
    value errors within 1e-4 of each other, so fp32 and fp64 take the same side of every min / max / clamp."""
    if categorical:
        z = rng.standard_normal((B, A)) * 2.0
        act = rng.integers(0, A, B)
        sat = np.arange(B) % 4 == 0
        for b in np.nonzero(sat)[0]:
            top = rng.integers(0, A)
            z[b, top] = z[b].max() + 30.0
            if A > 1 and b % 8 == 0:
                act[b] = (top + 1 + rng.integers(0, A - 1)) % A           # a clamped action
        for _ in range(100):
            p = np.exp(z - z.max(1, keepdims=True))
            p /= p.sum(1, keepdims=True)
            near = ((p > F32_EPS / 4) & (p < 4 * F32_EPS)) | ((1 - p > F32_EPS / 4) & (1 - p < 4 * F32_EPS))
            bad = near.any(1) & ~sat
            if not bad.any():
                break
            z[bad] = rng.standard_normal((int(bad.sum()), A)) * 2.0
        act_arr = act.astype(np.float32)
        logstd = None
    else:
        z = rng.standard_normal((B, A))
        logstd = np.linspace(-1.2, 0.3, A).astype(np.float32)
        act_arr = (z + np.exp(logstd) * rng.standard_normal((B, A))).astype(np.float32)
    z = z.astype(np.float32)
    value = rng.standard_normal(B).astype(np.float32)
    adv = rng.standard_normal(B).astype(np.float32)
    ret = rng.standard_normal(B).astype(np.float32)
    mom = np.array([adv.astype(np.float64).mean(), adv.astype(np.float64).std(ddof=1)], np.float32)
    zero = np.zeros(B)
    lp = _rows_reference(z, value, logstd, act_arr, adv, ret, zero, zero, mom, dict(hp, loss_kind="a2c"), categorical,
                         torch.float64)["logp"]
    lpo = (lp + 0.5 * rng.standard_normal(B)).astype(np.float32)
    vs = (value + 0.3 * rng.standard_normal(B)).astype(np.float32)
    e, dual = hp["eps_clip"], hp["dual_clip"]
    Adv = (adv - mom[0]) / (mom[1] + 1e-8) if hp["adv_norm"] else adv.astype(np.float64)
    for _ in range(100):
        ratio = np.exp(lp - lpo.astype(np.float64))
        bad = (np.abs(ratio - (1 - e)) < 1e-4) | (np.abs(ratio - (1 + e)) < 1e-4)
        if dual:
            bad |= np.abs(np.minimum(ratio * Adv, np.clip(ratio, 1 - e, 1 + e) * Adv) - dual * Adv) < 1e-4
        if not bad.any():
            break
        lpo[bad] = (lp[bad] + 0.5 * rng.standard_normal(int(bad.sum()))).astype(np.float32)
    for _ in range(100):
        dl = value.astype(np.float64) - vs
        vc = vs + np.clip(dl, -e, e)
        bad = (np.abs(np.abs(dl) - e) < 1e-4) | (np.abs((ret - value.astype(np.float64)) ** 2 - (ret - vc) ** 2) < 1e-4)
        if not bad.any():
            break
        vs[bad] = (value[bad] + 0.3 * rng.standard_normal(int(bad.sum()))).astype(np.float32)
    return z, value, logstd, act_arr, adv, ret, lpo, vs, mom


ROWS_CASES = [(True, A, h) for A in (2, 7, 18, 64) for h in ROWS_HP] + [(False, A, h) for A in (1, 6, 17) for h in ROWS_HP]


@pytest.mark.parametrize("categorical,A,hp_name", ROWS_CASES,
                         ids=[f"{'cat' if c else 'gauss'}-A{a}-{h}" for c, a, h in ROWS_CASES])
def test_ppo_rows_vs_fp64_autograd(categorical, A, hp_name):
    """ts_ppo_rows (the loss between the layer-wise forward and backward GEMMs): logp, per-row (objective, value loss,
    entropy), dhead, dvalue and the per-row log-std gradient against float64 autograd of the reference loss on the same
    head outputs.  Bound: 8x torch fp32's own error against float64 (the same autograd in float32) plus a floor of 1e-5
    of the largest value -- the kernel's operation order differs from torch's, and the softmax backward divides by
    probabilities down to eps."""
    from tianshou_b200._cabi import LOSS_A2C, LOSS_PPO, PPOHParams
    hp = ROWS_HP[hp_name]
    B = 1031
    rng = np.random.default_rng(A * 13 + len(hp_name) + int(categorical))
    z, value, logstd, act, adv, ret, lpo, vs, mom = _rows_inputs(rng, B, A, categorical, hp)
    h = PPOHParams(eps_clip=hp["eps_clip"], dual_clip=hp["dual_clip"], vf_coef=hp["vf_coef"], ent_coef=hp["ent_coef"],
                   max_grad_norm=0.0, adv_eps=1e-8, lr=0.0, beta1=0.9, beta2=0.999, adam_eps=1e-8, weight_decay=0.0,
                   value_clip=hp["value_clip"], advantage_normalization=hp["adv_norm"],
                   loss_kind=LOSS_A2C if hp["loss_kind"] == "a2c" else LOSS_PPO)
    live = []      # keeps every uploaded input alive until the kernel has run (the call below only sees raw pointers)
    D = lambda a: live.append(torch.as_tensor(np.ascontiguousarray(a)).to(DEV)) or live[-1]
    nan = lambda *s: torch.full(s, float("nan"), dtype=torch.float32, device=DEV)
    logp, dhead, dval, rows = nan(B), nan(B, A), nan(B), nan(B, 3)
    dls = None if categorical else nan(B, A)
    from tianshou_b200._cabi import call, ptr, stream_ptr
    call("ts_ppo_rows", ptr(D(z)), ptr(D(value)), None if categorical else ptr(D(logstd)), ptr(D(act)), ptr(D(adv)), ptr(D(ret)),
         ptr(D(lpo)), ptr(D(vs)), B, A, int(categorical), C.byref(h), B, ptr(D(mom)) if hp["adv_norm"] else None, ptr(logp),
         ptr(dhead), ptr(dval), ptr(dls), ptr(rows), stream_ptr(torch.device(DEV)))
    torch.cuda.synchronize()
    live.clear()
    args = (z, value, logstd, act, adv, ret, lpo, vs, mom, hp, categorical)
    r64 = _rows_reference(*args, torch.float64)
    r32 = _rows_reference(*args, torch.float32)
    got = dict(logp=logp, dhead=dhead, dvalue=dval, rows=rows, dlogstd=dls)
    tag = f"ppo_rows/{'cat' if categorical else 'gauss'}_A{A}_{hp_name}"
    for k in ("logp", "rows", "dhead", "dvalue", "dlogstd"):
        if r64[k] is None:
            continue
        ref = r64[k]
        scale = float(np.abs(ref).max())
        record_parity(f"{tag}/{k}", got[k].cpu().numpy(), ref, rtol=0.0,
                      atol=8.0 * float(np.abs(r32[k] - ref).max()) + 1e-5 * scale)


def test_ppo_rows_refuses_more_than_64_actions():
    """A = 65 is refused on the host with the library's error code and message; nothing is launched."""
    from tianshou_b200._cabi import LOSS_PPO, PPOHParams, load_library, ptr, stream_ptr
    lib = load_library()
    B, A = 4, 65
    z = torch.zeros(B, A, device=DEV)
    act = torch.zeros(B, device=DEV)
    out = torch.zeros(B, device=DEV)
    h = PPOHParams(eps_clip=0.2, loss_kind=LOSS_PPO)
    st = lib.ts_ppo_rows(ptr(z), None, None, ptr(act), None, None, None, None, B, A, 1, C.byref(h), B, None, ptr(out), None, None, None,
                         None, stream_ptr(torch.device(DEV)))
    assert st != 0
    assert "act_dim <= 64" in lib.ts_last_error().decode()
