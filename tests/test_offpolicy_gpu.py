"""Off-policy update bodies on the GPU (SURVEY 8(f) ranks 2-3) vs outputs of the imported reference
(tests/golden/sac_ref.npz, dqn_ref*.npz from oracle/gen_golden_offpolicy.py: same initial weights, same buffer contents,
same numpy / torch seeds): sampled indices bit-exact, n-step returns, losses, TD errors, post-update parameters of the
online and lagged networks."""
import numpy as np
import pytest
import torch

from offpolicy_testutil import DEV, Box, Discrete, check_params, load_params
from ts_testutil import load_golden, record_parity, set_buffer_state

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------------------ SAC
def _build_sac(g, **kw):
    from tianshou_b200.algorithm import AdamOptimizerFactory
    from tianshou_b200.algorithm.modelfree.sac import SAC, SACPolicy
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.continuous import ContinuousActorProbabilistic, ContinuousCritic
    O, A, H = int(g["cfg_obs"]), int(g["cfg_act"]), tuple(int(x) for x in g["cfg_hidden"])
    lr = float(g["cfg_lr"])
    actor = ContinuousActorProbabilistic(preprocess_net=Net(state_shape=(O,), hidden_sizes=H), action_shape=(A,), unbounded=True,
                                         conditioned_sigma=True).to(DEV)
    c1 = ContinuousCritic(preprocess_net=Net(state_shape=(O,), action_shape=(A,), hidden_sizes=H, concat=True)).to(DEV)
    c2 = ContinuousCritic(preprocess_net=Net(state_shape=(O,), action_shape=(A,), hidden_sizes=H, concat=True)).to(DEV)
    load_params(actor, g, "p0_actor_"); load_params(c1, g, "p0_c1_"); load_params(c2, g, "p0_c2_")
    policy = SACPolicy(actor=actor, action_space=Box(A))
    algo = SAC(policy=policy, policy_optim=AdamOptimizerFactory(lr=lr), critic=c1, critic_optim=AdamOptimizerFactory(lr=lr),
               critic2=c2, critic2_optim=AdamOptimizerFactory(lr=lr), tau=float(g["cfg_tau"]), gamma=float(g["cfg_gamma"]),
               alpha=float(g["cfg_alpha"]), n_step_return_horizon=int(g["cfg_n_step"]), **kw)
    return algo, actor, c1, c2, lr


@pytest.mark.parametrize("mirror", [False, True])
def test_sac_update_matches_reference(mirror):
    from tianshou_b200.data import Batch, VectorReplayBuffer
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden("sac_ref.npz")
    algo, actor, c1, c2, lr = _build_sac(g)
    E, cap = int(g["cfg_E"]), int(g["cfg_cap"])
    buf = VectorReplayBuffer(E * cap, E, device=DEV, device_mirror=mirror)
    buf.set_batch(Batch(**{k: g["buf_" + k].copy() for k in ("obs", "act", "rew", "terminated", "truncated", "done", "obs_next")}))
    set_buffer_state(buf, g["meta_last_index"], g["meta_lengths"])
    if mirror:
        buf.sync_device_mirror()
        assert buf.device_columns() is not None
    # the reference drew its rsample noise from torch's CPU generator (it ran on the CPU): same draws, uploaded
    algo._noise_fn = lambda shape: torch.normal(torch.zeros(shape), torch.ones(shape)).to(DEV)
    captured = {}
    orig = algo._preprocess_batch

    def hook(batch, buffer, indices):
        b = orig(batch, buffer, indices)
        captured["indices"], captured["returns"] = np.asarray(indices).copy(), b.returns.detach().cpu().numpy().copy()
        return b

    algo._preprocess_batch = hook
    for u in range(int(g["cfg_updates"])):
        torch.manual_seed(100 + u)
        with policy_within_training_step(algo.policy):
            stats = algo.update(buffer=buf, sample_size=int(g["cfg_bs"]))
        o, tag = f"u{u}_", f"sac_m{int(mirror)}_u{u}"
        assert np.array_equal(captured["indices"], g[o + "indices"]), "sampled indices differ from the reference's"
        ref_ret = g[o + "returns"]
        record_parity(f"{tag}/returns", captured["returns"].reshape(ref_ret.shape), ref_ret, rtol=1e-5, atol=1e-5 * float(np.abs(ref_ret).max()))
        got = np.array([stats.actor_loss, stats.critic1_loss, stats.critic2_loss])
        record_parity(f"{tag}/losses", got, g[o + "losses"], rtol=2e-5, atol=2e-6)
        check_params(tag, actor, g, o + "actor_", lr); check_params(tag, c1, g, o + "c1_", lr); check_params(tag, c2, g, o + "c2_", lr)
        check_params(tag, algo.critic_old, g, o + "c1old_", lr); check_params(tag, algo.critic2_old, g, o + "c2old_", lr)
        assert stats.alpha == pytest.approx(float(g["cfg_alpha"])) and stats.alpha_loss is None and stats.train_time > 0


def test_sac_cuda_graph_matches_reference():
    """``SAC(cuda_graph=True)``: update 0 runs eagerly, update 1 is captured and replayed, later updates are replays of the same
    graph — every one of them must still match the reference's update on the same indices / noise."""
    from tianshou_b200.data import Batch, VectorReplayBuffer
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden("sac_ref.npz")
    algo, actor, c1, c2, lr = _build_sac(g, cuda_graph=True)
    E, cap = int(g["cfg_E"]), int(g["cfg_cap"])
    buf = VectorReplayBuffer(E * cap, E, device=DEV, device_mirror=True)
    buf.set_batch(Batch(**{k: g["buf_" + k].copy() for k in ("obs", "act", "rew", "terminated", "truncated", "done", "obs_next")}))
    set_buffer_state(buf, g["meta_last_index"], g["meta_lengths"])
    buf.sync_device_mirror()
    algo._noise_fn = lambda shape: torch.normal(torch.zeros(shape), torch.ones(shape)).to(DEV)
    n_up = int(g["cfg_updates"])
    assert n_up >= 3, "need an eager, a capture and a pure-replay update"
    for u in range(n_up):
        torch.manual_seed(100 + u)
        with policy_within_training_step(algo.policy):
            stats = algo.update(buffer=buf, sample_size=int(g["cfg_bs"]))
        o, tag = f"u{u}_", f"sac_graph_u{u}"
        assert np.array_equal(algo._graph["h_idx"].numpy(), g[o + "indices"]), "sampled indices differ from the reference's"
        got = np.array([stats.actor_loss, stats.critic1_loss, stats.critic2_loss])
        record_parity(f"{tag}/losses", got, g[o + "losses"], rtol=2e-5, atol=2e-6)
        check_params(tag, actor, g, o + "actor_", lr); check_params(tag, c1, g, o + "c1_", lr); check_params(tag, c2, g, o + "c2_", lr)
        check_params(tag, algo.critic_old, g, o + "c1old_", lr); check_params(tag, algo.critic2_old, g, o + "c2old_", lr)
    assert algo._graph["graph"] is not None and algo._graph["calls"] == n_up
    for grp in algo._g_c:
        grp.sync_step_from_device()
        assert grp.step == n_up


def test_sac_policy_forward_collector_path():
    """``policy(batch)`` (the Collector's call, sac.py:108-131) keeps the Batch structure on the torch modules."""
    from tianshou_b200.data import Batch
    g = load_golden("sac_ref.npz")
    algo, actor, *_ = _build_sac(g)
    obs = np.random.default_rng(0).standard_normal((7, int(g["cfg_obs"]))).astype(np.float32)
    out = algo.policy(Batch(obs=obs, info=Batch()))
    assert out.act.shape == (7, int(g["cfg_act"])) and out.log_prob.shape == (7, 1) and float(out.act.abs().max()) <= 1.0
    assert algo.policy.map_action(out.act.detach().cpu().numpy()).shape == (7, int(g["cfg_act"]))


def test_sac_refuses_networks_off_one_cuda_device():
    """A critic outside the actor's CUDA device is refused, not silently moved there."""
    from tianshou_b200.algorithm import AdamOptimizerFactory, UnsupportedModelError
    from tianshou_b200.algorithm.modelfree.sac import SAC, SACPolicy
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.continuous import ContinuousActorProbabilistic, ContinuousCritic
    O, A = 4, 2
    actor = ContinuousActorProbabilistic(preprocess_net=Net(state_shape=(O,), hidden_sizes=(8,)), action_shape=(A,), unbounded=True,
                                         conditioned_sigma=True).to(DEV)
    critic = ContinuousCritic(preprocess_net=Net(state_shape=(O,), action_shape=(A,), hidden_sizes=(8,), concat=True))
    with pytest.raises(UnsupportedModelError, match="no CPU path"):
        SAC(policy=SACPolicy(actor=actor, action_space=Box(A)), policy_optim=AdamOptimizerFactory(lr=1e-3), critic=critic,
            critic_optim=AdamOptimizerFactory(lr=1e-3))
    assert next(critic.parameters()).device.type == "cpu"


# ------------------------------------------------------------------------------------------------------------ DQN
def _build_dqn(g):
    from tianshou_b200.algorithm import AdamOptimizerFactory
    from tianshou_b200.algorithm.modelfree.dqn import DQN, DiscreteQLearningPolicy
    from tianshou_b200.env.atari import DQNet, ScaledObsInputActionReprNet
    H, W, A = int(g["cfg_H"]), int(g["cfg_W"]), int(g["cfg_A"])
    lr = float(g["cfg_lr"])
    net = ScaledObsInputActionReprNet(DQNet(4, H, W, A)).to(DEV)
    load_params(net, g, "p0_q_")
    policy = DiscreteQLearningPolicy(model=net, action_space=Discrete(A))
    huber = float(g["cfg_huber"])
    algo = DQN(policy=policy, optim=AdamOptimizerFactory(lr=lr), gamma=float(g["cfg_gamma"]), n_step_return_horizon=int(g["cfg_n_step"]),
               target_update_freq=int(g["cfg_target_freq"]), is_double=bool(g["cfg_is_double"]),
               huber_loss_delta=None if np.isnan(huber) else huber)
    return algo, net, lr


@pytest.mark.parametrize("variant,mirror", [("", True), ("", False), ("_b", True)])
def test_dqn_update_matches_reference(variant, mirror):
    """NatureCNN DQN on uint8 single-frame storage (stack_num 4, save_only_last_obs, ignore_obs_next) with prioritised
    replay: the frame stacks are gathered by the first convolution's im2col from the device copy of the frames."""
    from tianshou_b200.data import Batch, PrioritizedVectorReplayBuffer
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden(f"dqn_ref{variant}.npz")
    algo, net, lr = _build_dqn(g)
    E, cap, steps = int(g["cfg_E"]), int(g["cfg_cap"]), int(g["cfg_steps"])
    buf = PrioritizedVectorReplayBuffer(E * cap, E, alpha=float(g["cfg_alpha"]), beta=float(g["cfg_beta"]), stack_num=4,
                                        ignore_obs_next=True, save_only_last_obs=True, device=DEV, device_mirror=mirror)
    for i in range(steps):
        last = g[f"roll{i}_obs"]
        stack = np.repeat(last[:, None], 4, axis=1)            # only the last frame is stored (save_only_last_obs)
        buf.add(Batch(obs=stack, act=g[f"roll{i}_act"], rew=g[f"roll{i}_rew"], terminated=g[f"roll{i}_terminated"],
                      truncated=g[f"roll{i}_truncated"], obs_next=stack), buffer_ids=np.arange(E))
    assert buf.obs.dtype == np.uint8 and buf.obs.shape[1:] == (int(g["cfg_H"]), int(g["cfg_W"]))
    if mirror:
        assert buf.device_columns() is not None and buf.device_columns()["obs"].dtype == torch.uint8
    captured = {}
    orig_pre, orig_post = algo._preprocess_batch, algo._postprocess_batch

    def pre(batch, buffer, indices):
        captured["is_weight"] = batch.weight.detach().cpu().numpy().copy()
        b = orig_pre(batch, buffer, indices)
        captured["indices"], captured["returns"] = np.asarray(indices).copy(), b.returns.detach().cpu().numpy().copy()
        return b

    def post(batch, buffer, indices):
        captured["td"] = batch.weight.detach().cpu().numpy().copy()
        return orig_post(batch, buffer, indices)

    algo._preprocess_batch, algo._postprocess_batch = pre, post
    n_up = int(g["cfg_updates"])
    for u in range(n_up):
        np.random.seed(500 + u)
        with policy_within_training_step(algo.policy):
            stats = algo.update(buffer=buf, sample_size=int(g["cfg_bs"]))
        o, tag = f"u{u}_", f"dqn{variant}_m{int(mirror)}_u{u}"
        assert np.array_equal(captured["indices"], g[o + "indices"]), f"update {u}: sampled indices differ from the reference's"
        record_parity(f"{tag}/is_weight", captured["is_weight"], g[o + "is_weight"], rtol=1e-4, atol=1e-6)
        ref_ret = g[o + "returns"]
        record_parity(f"{tag}/returns", captured["returns"].reshape(ref_ret.shape), ref_ret, rtol=1e-5, atol=1e-5 * float(np.abs(ref_ret).max()))
        record_parity(f"{tag}/td", captured["td"], g[o + "td"], rtol=1e-5, atol=2e-5 * float(np.abs(g[o + "td"]).max()))
        record_parity(f"{tag}/loss", np.array([stats.loss]), np.array([float(g[o + "loss"])]), rtol=2e-5, atol=1e-6)
        record_parity(f"{tag}/tree_leaves", np.asarray(buf.weight[np.arange(len(buf))]), g[o + "tree_leaves"], rtol=1e-4, atol=1e-7)
    o = f"u{n_up - 1}_"
    check_params(f"dqn{variant}_m{int(mirror)}", net, g, o + "q_", lr)
    if algo.model_old is not None:
        check_params(f"dqn{variant}_m{int(mirror)}", algo.model_old, g, o + "qold_", lr)


def test_dqn_policy_forward_and_eps_greedy():
    from tianshou_b200.data import Batch
    g = load_golden("dqn_ref_b.npz")
    algo, net, _ = _build_dqn(g)
    obs = np.random.default_rng(0).integers(0, 256, (5, 4, int(g["cfg_H"]), int(g["cfg_W"])), dtype=np.uint8)
    out = algo.policy(Batch(obs=obs, info=Batch()))
    assert out.logits.shape == (5, int(g["cfg_A"])) and out.act.shape == (5,)
    algo.policy.set_eps_inference(1.0)
    np.random.seed(0)
    act = algo.policy.add_exploration_noise(out.act.copy(), Batch(obs=obs))
    assert act.shape == (5,) and act.min() >= 0 and act.max() < int(g["cfg_A"])


# ------------------------------------------------------------------------ gradients of the update bodies vs autograd
class _GivenTanh(torch.autograd.Function):
    """Returns the kernel's own fp32 tanh output (as float64) with torch's tanh backward, grad * (1 - y^2), on it.  Near
    |y| = 1 the gradient is ill-conditioned in the last bit of y (fp32 y = 1 gives 0, float64 at x = 9.5 still 0.31), so
    the reference differentiates at the action the update actually used; the forward kernel's tanh is checked against
    float64 in test_offpolicy_kernels_gpu."""

    @staticmethod
    def forward(ctx, x, y):
        ctx.save_for_backward(y)
        return y.clone()

    @staticmethod
    def backward(ctx, g):
        (y,) = ctx.saved_tensors
        return g * (1.0 - y * y), None


def _copy64(mod, group, flat):
    """Deep copy of ``mod`` on the CPU in float64 with its parameters read from ``flat`` (a snapshot of ``group.flat``)."""
    import copy
    c = copy.deepcopy(mod).to("cpu", torch.float64)
    with torch.no_grad():
        for (_, p), (_, q) in zip(mod.named_parameters(), c.named_parameters(), strict=True):
            q.copy_(group.view(flat, p).view(p.shape).to(torch.float64))
    return c


def _check_grads(tag, mod, group, grad, ref_mod, rows=0):
    """Every parameter's gradient read through ``group.view``.  The GEMMs are fp32-faithful (bf16x3), the weight
    gradients sum B products per element: 2e-4 relative plus 1e-4 of the tensor's largest value (the three-product
    weight-gradient bound of test_tc_shapes_gpu), or the documented sum-length term of ``rows`` rows where that is larger."""
    from ts_testutil import sum_length_rel
    rel = max(1e-4, sum_length_rel(rows))
    for (name, p), (_, q) in zip(mod.named_parameters(), ref_mod.named_parameters(), strict=True):
        ref = q.grad.numpy()
        got = group.view(grad, p).view(p.shape).cpu().numpy()
        record_parity(f"{tag}/grad_{name}", got, ref, rtol=2e-4, atol=rel * float(np.abs(ref).max()) + 1e-12)


def sac_grad_case(O, A, H, separate_critic2, per, auto_alpha, seed, B=256, edge=""):
    """One SAC update at batch ``B`` checked against float64 autograd; returns the captured batch and the update's stats."""
    from tianshou_b200.algorithm import AdamOptimizerFactory
    from tianshou_b200.algorithm.modelfree.sac import SAC, AutoAlpha, SACPolicy
    from tianshou_b200.algorithm.flat_params import FlatGroup
    from tianshou_b200.data import Batch, PrioritizedVectorReplayBuffer, VectorReplayBuffer
    from tianshou_b200.utils import policy_within_training_step
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.continuous import ContinuousActorProbabilistic, ContinuousCritic
    from ts_testutil import synth_rollout
    torch.manual_seed(seed)
    actor = ContinuousActorProbabilistic(preprocess_net=Net(state_shape=(O,), hidden_sizes=H), action_shape=(A,), unbounded=True,
                                         conditioned_sigma=True).to(DEV)
    mk = lambda: ContinuousCritic(preprocess_net=Net(state_shape=(O,), action_shape=(A,), hidden_sizes=H, concat=True)).to(DEV)
    c1 = mk()
    c2 = mk() if separate_critic2 else None
    # head biases: log-sigma below / above the clamp range, mu saturating tanh.  With AutoAlpha no log-sigma sits at the
    # lower bound: at sigma = e^-20, fp32 mu + sigma * noise rounds to mu and the row's log-prob loses -noise^2 / 2 in
    # every fp32 evaluation, so only rows without it can have their log-prob (which drives alpha) checked against float64
    low_sigma = not auto_alpha
    with torch.no_grad():
        sb, mb = actor.sigma.model[0].bias, actor.mu.model[0].bias
        sb.copy_(torch.tensor([((-25.0, 3.0, 0.0, -1.0) if low_sigma else (3.0, -1.0, 0.0, 2.5))[a % 4] for a in range(A)]))
        mb.copy_(torch.tensor([(0.0, 0.0, 12.0, -12.0, 0.5)[a % 5] for a in range(A)]))
    alpha = AutoAlpha(target_entropy=-float(A), log_alpha=float(np.log(0.2)), optim=AdamOptimizerFactory(lr=3e-2)).to(DEV) \
        if auto_alpha else 0.2
    lr = 1e-3
    algo = SAC(policy=SACPolicy(actor=actor, action_space=Box(A)), policy_optim=AdamOptimizerFactory(lr=lr), critic=c1,
               critic_optim=AdamOptimizerFactory(lr=lr), critic2=c2, critic2_optim=AdamOptimizerFactory(lr=lr) if c2 else None,
               tau=0.005, gamma=0.99, alpha=alpha)
    E, T = 8, 64
    buf = (PrioritizedVectorReplayBuffer(E * T, E, alpha=0.6, beta=0.4, device=DEV) if per else VectorReplayBuffer(E * T, E, device=DEV))
    for s in synth_rollout(np.random.default_rng(seed), E, T, O, A, p_term=0.05, trunc_len=20):
        buf.add(Batch(**s), buffer_ids=np.arange(E))
    if per:
        buf.update_weight(np.arange(E * T), np.random.default_rng(seed + 1).uniform(0.1, 2.0, E * T))
    cap = {"noise": [], "adam": []}
    groups = [algo._g_c[0], algo._g_c[1], algo._g_actor]
    noise_fn = algo._noise_fn

    def noise(shape):
        n = noise_fn(shape)
        cap["noise"].append(n.clone())
        return n

    def adam(group, opt, mgn):
        cap["adam"].append((group, group.grad.clone(), [g.flat.clone() for g in groups]))
        FlatGroup.adam_step(group, opt, mgn)

    orig_pre, orig_post = algo._preprocess_batch, algo._postprocess_batch

    def pre(batch, buffer, indices):
        b = orig_pre(batch, buffer, indices)
        cap.update(obs=b.obs.clone(), act=b.act.clone(), returns=b.returns.detach().reshape(-1).clone(),
                   weight=None if getattr(b, "weight", None) is None else torch.as_tensor(b.weight).reshape(-1).clone())
        return b

    def post(batch, buffer, indices):
        cap["prio_td"] = torch.as_tensor(batch.weight).detach().reshape(-1).clone()
        return orig_post(batch, buffer, indices)

    algo._noise_fn, algo._adam, algo._preprocess_batch, algo._postprocess_batch = noise, adam, pre, post
    log_alpha0 = float(alpha._log_alpha.item()) if auto_alpha else None
    np.random.seed(seed)
    with policy_within_training_step(algo.policy):
        stats = algo.update(buffer=buf, sample_size=B)
    torch.cuda.synchronize()
    tag = f"sac_grad{edge}/{O}x{A}_c2{int(separate_critic2)}_per{int(per)}_auto{int(auto_alpha)}"
    assert [g for g, *_ in cap["adam"]] == groups and len(cap["noise"]) == 2
    obs, act, R = (cap[k].cpu().to(torch.float64) for k in ("obs", "act", "returns"))
    w = cap["weight"].cpu().to(torch.float64) if per else torch.ones(B, dtype=torch.float64)
    # critics: loss = mean((Q(s, a) - returns)^2 * w)  (ddpg.py:279-284), on the parameters before their own step
    tds = []
    for k, (mod, losskey) in enumerate(((c1, "critic1_loss"), (algo.critic2, "critic2_loss"))):
        group, grad, flats = cap["adam"][k]
        ref = _copy64(mod, group, flats[k])
        q = ref.last.model(ref.preprocess.model.model(torch.cat([obs, act], 1))).view(-1)
        td = q - R
        loss = (td.pow(2) * w).mean()
        loss.backward()
        tds.append(td.detach())
        _check_grads(f"{tag}/critic{k + 1}", mod, group, grad, ref, rows=B)
        record_parity(f"{tag}/{losskey}", np.array([getattr(stats, losskey)]), np.array([loss.item()]), rtol=2e-5, atol=1e-7)
    if per:          # the priority update (td1 + td2) / 2 (sac.py:318)
        record_parity(f"{tag}/prio_td", cap["prio_td"].cpu().numpy(), ((tds[0] + tds[1]) / 2).numpy(), rtol=1e-5,
                      atol=1e-5 * float(R.abs().max()))
    # actor: loss = mean(alpha * logp - min(Q1, Q2)(s, tanh(x))), x = mu + sigma * noise, critics after their steps
    group, grad, flats = cap["adam"][2]
    ra = _copy64(actor, group, flats[2])
    rc = [_copy64(m, algo._g_c[k], flats[k]) for k, m in enumerate((c1, algo.critic2))]
    h = ra.preprocess.model.model(obs)
    mu, raw = ra.mu.model(h), ra.sigma.model(h)
    sig = raw.clamp(-20.0, 2.0).exp()
    nz = cap["noise"][1].cpu().to(torch.float64)
    x = mu + sig * nz
    t = _GivenTanh.apply(x, algo._scratch["au_act"].cpu().to(torch.float64))
    logp = torch.distributions.Normal(mu, sig).log_prob(x).sum(-1) - torch.log(1 - t.pow(2) + np.finfo(np.float32).eps).sum(-1)
    qs = [m.last.model(m.preprocess.model.model(torch.cat([obs, t], 1))).view(-1) for m in rc]
    alpha0 = float(np.exp(log_alpha0)) if auto_alpha else 0.2
    (alpha0 * logp - torch.min(qs[0], qs[1])).mean().backward()
    _check_grads(f"{tag}/actor", actor, group, grad, ra, rows=B)
    sat = float((algo._scratch["au_act"].abs() == 1.0).float().mean())
    clamped = float(((raw < -20.0) | (raw > 2.0)).double().mean())
    if B >= 64:      # a handful of rows need not hit every head bias
        assert sat > 0.05 and clamped > 0.2, "the head biases must saturate some actions and clamp some log-sigmas"
    ties = float((qs[0] == qs[1]).double().mean())
    assert ties == (0.0 if separate_critic2 else 1.0), "critic2=None deep-copies the critic: every row ties"
    lp_k = algo._scratch["au_logp"].cpu().to(torch.float64)
    if low_sigma:
        # the actor loss is checked on the kernel's own log-prob rows: at sigma = e^-20 the fp32 rsample rounds to mu,
        # which every fp32 implementation shares (the forward kernel is checked against float64 in test_offpolicy_kernels_gpu)
        assert float(sig.min()) < 1e-8
    else:
        # no log-sigma at the lower bound: the log-prob rows the update used against float64 at the same action (fp32
        # terms of size up to ~17 x 16 per row: 1e-5 relative of the largest row)
        assert float(sig.min()) > 1e-3
        lp64 = logp.detach()
        record_parity(f"{tag}/logp", lp_k.numpy(), lp64.numpy(), rtol=1e-5, atol=1e-5 * float(lp64.abs().max()))
        lp_k = lp64
    record_parity(f"{tag}/actor_loss", np.array([stats.actor_loss]), np.array([(alpha0 * lp_k - torch.min(qs[0], qs[1])).mean().item()]),
                  rtol=2e-5, atol=1e-6)
    if auto_alpha:   # sac.py:203-215: alpha_loss = -(log_alpha * (target_entropy - entropy)).mean(), entropy = -logp; one Adam step
        deficit = -float(A) + lp_k
        ref_loss = -(log_alpha0 * deficit).mean().item()
        record_parity(f"{tag}/alpha_loss", np.array([stats.alpha_loss]), np.array([ref_loss]), rtol=1e-5, atol=1e-6)
        g_la = -deficit.mean().item()
        ref_la = log_alpha0 - 3e-2 * np.sign(g_la)        # Adam's first step: lr * g / (|g| + eps)
        record_parity(f"{tag}/log_alpha", np.array([alpha._log_alpha.item()]), np.array([ref_la]), rtol=0.0, atol=1e-6)
    else:
        assert stats.alpha_loss is None
    return cap, stats


SAC_GRAD_CASES = [
    (11, 4, (64, 64), False, False, False),
    (11, 4, (64, 64), True, False, False),
    (11, 5, (64, 64), False, True, True),
    (376, 17, (256, 256), False, False, False),
    (376, 17, (256, 256), True, True, True),
]


@pytest.mark.parametrize("O,A,H,separate_critic2,per,auto_alpha", SAC_GRAD_CASES,
                         ids=[f"obs{c[0]}-act{c[1]}-c2{int(c[3])}-per{int(c[4])}-auto{int(c[5])}" for c in SAC_GRAD_CASES])
def test_sac_update_gradients_vs_fp64_autograd(O, A, H, separate_critic2, per, auto_alpha):
    """One SAC update: the flat gradient of each of the three optimiser steps (snapshotted before the step) against
    float64 autograd of the reference losses on copies of the same modules with the same parameters, batch, returns and
    rsample noise.  Adam's first step is lr * sign(g), so a gradient off by a constant factor leaves the parameters
    unchanged; this is the check that sees it.  critic2=None (the default) deep-copies the critic, so both critics stay
    identical and every row of the actor step is a tie of min(Q1, Q2)."""
    sac_grad_case(O, A, H, separate_critic2, per, auto_alpha, seed=O + A)


def dqn_grad_setup(kind, A, seed, per, alpha_beta=(0.6, 0.4)):
    """A Q-network and a filled buffer.  kind: 'mlp' (Net on flat fp32 observations), 'mlp_scaled' (the same behind
    ScaledObsInputActionReprNet(denom=4): the flat gather divides by the denominator), 'cnn_stacked' (NatureCNN on
    stored uint8 [4, H, W] stacks: stack_num 1, obs_next = obs[next(i)])."""
    from tianshou_b200.data import Batch, PrioritizedVectorReplayBuffer, VectorReplayBuffer
    from tianshou_b200.env.atari import DQNet, ScaledObsInputActionReprNet
    from tianshou_b200.utils.net.common import Net
    torch.manual_seed(seed)
    rng = np.random.default_rng(seed)
    E, T = 4, 64
    if kind.startswith("mlp"):
        O = 12
        net = Net(state_shape=(O,), action_shape=(A,), hidden_sizes=(64, 64))
        if kind == "mlp_scaled":
            net = ScaledObsInputActionReprNet(net, denom=4.0)
        kw = {}
        obs_fn = lambda: rng.standard_normal((E, O)).astype(np.float32) * 3.0
    else:
        H = W = 36
        net = ScaledObsInputActionReprNet(DQNet(4, H, W, A))
        kw = dict(stack_num=1, ignore_obs_next=True)
        obs_fn = lambda: rng.integers(0, 256, (E, 4, H, W), dtype=np.uint8)
    net = net.to(DEV)
    buf = (PrioritizedVectorReplayBuffer(E * T, E, alpha=alpha_beta[0], beta=alpha_beta[1], device=DEV, **kw) if per
           else VectorReplayBuffer(E * T, E, device=DEV, **kw))
    obs = obs_fn()
    for t in range(T):
        nxt = obs_fn()
        term = rng.random(E) < 0.1
        trunc = (np.full(E, t % 17 == 16)) & ~term
        buf.add(Batch(obs=obs, act=rng.integers(0, A, E), rew=rng.standard_normal(E), terminated=term, truncated=trunc,
                      obs_next=nxt), buffer_ids=np.arange(E))
        obs = nxt
    if per:
        buf.update_weight(np.arange(E * T), rng.uniform(0.1, 2.0, E * T))
    return net, buf


def _q64(ref, kind, obs):
    """Q values of the float64 copy ``ref`` on host observations, with the input rounding of the reference's fp32 forward:
    fp32(obs / denom), the division in float64 as numpy does it."""
    if kind == "mlp":
        return ref.model.model(torch.as_tensor(obs).to(torch.float64))
    x = torch.as_tensor((np.asarray(obs, np.float64) / float(ref.denom)).astype(np.float32)).to(torch.float64)
    return ref.module.model.model(x) if kind == "mlp_scaled" else ref.module.net(x)


DQN_GRAD_CASES = [
    ("mlp", "mse", True, True, 0),
    ("mlp_scaled", "huber", False, False, 3),
    ("mlp", "huber", True, False, 3),
    ("cnn_stacked", "mse", True, True, 3),
    ("cnn_stacked", "huber", False, False, 0),
]


@pytest.mark.parametrize("kind,loss,per,is_double,tuf", DQN_GRAD_CASES,
                         ids=[f"{c[0]}-{c[1]}-per{int(c[2])}-double{int(c[3])}-tuf{c[4]}" for c in DQN_GRAD_CASES])
def test_dqn_update_gradients_vs_fp64_autograd(kind, loss, per, is_double, tuf):
    dqn_grad_case(kind, loss, per, is_double, tuf)


def dqn_grad_case(kind, loss, per, is_double, tuf, B=None, edge=""):
    """Two DQN updates: the flat gradient snapshotted at FlatGroup.adam_step against float64 autograd of the reference loss
    (dqn.py:384-401: MSE weighted by the PER importance weights, or the unweighted Huber loss with delta 0.5, which puts
    rows on both sides) on a copy of the same module with the same parameters and batch; the TD errors handed to the
    priority update; and the 1-step returns r + gamma (1 - terminated) Q_target(s', a*), a* = argmax of the online
    (double) or the target network.  The second update tells the target paths apart: with target_update_freq 3 the
    target network still holds the initial weights, with 0 there is no target network and the online one is used."""
    import copy

    from tianshou_b200.algorithm import AdamOptimizerFactory
    from tianshou_b200.algorithm.modelfree.dqn import DQN, DiscreteQLearningPolicy
    from tianshou_b200.utils import policy_within_training_step
    A, gamma, delta = 6, 0.9, 0.5
    net, buf = dqn_grad_setup(kind, A, seed=len(kind) * 10 + int(per), per=per)
    init64 = copy.deepcopy(net).to("cpu", torch.float64)
    algo = DQN(policy=DiscreteQLearningPolicy(model=net, action_space=Discrete(A)), optim=AdamOptimizerFactory(lr=1e-3),
               gamma=gamma, n_step_return_horizon=1, target_update_freq=tuf, is_double=is_double,
               huber_loss_delta=delta if loss == "huber" else None)
    assert (algo.model_old is None) == (tuf == 0)
    group = algo._group
    cap = []
    real_step = group.adam_step

    def adam_step(optimizer, max_grad_norm):
        cap[-1].update(grad=group.grad.clone(), flat=group.flat.clone())
        real_step(optimizer, max_grad_norm)

    group.adam_step = adam_step
    orig_pre, orig_post = algo._preprocess_batch, algo._postprocess_batch

    def pre(batch, buffer, indices):
        w = batch.__dict__.get("weight")
        cap.append(dict(indices=np.asarray(indices).copy(), weight=None if w is None else w.detach().cpu().clone()))
        b = orig_pre(batch, buffer, indices)
        cap[-1]["returns"] = b.returns.detach().reshape(-1).cpu().clone()
        return b

    def post(batch, buffer, indices):
        cap[-1]["td"] = torch.as_tensor(batch.weight).detach().reshape(-1).cpu().clone()
        return orig_post(batch, buffer, indices)

    algo._preprocess_batch, algo._postprocess_batch = pre, post
    if B is None:
        B = 64 if kind == "cnn_stacked" else 256
    sides = set()
    for u in range(2):
        np.random.seed(700 + u)
        with policy_within_training_step(algo.policy):
            stats = algo.update(buffer=buf, sample_size=B)
        c = cap[u]
        tag = f"dqn_grad{edge}/{kind}_{loss}_per{int(per)}_d{int(is_double)}_tuf{tuf}_u{u}"
        idx = c["indices"]
        ref = _copy64(net, group, c["flat"])
        obs = np.asarray(buf.obs)[idx]
        obs_next = np.asarray(buf.obs)[buf.next(idx)] if kind == "cnn_stacked" else np.asarray(buf.obs_next)[idx]
        # target: online = the parameters of this update before its step; lagged = the initial weights (tuf 3, u <= 1)
        with torch.no_grad():
            q_on = _q64(ref, kind, obs_next)
            q_tg = _q64(init64, kind, obs_next) if tuf > 0 else q_on
            a_star = (q_on if is_double else q_tg).argmax(1, keepdim=True)
            tq = q_tg.gather(1, a_star).view(-1)
        term = torch.as_tensor(np.asarray(buf.terminated)[idx].astype(np.float64))
        R = torch.as_tensor(np.asarray(buf.rew)[idx].astype(np.float64)) + gamma * (1.0 - term) * tq
        record_parity(f"{tag}/returns", c["returns"].numpy(), R.numpy(), rtol=1e-5, atol=1e-5 * float(R.abs().max()))
        R = c["returns"].to(torch.float64)         # the loss below on the returns the update used
        q = _q64(ref, kind, obs)
        act = torch.as_tensor(np.asarray(buf.act)[idx].astype(np.int64)).view(-1, 1)
        q_sel = q.gather(1, act).view(-1)
        if loss == "huber":
            L = torch.nn.functional.huber_loss(q_sel, R, delta=delta, reduction="mean")
            d = (q_sel - R).detach().abs()
            sides |= ({"inside"} if bool((d < delta).any()) else set()) | ({"outside"} if bool((d > delta).any()) else set())
        else:
            w = c["weight"].to(torch.float64) if per else 1.0
            L = ((R - q_sel).pow(2) * w).mean()
        L.backward()
        _check_grads(tag, net, group, c["grad"], ref, rows=B)
        record_parity(f"{tag}/loss", np.array([stats.loss]), np.array([L.item()]), rtol=2e-5, atol=1e-7)
        record_parity(f"{tag}/td", c["td"].numpy(), (R - q_sel).detach().numpy(), rtol=1e-5, atol=1e-5 * float(R.abs().max()))
        assert len(idx) == B and c["td"].numel() == B, "the update must run on the B sampled rows"
    if loss == "huber" and B >= 64:
        assert sides == {"inside", "outside"}, "the Huber rows must lie on both sides of delta"


def test_dqn_stored_stacks_bit_identical_to_single_frame_storage():
    """NatureCNN DQN on stored uint8 stacks (stack_num 1, obs [4, H, W] per slot: frame slot idx * 4 + c of the flattened
    column) and on single-frame storage (stack_num 4, save_only_last_obs: the slots come from the prev() chain) of the
    SAME stacks: the first convolution's im2col gathers the same bytes, so the Q values of the update batch, the targets,
    the losses and the flat gradients must agree bit for bit."""
    import copy

    from tianshou_b200.algorithm import AdamOptimizerFactory
    from tianshou_b200.algorithm.modelfree.dqn import DQN, DiscreteQLearningPolicy
    from tianshou_b200.data import Batch, VectorReplayBuffer
    from tianshou_b200.env.atari import DQNet, ScaledObsInputActionReprNet
    from tianshou_b200.utils import policy_within_training_step
    E, T, H, W, A = 4, 64, 36, 36, 5
    rng = np.random.default_rng(11)
    single = VectorReplayBuffer(E * T, E, stack_num=4, save_only_last_obs=True, ignore_obs_next=True, device=DEV)
    for t in range(T):
        frame = rng.integers(0, 256, (E, H, W), dtype=np.uint8)
        stack = np.repeat(frame[:, None], 4, axis=1)           # only the last frame is stored
        term = rng.random(E) < 0.1
        trunc = np.full(E, t % 13 == 12) & ~term
        single.add(Batch(obs=stack, act=rng.integers(0, A, E), rew=rng.standard_normal(E), terminated=term, truncated=trunc,
                         obs_next=stack), buffer_ids=np.arange(E))
    N = E * T
    stacks = single.get(np.arange(N), "obs")
    assert stacks.shape == (N, 4, H, W) and stacks.dtype == np.uint8
    stored = VectorReplayBuffer(N, E, stack_num=1, ignore_obs_next=True, device=DEV)
    stored.set_batch(Batch(obs=stacks, act=np.asarray(single.act).copy(), rew=np.asarray(single.rew).copy(),
                           terminated=np.asarray(single.terminated).copy(), truncated=np.asarray(single.truncated).copy(),
                           done=np.asarray(single.done).copy()))
    set_buffer_state(stored, single.last_index.copy(), single._sizes.copy())
    torch.manual_seed(4)
    net0 = ScaledObsInputActionReprNet(DQNet(4, H, W, A)).to(DEV)
    out = []
    for buf in (single, stored):
        algo = DQN(policy=DiscreteQLearningPolicy(model=copy.deepcopy(net0), action_space=Discrete(A)),
                   optim=AdamOptimizerFactory(lr=1e-3), gamma=0.9, n_step_return_horizon=1, is_double=True)
        rec = {"q": [], "grad": [], "idx": [], "returns": []}
        real_q, real_step, orig_pre = algo._q_values, algo._group.adam_step, algo._preprocess_batch

        def q_values(src, tag, target=False, _rec=rec, _real=real_q):
            acts, q = _real(src, tag, target)
            _rec["q"].append(q.clone())
            return acts, q

        def adam_step(optimizer, mgn, _rec=rec, _g=algo._group, _real=real_step):
            _rec["grad"].append(_g.grad.clone())
            _real(optimizer, mgn)

        def pre(batch, buffer, indices, _rec=rec, _orig=orig_pre):
            b = _orig(batch, buffer, indices)
            _rec["idx"].append(np.asarray(indices).copy())
            _rec["returns"].append(b.returns.detach().clone())
            return b

        algo._q_values, algo._group.adam_step, algo._preprocess_batch = q_values, adam_step, pre
        for u in range(2):
            np.random.seed(900 + u)
            with policy_within_training_step(algo.policy):
                rec.setdefault("loss", []).append(algo.update(buffer=buf, sample_size=64).loss)
        rec["flat"] = algo._group.flat.clone()
        out.append(rec)
    a, b = out
    for u in range(2):
        assert np.array_equal(a["idx"][u], b["idx"][u]), "both buffers must sample the same transitions"
    assert len(a["q"]) == len(b["q"]) and all(torch.equal(x, y) for x, y in zip(a["q"], b["q"], strict=True))
    assert all(torch.equal(x, y) for x, y in zip(a["returns"], b["returns"], strict=True))
    assert all(torch.equal(x, y) for x, y in zip(a["grad"], b["grad"], strict=True))
    assert a["loss"] == b["loss"] and torch.equal(a["flat"], b["flat"])


def test_dqn_state_dict_keys():
    """The reference's keys (test_oracle_offpolicy.py checks them against the reference): the lagged copy under ``.module``."""
    from test_oracle_offpolicy import DQN_MLP_STATE_DICT_KEYS

    from tianshou_b200.algorithm import AdamOptimizerFactory
    from tianshou_b200.algorithm.modelfree.dqn import DQN, DiscreteQLearningPolicy
    from tianshou_b200.utils.net.common import Net
    policy = DiscreteQLearningPolicy(model=Net(state_shape=(4,), action_shape=3, hidden_sizes=(16,)).to(DEV), action_space=Discrete(3))
    algo = DQN(policy=policy, optim=AdamOptimizerFactory(lr=1e-3), target_update_freq=10)
    assert list(algo.state_dict().keys()) == DQN_MLP_STATE_DICT_KEYS


def test_dqn_state_dict_round_trip_continues_identically():
    """A fresh DQN with other initial weights, loaded from another's ``state_dict()``, continues bit for bit: online, lagged
    and optimiser state.  With ``target_update_freq`` 10 the six updates copy the lagged network once, in the first, so
    the loaded algorithm's targets come from the lagged network the load restored.  ``_iter`` is a plain attribute, as in
    the reference: whoever restores a run restores it too."""
    import copy

    from tianshou_b200.algorithm import AdamOptimizerFactory
    from tianshou_b200.algorithm.modelfree.dqn import DQN, DiscreteQLearningPolicy
    from tianshou_b200.utils import policy_within_training_step
    A = 6

    def build(seed):
        net, buf = dqn_grad_setup("mlp", A, seed=seed, per=False)
        return DQN(policy=DiscreteQLearningPolicy(model=net, action_space=Discrete(A)), optim=AdamOptimizerFactory(lr=1e-3),
                   gamma=0.9, n_step_return_horizon=2, target_update_freq=10), buf

    a, buf_a = build(5)
    for u in range(3):
        np.random.seed(u)
        with policy_within_training_step(a.policy):
            a.update(buffer=buf_a, sample_size=64)
    b, _ = build(6)
    b.load_state_dict(copy.deepcopy(a.state_dict()))
    b._iter = a._iter
    for algo in (a, b):
        buf = dqn_grad_setup("mlp", A, seed=5, per=False)[1]
        for u in range(3):
            np.random.seed(10 + u)
            with policy_within_training_step(algo.policy):
                algo.update(buffer=buf, sample_size=64)
    for ga, gb in ((a._group, b._group), (a._g_old, b._g_old)):
        assert torch.equal(ga.flat, gb.flat) and torch.equal(ga.exp_avg, gb.exp_avg) and torch.equal(ga.exp_avg_sq, gb.exp_avg_sq)
    assert a._group.step == b._group.step


@pytest.mark.parametrize("algo_name", ["dqn", "discrete_sac"])
@pytest.mark.parametrize("bad", ["A", "-1"])
def test_drawn_actions_outside_the_network_outputs_are_refused(algo_name, bad):
    """The loss kernels index a row of A values with each drawn action: a buffer holding A or -1 is refused on the host
    while the batch is drawn, before anything is launched."""
    from tianshou_b200.algorithm import AdamOptimizerFactory, DiscreteSAC
    from tianshou_b200.algorithm.modelfree.discrete_sac import DiscreteSACPolicy
    from tianshou_b200.algorithm.modelfree.dqn import DQN, DiscreteQLearningPolicy
    from tianshou_b200.data import Batch, VectorReplayBuffer
    from tianshou_b200.utils import policy_within_training_step
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.discrete import DiscreteActor, DiscreteCritic
    A = 3
    net = lambda **kw: Net(state_shape=(4,), hidden_sizes=(16,), **kw).to(DEV)
    if algo_name == "dqn":
        algo = DQN(policy=DiscreteQLearningPolicy(model=net(action_shape=A), action_space=Discrete(A)),
                   optim=AdamOptimizerFactory(lr=1e-3), target_update_freq=2)
    else:
        actor = DiscreteActor(preprocess_net=net(), action_shape=A, softmax_output=False).to(DEV)
        algo = DiscreteSAC(policy=DiscreteSACPolicy(actor=actor, action_space=Discrete(A)), policy_optim=AdamOptimizerFactory(lr=1e-3),
                           critic=DiscreteCritic(preprocess_net=net(), last_size=A).to(DEV), critic_optim=AdamOptimizerFactory(lr=1e-3))
    buf = VectorReplayBuffer(40, 4, device=DEV)
    rng = np.random.default_rng(0)
    for _ in range(8):
        buf.add(Batch(obs=rng.standard_normal((4, 4)).astype(np.float32), act=np.array([0, 1, A if bad == "A" else -1, 2]),
                      rew=np.zeros(4), terminated=np.zeros(4, bool), truncated=np.zeros(4, bool),
                      obs_next=rng.standard_normal((4, 4)).astype(np.float32)), buffer_ids=np.arange(4))
    np.random.seed(0)
    with pytest.raises(ValueError, match="actions in"), policy_within_training_step(algo.policy):
        algo.update(buffer=buf, sample_size=32)
