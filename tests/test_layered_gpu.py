"""Layer-wise actor-critic path (algorithm/layered.py: every Linear forward / backward = one wgmma GEMM launch, loss rows
in between) -- the path networks OUTSIDE the fused 17-64-64 kernels' envelope take.  Checked (a) on the reference's own
goldens by forcing the path onto shapes the fused kernels also cover (discrete shared-trunk ReLU net ppo_ref_C1*, MuJoCo
tanh net ppo_ref_A/B), and (b) on shapes only this path accepts (obs 376, MLP[256,256] -- Humanoid / BASELINE configs[3]
width; a three-layer trunk) against the numpy oracle / torch autograd."""
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
    """A deeper trunk (three hidden layers, different widths) -- gradients of one layered minibatch step vs torch autograd of
    the same PPO loss on the same modules."""
    from tianshou_b200.algorithm import PPO, AdamOptimizerFactory, ProbabilisticActorPolicy
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.continuous import ContinuousActorProbabilistic, ContinuousCritic
    from ts_testutil import Box, gaussian_dist
    O, A, H = 29, 4, (96, 80, 40)
    torch.manual_seed(1)
    actor = ContinuousActorProbabilistic(preprocess_net=Net(state_shape=(O,), hidden_sizes=H), action_shape=(A,), unbounded=True).to(DEV)
    critic = ContinuousCritic(preprocess_net=Net(state_shape=(O,), hidden_sizes=H)).to(DEV)
    policy = ProbabilisticActorPolicy(actor=actor, dist_fn=gaussian_dist, action_scaling=True, action_bound_method="clip",
                                      action_space=Box(A))
    algo = PPO(policy=policy, critic=critic, optim=AdamOptimizerFactory(lr=0.0), eps_clip=0.2, vf_coef=0.5, ent_coef=0.02,
               value_clip=False, advantage_normalization=False, max_grad_norm=None)
    L = algo._layered
    assert L is not None and len(L.a_trunk.layers) == 3
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
    # torch autograd reference of ppo.py:183-211 on the same modules (lr = 0: the step did not move the parameters)
    (mu, sig), _ = actor(obs)
    dist = gaussian_dist((mu, sig))
    ratio = (dist.log_prob(act) - lpo).exp()
    surr = torch.min(ratio * adv, ratio.clamp(0.8, 1.2) * adv)
    value = critic(obs).flatten()
    loss = -surr.mean() + 0.5 * (ret - value).pow(2).mean() - 0.02 * dist.entropy().mean()
    for p_ in L.group.params:
        p_.grad = None
    loss.backward()
    record_parity("layered_deep/loss", stats_row[:1].cpu().numpy(), np.array([float(loss)]), rtol=2e-5, atol=1e-6)
    for i, p_ in enumerate(L.group.params):
        got = L.group.view(L.group.grad, p_).view(p_.shape).cpu().numpy()
        ref = p_.grad.cpu().numpy()
        record_parity(f"layered_deep/grad{i}", got, ref, rtol=2e-4, atol=2e-5 * float(np.abs(ref).max()) + 1e-9)
