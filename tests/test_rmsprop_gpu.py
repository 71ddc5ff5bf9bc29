"""torch.optim.RMSprop on the device update (``ts_ppo_hparams.optimizer = TS_OPT_RMSPROP``): the SIMT / NCCL step
(``ts_clip_adam_step``) and the layer-wise step (``ts_rmsprop_step``) against clip_grad_norm_ + torch.optim.RMSprop, and
``A2C.update()`` / ``NPG.update()`` on every path against the imported reference's runs with RMSprop
(tests/golden/a2c_rmsprop_ref*.npz, npg_rmsprop_ref.npz, oracle/gen_golden_rmsprop.py).

Parameter bars: RMSprop moves an element by at most lr / sqrt(1 - alpha) per step (10 lr at alpha = 0.99), where Adam moves
it by about lr, so the absolute part of each Adam bar that scales with lr is taken in units of lr / sqrt(1 - alpha) here."""
import ctypes as C
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch

from ts_testutil import PARAM_ORDER, Box, build_actor_critic, gaussian_dist, load_golden, load_params, named_params, record_parity
from ts_testutil import restore_vector_buffer

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _sms() -> int:
    return torch.cuda.get_device_properties(0).multi_processor_count


def _step_bound(lr: float, alpha: float) -> float:
    return lr / np.sqrt(1.0 - alpha)


# --------------------------------------------------------------------------------------------- the step kernels
STEP_N = ["1", "255", "4097", "wave"]
STEP_PARTIALS = ["0", "1", "sms"]


def _resolve(x, sms):
    return {"wave": sms * 256 - 4, "sms": sms}.get(x) or int(x)


def _torch_rmsprop(p0, sq0, step0, lr, alpha, eps, wd):
    p_ref = p0.clone().to(DEV).requires_grad_(True)
    opt = torch.optim.RMSprop([p_ref], lr=lr, alpha=alpha, eps=eps, weight_decay=wd, foreach=False)
    if step0:
        opt.state[p_ref] = {"step": torch.tensor(float(step0)), "square_avg": sq0.to(DEV).clone()}
    return p_ref, opt


@pytest.mark.parametrize("n_partials", STEP_PARTIALS)
@pytest.mark.parametrize("n", STEP_N)
def test_clip_step_rmsprop_vs_torch(n, n_partials):
    """ts_clip_adam_step with hp.optimizer = TS_OPT_RMSPROP (the SIMT / NCCL step): partial rows folded, clip off / above /
    below, weight decay 0 / 0.01, three steps from step 0 and from step 57, against the fold in fp64 + clip_grad_norm_ +
    torch.optim.RMSprop(foreach=False); exp_avg is left as it was, the step count advances."""
    from tianshou_b200._cabi import OPT_RMSPROP, ActorCriticDesc, PPOHParams, call, ptr, stream_ptr
    sms = _sms()
    n, n_p = _resolve(n, sms), _resolve(n_partials, sms)
    W = n + 4
    desc = ActorCriticDesc()
    desc.n_params = n
    gen = torch.Generator().manual_seed(n * 1000 + n_p + 7)
    fold_rel = (n_p / 32 + 12) * 2.0 ** -24        # fp32 fold of same-sign rows (see test_simt_kernels_gpu)
    sign = torch.where(torch.randn(n, generator=gen) >= 0, 1.0, -1.0)

    def grad_rows(k):
        g = sign.double() * torch.randn(n, generator=gen, dtype=torch.float64).abs() * (1.0 + k)
        target = torch.cat([g, torch.tensor([1.0, 2.0, 0.5, 0.0], dtype=torch.float64)])
        if n_p == 0:
            row = target.float()
            row[n + 3] = 300.0
            return None, row.double()
        w = 0.5 + torch.rand(n_p, W, generator=gen, dtype=torch.float64)
        rows = (target * (w / w.sum(0))).float()
        rows[:, n + 3] = 128.0
        return rows, rows.double().sum(0)

    lr, alpha, eps = 7e-4, 0.99, 1e-5
    bound = _step_bound(lr, alpha)
    sq = float(np.sqrt(n))
    for clip_name, max_norm in (("off", 0.0), ("above", 100.0 * sq), ("below", 1e-2 * sq)):
        for wd in (0.0, 0.01):
            for step0 in (0, 57):
                cfg = f"simt_rmsprop/n{n}_p{n_p}/clip_{clip_name}_wd{wd}_step{step0}"
                p0 = sign * torch.randn(n, generator=gen).abs()
                sq0 = 0.01 * torch.rand(n, generator=gen) + 1e-4 if step0 else torch.zeros(n)
                p_ref, opt = _torch_rmsprop(p0, sq0, step0, lr, alpha, eps, wd)
                pk, sk = p0.to(DEV).clone(), sq0.to(DEV).clone()
                mk = torch.full((n,), 3.25, device=DEV)          # exp_avg: not RMSprop state, must stay untouched
                step = torch.tensor([step0], dtype=torch.int64, device=DEV)
                hp = PPOHParams(vf_coef=0.25, ent_coef=0.01, max_grad_norm=max_norm, adv_eps=1e-8, lr=lr, adam_eps=eps,
                                weight_decay=wd, optimizer=OPT_RMSPROP, beta2=alpha)
                for k in range(3):
                    rows, fold = grad_rows(k)
                    q = torch.zeros(n, dtype=torch.float64, requires_grad=True)
                    q.grad = fold[:n].clone()
                    norm = float(torch.nn.utils.clip_grad_norm_([q], max_norm)) if max_norm > 0 else float(q.grad.norm())
                    if max_norm > 0:
                        assert (norm > max_norm) == (clip_name == "below")
                    p_ref.grad = q.grad.float().to(DEV)
                    opt.step()
                    grad = fold.float().to(DEV) if rows is None else torch.full((W,), float("nan"), device=DEV)
                    stats = torch.full((8,), float("nan"), device=DEV)
                    call("ts_clip_adam_step", ptr(pk), ptr(grad), ptr(None if rows is None else rows.to(DEV)), n_p, ptr(mk),
                         ptr(sk), ptr(step), C.byref(desc), C.byref(hp), ptr(stats), stream_ptr())
                    assert int(step.item()) == step0 + k + 1
                    record_parity(f"{cfg}/grad_norm", stats[4:5].cpu().numpy(), np.array([norm]), rtol=fold_rel + 1e-6, atol=0.0)
                    # square_avg: g^2 carries twice the fold's relative error; parameters: the Adam step test's bar (1e-6
                    # relative + 2e-3 lr) with lr replaced by RMSprop's per-step bound, widened by the fold's error
                    sa = opt.state[p_ref]["square_avg"].cpu().numpy()
                    record_parity(f"{cfg}/square_avg", sk.cpu().numpy(), sa, rtol=4e-6 + 2 * fold_rel, atol=0.0)
                    record_parity(f"{cfg}/params", pk.cpu().numpy(), p_ref.detach().cpu().numpy(), rtol=1e-6,
                                  atol=bound * (2e-4 + 2 * fold_rel))
                assert torch.equal(mk, torch.full_like(mk, 3.25))


@pytest.mark.parametrize("n", [1, 1000, 300_001])
def test_rmsprop_step_vs_torch(n):
    """ts_rmsprop_step (layer-wise step): clip off / above / below, weight decay 0 / 0.01, three steps from an empty and from
    a warm square_avg, against clip_grad_norm_ + torch.optim.RMSprop(foreach=False)."""
    from tianshou_b200._cabi import call, ptr, stream_ptr
    gen = torch.Generator().manual_seed(n)
    lr, alpha, eps = 1e-3, 0.99, 1e-5
    scratch = torch.zeros(256, dtype=torch.float64, device=DEV)
    sign = torch.where(torch.randn(n, generator=gen) >= 0, 1.0, -1.0)
    sq = float(np.sqrt(n))
    for clip_name, max_norm in (("off", 0.0), ("above", 100.0 * sq), ("below", 1e-2 * sq)):
        for wd in (0.0, 0.01):
            for step0 in (0, 57):
                cfg = f"rmsprop_step/n{n}/clip_{clip_name}_wd{wd}_step{step0}"
                p0 = sign * torch.randn(n, generator=gen).abs()
                sq0 = 0.01 * torch.rand(n, generator=gen) + 1e-4 if step0 else torch.zeros(n)
                p_ref, opt = _torch_rmsprop(p0, sq0, step0, lr, alpha, eps, wd)
                pk, sk = p0.to(DEV).clone(), sq0.to(DEV).clone()
                for k in range(3):
                    gk = (sign * torch.randn(n, generator=gen).abs() * (1.0 + k)).to(DEV)
                    p_ref.grad = gk.clone()
                    if max_norm > 0:
                        torch.nn.utils.clip_grad_norm_([p_ref], max_norm)
                    opt.step()
                    call("ts_rmsprop_step", ptr(pk), ptr(gk), ptr(sk), n, lr, alpha, eps, wd, max_norm, ptr(scratch), stream_ptr())
                    record_parity(f"{cfg}/square_avg", sk.cpu().numpy(), opt.state[p_ref]["square_avg"].cpu().numpy(),
                                  rtol=4e-6, atol=0.0)
                    record_parity(f"{cfg}/params", pk.cpu().numpy(), p_ref.detach().cpu().numpy(), rtol=1e-6,
                                  atol=_step_bound(lr, alpha) * 2e-4)


# --------------------------------------------------------------------------------------------- updates vs the goldens
def _rmsprop_factory(g, schedule=True):
    from tianshou_b200.algorithm.optim import LRSchedulerFactoryLinear, RMSpropOptimizerFactory
    f = RMSpropOptimizerFactory(lr=float(g["opt_lr"]), eps=float(g["opt_eps"]), alpha=float(g["opt_alpha"]))
    if schedule:      # the recipe's schedule: two updates, lr then lr / 2
        f.with_lr_scheduler_factory(LRSchedulerFactoryLinear(max_epochs=1, epoch_num_steps=1024, collection_step_num_env_steps=512))
    return f


def _a2c_kwargs(g):
    return dict(gamma=float(g["kw_gamma"]), gae_lambda=float(g["kw_gae_lambda"]), max_grad_norm=float(g["kw_max_grad_norm"]),
                vf_coef=float(g["kw_vf_coef"]), ent_coef=float(g["kw_ent_coef"]), return_scaling=bool(g["kw_return_scaling"]))


def _gauss_a2c(g, device=DEV):
    from tianshou_b200.algorithm import A2C, ProbabilisticActorPolicy
    actor, critic = build_actor_critic(17, 6, device)
    load_params(actor, critic, {k: g["p0_" + k] for k in PARAM_ORDER})
    policy = ProbabilisticActorPolicy(actor=actor, dist_fn=gaussian_dist, action_scaling=True, action_bound_method="clip",
                                      action_space=Box(6))
    return A2C(policy=policy, critic=critic, optim=_rmsprop_factory(g), **_a2c_kwargs(g)), named_params(actor, critic)


def _discrete_a2c(g):
    from test_ppo_discrete_gpu import Discrete
    from test_ppo_discrete_gpu import named_params as discrete_named
    from tianshou_b200.algorithm import A2C, DiscreteActorPolicy
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.discrete import DiscreteActor, DiscreteCritic
    net = Net(state_shape=(4,), hidden_sizes=(64, 64))
    actor, critic = DiscreteActor(preprocess_net=net, action_shape=(2,)).to(DEV), DiscreteCritic(preprocess_net=net).to(DEV)
    named = discrete_named(actor, critic)
    with torch.no_grad():
        for k, p in named.items():
            p.copy_(torch.as_tensor(g["p0_" + k]).reshape(p.shape))
    policy = DiscreteActorPolicy(actor=actor, dist_fn=torch.distributions.Categorical, action_space=Discrete(2),
                                 deterministic_eval=True)
    return A2C(policy=policy, critic=critic, optim=_rmsprop_factory(g), **_a2c_kwargs(g)), named


def _run_vs_golden(tag, g, algo, named, path):
    """Two updates vs the reference run: v_s / returns / adv, the loss table row by row, the parameters after each update."""
    from tianshou_b200.utils import policy_within_training_step
    assert algo._layered is None if path in ("fused", "simt") else algo._layered is not None
    captured = {}
    orig = algo._preprocess_batch

    def hook(batch, buffer, indices):
        b = orig(batch, buffer, indices)
        captured.update({k: b[k].detach().cpu().numpy().copy() for k in ("v_s", "returns", "adv")})
        return b

    algo._preprocess_batch = hook
    E, cap = int(g["cfg_E"]), int(g["cfg_cap"])
    alpha = float(g["opt_alpha"])
    for u in range(2):
        o = f"u{u}_"
        lr = float(g[o + "lr"])
        assert algo.optim._optim.param_groups[0]["lr"] == pytest.approx(lr)
        buf = restore_vector_buffer(g, o, E, cap, device=DEV)
        np.random.seed(1000 + u)
        with policy_within_training_step(algo.policy):
            stats = algo.update(buffer=buf, batch_size=int(g["cfg_bs"]), repeat=int(g["cfg_repeat"]))
        assert stats.gradient_steps == int(g[o + "gradient_steps"])
        # update 0 starts from the reference's parameters: test_ppo_gpu's bars; update 1 runs on parameters that already
        # carry update 0's differences
        for k, rt in (("v_s", 2e-5), ("returns", 2e-5), ("adv", 2e-5)):
            ref = g[o + k]
            bar = rt if u == 0 else 1e-3
            record_parity(f"{tag}_u{u}/{k}", captured[k], ref, rtol=bar, atol=bar * max(1.0, float(np.abs(ref).max())))
        ref = g[o + "losses"]
        record_parity(f"{tag}_u{u}/loss_table", algo.last_loss_table[:, :4], ref, rtol=2e-3,
                      atol=1e-4 * max(1.0, float(np.abs(ref).max())))
        for k, pv in named.items():
            # Adam's bar atol 3e-5 at lr 3e-4 is 0.1 lr; here 0.05 x lr / sqrt(1 - alpha) of this update's lr
            record_parity(f"{tag}_u{u}/{k}", pv.detach().cpu().numpy(), g[o + "p_" + k], rtol=2e-3,
                          atol=0.05 * _step_bound(lr, alpha))


@pytest.mark.parametrize("path", ["fused", "layered", "simt"])
def test_a2c_rmsprop_matches_reference(path, monkeypatch):
    """mujoco_a2c's optimiser on the fused tensor-core path, and the same run forced through the layer-wise path and the
    SIMT kernels."""
    if path == "layered":
        monkeypatch.setenv("TS_B200_FORCE_LAYERED", "1")
    if path == "simt" and os.environ.get("TS_B200_FORCE_SIMT") != "1":
        # the library reads TS_B200_FORCE_SIMT once per process: this case runs in a fresh one
        r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider",
                            f"{os.path.abspath(__file__)}::test_a2c_rmsprop_matches_reference[simt]"],
                           env={**os.environ, "TS_B200_FORCE_SIMT": "1"}, capture_output=True, text=True)
        assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-2000:]
        return
    g = load_golden("a2c_rmsprop_ref.npz")
    algo, named = _gauss_a2c(g)
    if path == "fused":
        assert algo._flat.weight_image is not None            # the tensor-core epoch kernel runs this shape
    _run_vs_golden(f"a2c_rmsprop/{path}", g, algo, named, path)


def test_a2c_rmsprop_discrete_shared_trunk_matches_reference():
    """The reference's discrete shared-ReLU-trunk network (SIMT kernels) with RMSprop."""
    g = load_golden("a2c_rmsprop_ref_C1.npz")
    algo, named = _discrete_a2c(g)
    assert algo._flat.weight_image is None
    _run_vs_golden("a2c_rmsprop/C1", g, algo, named, "simt")


def test_npg_rmsprop_critic_matches_reference():
    """NPG with an RMSprop critic optimiser: the layer-wise critic step is ts_rmsprop_step."""
    from test_npg_gpu import _nets
    from tianshou_b200.algorithm import NPG, ProbabilisticActorPolicy
    from tianshou_b200.algorithm.optim import RMSpropOptimizerFactory
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden("npg_rmsprop_ref.npz")
    O, A = int(g["cfg_obs"]), int(g["cfg_act"])
    actor, critic = _nets(False, O, A)
    with torch.no_grad():
        for mod, tag in ((actor, "actor"), (critic, "critic")):
            for i, p in enumerate(mod.parameters()):
                p.copy_(torch.as_tensor(g[f"p0_{tag}_{i}"]).reshape(p.shape))
    lr, alpha = float(g["cfg_lr"]), float(g["opt_alpha"])
    policy = ProbabilisticActorPolicy(actor=actor, dist_fn=gaussian_dist, action_scaling=True, action_bound_method="clip",
                                      action_space=Box(A))
    algo = NPG(policy=policy, critic=critic, optim=RMSpropOptimizerFactory(lr=lr, eps=float(g["opt_eps"]), alpha=alpha),
               return_scaling=bool(g["kw_return_scaling"]), advantage_normalization=bool(g["kw_advantage_normalization"]),
               optim_critic_iters=int(g["kw_optim_critic_iters"]), trust_region_size=float(g["kw_trust_region_size"]))
    E, cap = int(g["cfg_E"]), int(g["cfg_cap"])
    for u in range(2):
        o = f"u{u}_"
        buf = restore_vector_buffer(g, o, E, cap, device=DEV)
        np.random.seed(int(g[o + "np_seed"]))
        with policy_within_training_step(algo.policy):
            algo.update(buffer=buf, batch_size=None, repeat=int(g["cfg_repeat"]))
        table = algo.last_stats_table
        for name, col in (("actor_loss", 0), ("vf_loss", 1), ("kl", 2)):
            ref = g[o + name]
            record_parity(f"npg_rmsprop_u{u}/{name}", table[:, col], ref, rtol=2e-3, atol=1e-6 + 1e-4 * max(1e-3, float(np.abs(ref).max())))
        for mod, tag in ((actor, "actor"), (critic, "critic")):
            for i, p in enumerate(mod.parameters()):
                ref = g[f"{o}{tag}_{i}"]
                # test_npg_gpu's bar with the critic's lr in units of RMSprop's per-step bound
                record_parity(f"npg_rmsprop_u{u}/{tag}_{i}", p.detach().cpu().numpy(), ref.reshape(p.shape), rtol=2e-3,
                              atol=0.1 * _step_bound(lr, alpha) + 1e-3 * float(np.abs(ref).max()))


def test_wide_layered_update_vs_oracle():
    """obs 376 / [256, 256] (a Humanoid-sized network, outside the fused envelope: the layer-wise path) with RMSprop, two
    minibatch steps against the numpy restatement (oracle/oracle_rmsprop.py) of the same update."""
    from oracle import oracle_np as onp
    from oracle import oracle_rmsprop as orm
    from tianshou_b200.algorithm import A2C, ProbabilisticActorPolicy
    from tianshou_b200.algorithm.optim import RMSpropOptimizerFactory
    from tianshou_b200.data import Batch, VectorReplayBuffer
    from tianshou_b200.utils import policy_within_training_step
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.continuous import ContinuousActorProbabilistic, ContinuousCritic
    from ts_testutil import synth_rollout
    O, A, H, E, T = 376, 17, 256, 16, 16
    torch.manual_seed(3)
    actor = ContinuousActorProbabilistic(preprocess_net=Net(state_shape=(O,), hidden_sizes=(H, H), activation=torch.nn.Tanh),
                                         action_shape=(A,), unbounded=True).to(DEV)
    critic = ContinuousCritic(preprocess_net=Net(state_shape=(O,), hidden_sizes=(H, H), activation=torch.nn.Tanh)).to(DEV)
    named = named_params(actor, critic)
    p = {k: v.detach().cpu().numpy().astype(np.float32).copy() for k, v in named.items()}
    policy = ProbabilisticActorPolicy(actor=actor, dist_fn=gaussian_dist, action_scaling=True, action_bound_method="clip",
                                      action_space=Box(A))
    lr, alpha, eps = 7e-4, 0.99, 1e-5
    algo = A2C(policy=policy, critic=critic, optim=RMSpropOptimizerFactory(lr=lr, eps=eps, alpha=alpha), max_grad_norm=0.5,
               return_scaling=False)
    assert algo._layered is not None
    buf = VectorReplayBuffer(E * T, E, device=DEV)
    for s in synth_rollout(np.random.default_rng(4), E, T, O, A, p_term=0.05, trunc_len=9):
        buf.add(Batch(**s), buffer_ids=np.arange(E))
    N = E * T
    last = np.arange(E) * T + T - 1
    unf = np.zeros(N, dtype=bool)
    unf[last] = ~buf.done[last]
    roll = dict(obs=buf.obs.copy(), obs_next=buf.obs_next.copy(), act=buf.act.copy(), rew=buf.rew.copy(),
                terminated=buf.terminated.copy(), truncated=buf.truncated.copy(), unfinished=unf)
    np.random.seed(0)
    perms = np.stack([np.random.permutation(N)])
    hp = dict(eps_clip=0.0, dual_clip=None, vf_coef=0.5, ent_coef=0.01, max_grad_norm=0.5, adv_eps=1e-8, value_clip=False,
              advantage_normalization=False, optimizer="rmsprop", lr=lr, alpha=alpha, eps=eps, weight_decay=0.0, loss_kind="a2c")
    res = orm.ppo_update(p, orm.init_state(p, hp), 0, roll, perms, N // 2, 1, hp, None, 0.99, 0.95, False)
    np.random.seed(0)
    with policy_within_training_step(algo.policy):
        algo.update(buffer=buf, batch_size=N // 2, repeat=1)
    record_parity("a2c_rmsprop/wide_layered/loss_table", algo.last_loss_table[:, :4], res["losses"], rtol=2e-3, atol=1e-4)
    for k, pv in named.items():
        record_parity(f"a2c_rmsprop/wide_layered/{k}", pv.detach().cpu().numpy(), p[k], rtol=2e-3,
                      atol=0.05 * _step_bound(lr, alpha))
    assert onp.PARAM_ORDER == PARAM_ORDER


# --------------------------------------------------------------------------------------------- state and refusals
def test_state_dict_round_trip_is_bit_identical():
    """state_dict() -> a fresh algorithm -> load_state_dict() -> the next update equals an uninterrupted run bit for bit; the
    exported state is torch RMSprop's (step, square_avg)."""
    import copy

    from tianshou_b200.utils import policy_within_training_step
    g = load_golden("a2c_rmsprop_ref.npz")
    E, cap, bs, rep = int(g["cfg_E"]), int(g["cfg_cap"]), int(g["cfg_bs"]), int(g["cfg_repeat"])
    a, named_a = _gauss_a2c(g)
    buf = restore_vector_buffer(g, "u0_", E, cap, device=DEV)
    np.random.seed(1000)
    with policy_within_training_step(a.policy):
        a.update(buffer=buf, batch_size=bs, repeat=rep)
    sd = a.state_dict()
    st = sd["_optimizers"][0]["state"]
    assert len(st) == 13 and set(st[0]) == {"step", "square_avg"} and float(st[0]["step"]) == int(g["u0_gradient_steps"])
    b, named_b = _gauss_a2c(g)
    b.load_state_dict(sd)
    b.lr_schedulers[0].load_state_dict(a.lr_schedulers[0].state_dict())
    b.ret_rms = copy.deepcopy(a.ret_rms)
    assert torch.equal(a._flat.exp_avg_sq, b._flat.exp_avg_sq) and torch.equal(a._flat.flat, b._flat.flat)
    buf1 = restore_vector_buffer(g, "u1_", E, cap, device=DEV)
    for x in (a, b):
        np.random.seed(1001)
        with policy_within_training_step(x.policy):
            x.update(buffer=buf1, batch_size=bs, repeat=rep)
    assert torch.equal(a._flat.flat, b._flat.flat) and torch.equal(a._flat.exp_avg_sq, b._flat.exp_avg_sq)


def test_eager_step_then_device_update_matches_torch():
    """An eager ``Algorithm.Optimizer.step(loss)`` (torch's own RMSprop on the module views, clip_grad_norm_ 0.5) matches the
    same step on plain copies of the parameters, its square_avg lands in the flat buffer, and the device update continues
    from it (step count and state carried over)."""
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden("a2c_rmsprop_ref.npz")
    algo, named = _gauss_a2c(g)
    obs = torch.as_tensor(g["u0_buf_obs"][:64], device=DEV)
    copies = {k: p.detach().clone().requires_grad_(True) for k, p in named.items()}
    algo.optim.step(algo.critic(obs).pow(2).mean() + algo.policy.actor(obs)[0][0].pow(2).mean())
    # the same loss on the copies: swap them into the modules' places functionally
    from torch.func import functional_call
    ac = algo._actor_critic
    by_id = {id(p): k for k, p in named.items()}
    params = {n: copies[by_id[id(p)]] for n, p in ac.named_parameters()}
    crit = {n[len("critic."):]: v for n, v in params.items() if n.startswith("critic.")}
    act = {n[len("actor."):]: v for n, v in params.items() if n.startswith("actor.")}
    loss = functional_call(algo.critic, crit, (obs,)).pow(2).mean() + functional_call(algo.policy.actor, act, (obs,))[0][0].pow(2).mean()
    loss.backward()
    torch.nn.utils.clip_grad_norm_(list(copies.values()), 0.5)
    opt = torch.optim.RMSprop(list(copies.values()), lr=float(g["opt_lr"]), eps=float(g["opt_eps"]), alpha=float(g["opt_alpha"]),
                              foreach=False)
    opt.step()
    for k, p in named.items():
        record_parity(f"a2c_rmsprop/eager/{k}", p.detach().cpu().numpy(), copies[k].detach().cpu().numpy(), rtol=1e-6, atol=1e-7)
        if copies[k].grad is None:          # not in this loss (the log-std): torch keeps no state for it, the flat view stays 0
            assert not bool(algo._flat.view(algo._flat.exp_avg_sq, p).any())
            continue
        assert algo.optim._optim.state[p]["square_avg"].data_ptr() == algo._flat.view(algo._flat.exp_avg_sq, p).data_ptr()
        record_parity(f"a2c_rmsprop/eager/{k}_square_avg", algo._flat.view(algo._flat.exp_avg_sq, p).cpu().numpy(),
                      opt.state[copies[k]]["square_avg"].reshape(-1).cpu().numpy(), rtol=1e-5, atol=1e-12)
    assert int(algo._flat.step.item()) == 1
    E, cap = int(g["cfg_E"]), int(g["cfg_cap"])
    buf = restore_vector_buffer(g, "u0_", E, cap, device=DEV)
    np.random.seed(1000)
    with policy_within_training_step(algo.policy):
        algo.update(buffer=buf, batch_size=int(g["cfg_bs"]), repeat=1)
    assert int(algo._flat.step.item()) == 1 + int(g["u0_gradient_steps"]) // int(g["cfg_repeat"])
    st = algo.optim._optim.state[named["a_w1"]]
    assert set(st) == {"step", "square_avg"} and float(st["step"]) == float(algo._flat.step.item())


def _factories():
    from tianshou_b200.algorithm.optim import RMSpropOptimizerFactory, TorchOptimizerFactory
    return {"momentum": RMSpropOptimizerFactory(lr=1e-3, momentum=0.9), "centered": RMSpropOptimizerFactory(lr=1e-3, centered=True),
            "maximize": TorchOptimizerFactory(torch.optim.RMSprop, lr=1e-3, maximize=True)}


@pytest.mark.parametrize("case", ["momentum", "centered", "maximize", "two_groups"])
def test_unsupported_rmsprop_options_are_refused(case):
    from tianshou_b200.algorithm import A2C, ProbabilisticActorPolicy
    from tianshou_b200.algorithm.flat_params import UnsupportedModelError
    from tianshou_b200.algorithm.optim import OptimizerFactory
    actor, critic = build_actor_critic(17, 6, DEV)
    policy = ProbabilisticActorPolicy(actor=actor, dist_fn=gaussian_dist, action_scaling=True, action_bound_method="clip",
                                      action_space=Box(6))

    class TwoGroups(OptimizerFactory):
        def _create_optimizer_for_params(self, params):
            params = list(params)
            return torch.optim.RMSprop([{"params": params[:2]}, {"params": params[2:], "lr": 1e-4}], lr=1e-3)

    factory = TwoGroups() if case == "two_groups" else _factories()[case]
    with pytest.raises(UnsupportedModelError):
        A2C(policy=policy, critic=critic, optim=factory)


def test_gail_discriminator_stays_adam_only():
    """GAIL's actor-critic takes RMSprop (it is a PPO); its discriminator step stays Adam-only."""
    from test_gail_gpu import _nets
    from tianshou_b200.algorithm import GAIL, ProbabilisticActorPolicy
    from tianshou_b200.algorithm.flat_params import UnsupportedModelError
    from tianshou_b200.algorithm.optim import AdamOptimizerFactory, RMSpropOptimizerFactory
    from tianshou_b200.data import ReplayBuffer
    O, A, n = 11, 3, 64
    rng = np.random.default_rng(0)
    term = rng.random(n) < 0.1
    expert = ReplayBuffer.from_data(rng.standard_normal((n, O)).astype(np.float32), rng.standard_normal((n, A)).astype(np.float32),
                                    rng.standard_normal(n), term, np.zeros(n, bool), term,
                                    rng.standard_normal((n, O)).astype(np.float32))

    def build(optim, disc_optim):
        actor, critic, disc = _nets(O, A)
        policy = ProbabilisticActorPolicy(actor=actor, dist_fn=gaussian_dist, action_scaling=True, action_bound_method="clip",
                                          action_space=Box(A))
        return GAIL(policy=policy, critic=critic, optim=optim, expert_buffer=expert, disc_net=disc, disc_optim=disc_optim)

    with pytest.raises(UnsupportedModelError, match="Adam only"):
        build(AdamOptimizerFactory(lr=3e-4), RMSpropOptimizerFactory(lr=1e-3))
    algo = build(RMSpropOptimizerFactory(lr=7e-4, eps=1e-5, alpha=0.99), AdamOptimizerFactory(lr=5e-4))
    assert type(algo.optim._optim) is torch.optim.RMSprop


# --------------------------------------------------------------------------------------------- two ranks
def _free_port() -> int:
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank: int, world_size: int, port: int, path: str, out_dir: str) -> None:
    import torch.distributed as dist

    from tianshou_b200.utils import policy_within_training_step
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world_size),
                      TS_B200_NO_P2P="1" if path == "nccl" else "0")
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world_size, device_id=dev)
    try:
        g = load_golden("a2c_rmsprop_ref.npz")
        algo, named = _gauss_a2c(g, dev)
        for u in range(2):
            o = f"u{u}_"
            buf = restore_vector_buffer(g, o, int(g["cfg_E"]), int(g["cfg_cap"]), device=dev)      # the same shard on both ranks
            np.random.seed(1000 + u)
            with policy_within_training_step(algo.policy):
                stats = algo.update(buffer=buf, batch_size=int(g["cfg_bs"]), repeat=int(g["cfg_repeat"]))
            assert (algo._scratch.get("peer_exchange") is not None) == (path == "p2p"), "wrong multi-GPU path"
            ref_losses = g[o + "losses"]
            np.testing.assert_allclose(stats.loss.mean, ref_losses[:, 0].mean(), rtol=5e-4, atol=2e-5)
            lr = float(g[o + "lr"])
            for k, pv in named.items():
                np.testing.assert_allclose(pv.detach().cpu().numpy(), g[o + "p_" + k], rtol=2e-3,
                                           atol=0.05 * _step_bound(lr, float(g["opt_alpha"])), err_msg=f"rank {rank} u{u} {k}")
        torch.save(algo._flat.flat.cpu(), os.path.join(out_dir, f"flat{rank}.pt"))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("path", ["p2p", "nccl"])
def test_two_rank_rmsprop_update_matches_reference(path, tmp_path):
    """Identical shards on two ranks: the averaged gradient is the single-GPU one, so both multi-GPU paths reproduce the
    reference run, and the replicas stay bit-identical."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    mp.spawn(_worker, args=(2, _free_port(), path, str(tmp_path)), nprocs=2, join=True)
    a, b = torch.load(tmp_path / "flat0.pt"), torch.load(tmp_path / "flat1.pt")
    assert torch.equal(a, b), "replicas diverged"
