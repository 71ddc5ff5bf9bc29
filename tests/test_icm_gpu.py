"""The intrinsic curiosity module on the GPU (algorithm/modelbased/icm.py, csrc/icm.cu): the kernels against float64, ``update()``
of both wrappers against the reference's goldens (tests/golden/icm_ref_*.npz, oracle/gen_golden_icm.py) with the device mirror on
and off, the reference's two quirks (an off-policy wrapped update is the unwrapped one; a wrapped algorithm's scheduler does not
advance), the safety of the buffer's device reward column, a second batch size, the ``state_dict()`` round trip, every refusal,
the reference's own constructions and the register report."""
import copy

import numpy as np
import pytest
import torch

from offpolicy_testutil import (DEV, Discrete, MultiDiscrete, assert_spill_free, ptxas_report, rng_state, set_rng_state, stream,
                                vector_buffer_from_golden)
from oracle import oracle_discrete_sac as ods
from oracle import oracle_icm as oic
from ts_testutil import load_golden, record_parity

pytestmark = pytest.mark.gpu

VARIANTS = ["dqn_mlp", "dqn_per", "dqn_cnn", "ppo_shared", "a2c_sep"]


def _cfg(g):
    return {k[4:]: (g[k].item() if g[k].ndim == 0 else tuple(g[k].tolist())) for k in g.files if k.startswith("cfg_")}


def build(g_or_cfg):
    cfg = _cfg(g_or_cfg) if hasattr(g_or_cfg, "files") else g_or_cfg
    return oic.build(cfg, oic.b200_mods(Discrete), DEV)


def on_policy_buffer(g, mirror):
    from tianshou_b200.data import Batch, VectorReplayBuffer
    E, T = int(g["cfg_E"]), int(g["cfg_steps"])
    buf = VectorReplayBuffer(E * T, E, device=DEV, device_mirror=mirror)
    for i in range(T):
        buf.add(Batch(**{k: g[f"roll{i}_{k}"] for k in ("obs", "act", "rew", "terminated", "truncated", "obs_next")}),
                buffer_ids=np.arange(E))
    return buf


def buffer_for(g, mirror=False):
    return on_policy_buffer(g, mirror) if str(g["cfg_algo"]) in ("ppo", "a2c") else vector_buffer_from_golden(g, mirror)


def run_update(wrapper, buf, g, u):
    from tianshou_b200.utils import policy_within_training_step
    np.random.seed(500 + u)
    with policy_within_training_step(wrapper.policy):
        if str(g["cfg_algo"]) in ("ppo", "a2c"):
            return wrapper.update(buffer=buf, batch_size=int(g["cfg_bs"]), repeat=int(g["cfg_repeat"]))
        return wrapper.update(buffer=buf, sample_size=int(g["cfg_bs"]))


def hook(wrapper, algo):
    """Records per update the indices, the intrinsic reward and (on-policy) the first pass's returns / advantages."""
    cap = {}
    orig = algo._preprocess_batch

    def pre(batch, buffer, indices):
        cap["indices"] = indices.cpu().numpy() if isinstance(indices, torch.Tensor) else np.asarray(indices).copy()
        b = orig(batch, buffer, indices)
        if hasattr(b, "adv") and isinstance(b.adv, torch.Tensor):
            cap["returns"], cap["adv"] = b.returns.double().cpu().numpy(), b.adv.double().cpu().numpy()
        return b

    algo._preprocess_batch = pre
    return cap


def check_group(tag, g, params, group, prefix, lr):
    for i, p in enumerate(params):
        record_parity(f"{tag}/{prefix}pf_{i}", ods.golden_view(p), g[f"{prefix}pf_{i}"], rtol=1e-3, atol=0.1 * lr)
        m, v = g[f"{prefix}m_{i}"], g[f"{prefix}v_{i}"]
        record_parity(f"{tag}/{prefix}m_{i}", ods.golden_view(group.view(group.exp_avg, p)), m, rtol=2e-3,
                      atol=2e-3 * float(np.abs(m).max()) + 1e-12)
        record_parity(f"{tag}/{prefix}v_{i}", ods.golden_view(group.view(group.exp_avg_sq, p)), v, rtol=4e-3,
                      atol=4e-3 * float(np.abs(v).max()) + 1e-20)


# ------------------------------------------------------------------------------------------------------------ kernels
def _rows_fp64(phi, ph, ah, act, B, lr_scale, w, rew, reward_scale):
    r = oic.icm_rows(ph, phi[B:], ah, act, lr_scale, w)
    return r, rew + (r["mse"].astype(np.float32) * np.float32(reward_scale)).astype(np.float64)


@pytest.mark.parametrize("A", [1, 2, 6, 33, 70])
@pytest.mark.parametrize("B", [1, 37, 17000])
@pytest.mark.parametrize("act_f32", [False, True], ids=["i64", "f32"])
def test_icm_kernels_vs_fp64(A, B, act_f32):
    """``ts_icm_inputs``, ``ts_icm_rows`` and ``ts_icm_feature_grad`` against float64 at F = 45 (not a multiple of 32); B = 17000
    is past the row kernel's grid cap, so warps stride over rows."""
    from tianshou_b200._cabi import ABI, call, ptr
    rng = np.random.default_rng(A * 7 + B)
    F_, lr_scale, w, rs = 45, 0.7, 0.3, 0.2
    phi = rng.standard_normal((2 * B, F_)).astype(np.float32)
    ph = rng.standard_normal((B, F_)).astype(np.float32)
    ah = (rng.standard_normal((B, A)) * 3).astype(np.float32)
    act = rng.integers(0, A, B)
    rew = rng.standard_normal(B)
    t = {k: torch.as_tensor(v, device=DEV) for k, v in dict(phi=phi, ph=ph, ah=ah, rew=rew).items()}
    a_dev = torch.as_tensor(act.astype(np.float32 if act_f32 else np.int64), device=DEV)
    fwd_in, inv_in = torch.empty(B, F_ + A, device=DEV), torch.empty(B, 2 * F_, device=DEV)
    call("ts_icm_inputs", ptr(t["phi"]), ptr(a_dev), int(act_f32), B, F_, A, ptr(fwd_in), ptr(inv_in), stream())
    oh = np.eye(A, dtype=np.float32)[act]
    assert np.array_equal(fwd_in.cpu().numpy(), np.concatenate([phi[:B], oh], 1))
    assert np.array_equal(inv_in.cpu().numpy(), np.concatenate([phi[:B], phi[B:]], 1))
    dphi, dfh, dah = torch.full((2 * B, F_), 7.0, device=DEV), torch.empty(B, F_, device=DEV), torch.empty(B, A, device=DEV)
    rows, losses, rew_out = torch.empty(2, B, device=DEV), torch.empty(3, device=DEV), torch.empty(B, dtype=torch.float64, device=DEV)
    out = []
    for _ in range(2):
        call("ts_icm_rows", ptr(t["phi"]), ptr(t["ph"]), ptr(t["ah"]), ptr(a_dev), int(act_f32), B, F_, A, lr_scale, w, ptr(t["rew"]),
             rs, ptr(rew_out), ptr(dphi), ptr(dfh), ptr(dah), ptr(rows), ptr(losses), stream())
        out.append(losses.clone())
    assert torch.equal(out[0], out[1])          # fixed-order sums: bit-identical
    r, want_rew = _rows_fp64(phi, ph, ah, act, B, lr_scale, w, rew, rs)
    np.testing.assert_allclose(losses.cpu().numpy(), [r["loss"], r["forward"], r["inverse"]], rtol=2e-5, atol=1e-6)
    np.testing.assert_allclose(rows.cpu().numpy(), np.stack([r["mse"], r["ce"]]), rtol=2e-5, atol=2e-5)
    np.testing.assert_allclose(dfh.cpu().numpy(), r["d_phi2_hat"], rtol=1e-5, atol=1e-9)
    np.testing.assert_allclose(dah.cpu().numpy(), r["d_act_hat"], rtol=1e-4, atol=1e-9)
    np.testing.assert_allclose(rew_out.cpu().numpy(), want_rew, rtol=1e-6, atol=1e-6)
    assert np.all(dphi[:B].cpu().numpy() == 7.0)         # rows [0, B) are the combine's
    np.testing.assert_allclose(dphi[B:].cpu().numpy(), r["d_phi2"], rtol=1e-5, atol=1e-9)
    dinv = torch.as_tensor(rng.standard_normal((B, 2 * F_)).astype(np.float32), device=DEV)
    dfwd = torch.as_tensor(rng.standard_normal((B, F_)).astype(np.float32), device=DEV)
    for act_kind in (ABI.consts["TS_ACT_NONE"], ABI.consts["TS_ACT_RELU"], ABI.consts["TS_ACT_TANH"]):
        d = dphi.clone()
        y = torch.tanh(t["phi"]) if act_kind == ABI.consts["TS_ACT_TANH"] else t["phi"]
        call("ts_icm_feature_grad", ptr(d), ptr(dinv), ptr(dfwd), ptr(y), act_kind, B, F_, stream())
        want = np.concatenate([dinv[:, :F_].double().cpu().numpy() + dfwd.double().cpu().numpy(),
                               r["d_phi2"] + dinv[:, F_:].double().cpu().numpy()])
        yn = y.double().cpu().numpy()
        want = want * (yn > 0) if act_kind == ABI.consts["TS_ACT_RELU"] else want * (1 - yn * yn) if act_kind == ABI.consts["TS_ACT_TANH"] else want
        np.testing.assert_allclose(d.cpu().numpy(), want, rtol=1e-5, atol=1e-6)


# ------------------------------------------------------------------------------------------------------------ goldens
@pytest.mark.parametrize("mirror", [False, True], ids=["host", "mirror"])
@pytest.mark.parametrize("variant", VARIANTS)
def test_update_matches_reference(variant, mirror):
    g = load_golden(f"icm_ref_{variant}.npz")
    wrapper, algo, icm = build(g)
    buf = buffer_for(g, mirror)
    on_policy = str(g["cfg_algo"]) in ("ppo", "a2c")
    # the reference's keys, plus the ``_actor_critic`` view this package's PPO / A2C already add to their own state_dict()
    keys = [str(k) for k in wrapper.state_dict().keys() if "._actor_critic." not in str(k)]
    assert keys == [str(k) for k in g["state_dict_keys"]]
    cap = hook(wrapper, algo)
    tag = f"icm_{variant}_m{int(mirror)}"
    for u in range(int(g["cfg_updates"])):
        stats = run_update(wrapper, buf, g, u)
        if not on_policy:
            assert np.array_equal(cap["indices"], g[f"u{u}_indices"])
        for k in ("icm_loss", "icm_forward_loss", "icm_inverse_loss"):
            record_parity(f"{tag}_u{u}/{k}", np.array([getattr(stats, k)]), np.array([float(g[f"u{u}_{k}"])]), rtol=1e-4, atol=1e-6)
        want = g[f"u{u}_intrinsic"]
        got = wrapper.icm_reward.cpu().numpy() - (np.asarray(buf.rew)[cap["indices"]] if not on_policy else g_rew(g))
        record_parity(f"{tag}_u{u}/intrinsic", got, want, rtol=1e-4, atol=1e-5 * float(np.abs(want).max()) + 1e-9)
        loss = stats.loss.mean if on_policy else stats.loss
        record_parity(f"{tag}_u{u}/loss", np.array([loss]), np.array([float(g[f"u{u}_loss"])]), rtol=2e-3, atol=1e-5)
        if on_policy and u == 0:
            record_parity(f"{tag}_u0/returns", cap["returns"], g["u0_returns"], rtol=1e-4, atol=1e-5)
            record_parity(f"{tag}_u0/adv", cap["adv"], g["u0_adv"], rtol=1e-4, atol=1e-5)
        np.testing.assert_allclose(wrapper.optim._optim.param_groups[0]["lr"], float(g[f"u{u}_icm_lr"]), rtol=1e-12)
    lr = float(g["cfg_lr"])
    check_group(tag, g, list(icm.parameters()), wrapper._icm_group, "icm_", lr)
    assert wrapper._icm_group.sync_step_from_device() == int(g["icm_adam_step"])
    if not on_policy:
        check_group(tag, g, list(algo.optim._optim.param_groups[0]["params"]), algo._group, "w_", lr)


def g_rew(g):
    """The on-policy rollout's rewards in the order of the buffer's slots (env-major), as ``sample(0)`` of a full buffer reads them."""
    E, T = int(g["cfg_E"]), int(g["cfg_steps"])
    return np.stack([g[f"roll{i}_rew"] for i in range(T)], 1).reshape(E * T)


# ------------------------------------------------------------------------------------------------------------ quirks
def test_off_policy_wrapped_update_is_the_unwrapped_one():
    """Quirk 1: the curiosity reward never reaches the n-step return, so the wrapped DQN's parameters, loss and written-back
    priorities are bit-identical to the same updates without the wrapper."""
    g = load_golden("icm_ref_dqn_per.npz")
    wrapper, algo, _ = build(g)
    _, plain, _ = build(g)
    bufs = [vector_buffer_from_golden(g), vector_buffer_from_golden(g)]
    for u in range(3):
        s1 = run_update(wrapper, bufs[0], g, u)
        s2 = run_update(plain, bufs[1], g, u)
        assert s1.loss == s2.loss
    assert torch.equal(algo._group.flat, plain._group.flat)
    assert np.array_equal(np.asarray(bufs[0].weight[np.arange(bufs[0].maxsize)]), np.asarray(bufs[1].weight[np.arange(bufs[1].maxsize)]))


def test_wrapped_scheduler_does_not_advance():
    """Quirk 2: only the wrapper's schedulers step; the wrapped A2C's own linear schedule stays at its first lr."""
    from tianshou_b200.algorithm import LRSchedulerFactoryLinear
    g = load_golden("icm_ref_a2c_sep.npz")
    cfg = _cfg(g)
    wrapper, algo, _ = build(cfg)
    sched = LRSchedulerFactoryLinear(max_epochs=2, epoch_num_steps=16, collection_step_num_env_steps=16).create_scheduler(
        algo.optim._optim)
    algo.lr_schedulers.append(sched)
    buf = on_policy_buffer(g, False)
    lr0 = algo.optim._optim.param_groups[0]["lr"]
    for u in range(2):
        run_update(wrapper, buf, g, u)
    assert algo.optim._optim.param_groups[0]["lr"] == lr0 and sched.last_epoch == 0
    assert wrapper.optim._optim.param_groups[0]["lr"] < float(cfg["lr"])


@pytest.mark.parametrize("variant", ["ppo_shared", "a2c_sep"])
def test_mirror_reward_column_is_untouched(variant):
    """A full mirrored buffer hands its device reward column to the rollout batch; the curiosity reward goes to a tensor of its
    own, so after the update the device column still equals the host array."""
    g = load_golden(f"icm_ref_{variant}.npz")
    wrapper, _, _ = build(g)
    buf = on_policy_buffer(g, True)
    run_update(wrapper, buf, g, 0)
    cols = buf.device_columns()
    assert cols is not None and np.array_equal(cols["rew"].double().cpu().numpy(), np.asarray(buf.rew, np.float64))


# ------------------------------------------------------------------------------------------------------------ sizes, state
def test_second_batch_size_and_state_dict_round_trip():
    """An update at B = 17 after one at B = 200 equals the B = 17 update of a fresh wrapper loaded from the first one's
    ``state_dict()``, bit for bit, from the same RNG state: the scratch of the larger batch leaks into nothing, and the round trip
    carries the ICM, its Adam moments and the wrapped algorithm with its optimiser."""
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden("icm_ref_dqn_mlp.npz")
    cfg = _cfg(g)
    w1, a1, _ = build(cfg)
    buf = vector_buffer_from_golden(g)
    np.random.seed(1)
    with policy_within_training_step(w1.policy):
        w1.update(buffer=buf, sample_size=200)
    sd = copy.deepcopy(w1.state_dict())
    w2, a2, _ = build(cfg)
    w2.load_state_dict(sd)
    a2._iter = a1._iter          # the reference keeps the update counter outside state_dict()
    state = rng_state(buf)
    outs = []
    for w in (w1, w2):
        set_rng_state(buf, state)
        np.random.seed(2)
        with policy_within_training_step(w.policy):
            outs.append(w.update(buffer=buf, sample_size=17))
    assert outs[0].icm_loss == outs[1].icm_loss and outs[0].loss == outs[1].loss
    for attr in ("flat", "exp_avg", "exp_avg_sq"):
        assert torch.equal(getattr(w1._icm_group, attr), getattr(w2._icm_group, attr))
        assert torch.equal(getattr(a1._group, attr), getattr(a2._group, attr))


# ------------------------------------------------------------------------------------------------------------ refusals
def test_refusals():
    from tianshou_b200.algorithm import AdamOptimizerFactory, ICMOffPolicyWrapper, UnsupportedModelError
    from tianshou_b200.utils.net.common import MLP
    from tianshou_b200.utils.net.discrete import IntrinsicCuriosityModule
    g = load_golden("icm_ref_dqn_mlp.npz")
    cfg = _cfg(g)
    _, algo, _ = build(cfg)

    def icm(feat=None, F_=32, A=3, dev=DEV):
        feat = feat if feat is not None else MLP(input_dim=4, output_dim=F_, hidden_sizes=(32,))
        return IntrinsicCuriosityModule(feature_net=feat, feature_dim=F_, action_dim=A, hidden_sizes=(16,)).to(dev)

    def wrap(model, wrapped=algo):
        return ICMOffPolicyWrapper(wrapped_algorithm=wrapped, model=model, optim=AdamOptimizerFactory(lr=1e-3), lr_scale=1.0,
                                   reward_scale=0.1, forward_loss_weight=0.2)

    with pytest.raises(UnsupportedModelError, match="no CPU path"):
        wrap(icm(dev="cpu"))
    with pytest.raises(UnsupportedModelError, match="action_dim"):
        wrap(icm(A=4))
    with pytest.raises(UnsupportedModelError, match="feature net"):
        wrap(icm(feat=torch.nn.Sequential(torch.nn.Linear(4, 32), torch.nn.Sigmoid())))
    with pytest.raises(UnsupportedModelError, match="feature_dim"):
        wrap(icm(feat=MLP(input_dim=4, output_dim=16), F_=32))
    space = algo.policy.action_space
    algo.policy.action_space = MultiDiscrete([3, 3])
    with pytest.raises(UnsupportedModelError, match="Discrete action space"):
        wrap(icm())
    algo.policy.action_space = space
    algo._seq = True
    with pytest.raises(UnsupportedModelError, match="Recurrent"):
        wrap(icm())
    algo._seq = False
    w = wrap(icm())
    buf = vector_buffer_from_golden(g)
    buf.act[0] = 3
    with pytest.raises(ValueError, match="actions in"):
        from tianshou_b200.utils import policy_within_training_step
        with policy_within_training_step(w.policy):
            np.random.seed(0)
            for _ in range(20):
                w.update(buffer=buf, sample_size=64)
    # on-policy: only PPO / A2C with one rank
    from tianshou_b200.algorithm import ICMOnPolicyWrapper
    gp = load_golden("icm_ref_a2c_sep.npz")
    _, a2c, _ = build(gp)
    a2c._ranks = lambda: (0, 2)
    with pytest.raises(UnsupportedModelError, match="data-parallel"):
        ICMOnPolicyWrapper(wrapped_algorithm=a2c, model=icm(feat=MLP(input_dim=5, output_dim=24), F_=24), optim=AdamOptimizerFactory(lr=1e-3),
                           lr_scale=1.0, reward_scale=0.1, forward_loss_weight=0.2)
    with pytest.raises(UnsupportedModelError, match="PPO and A2C"):
        ICMOnPolicyWrapper(wrapped_algorithm=_npg(), model=icm(), optim=AdamOptimizerFactory(lr=1e-3), lr_scale=1.0, reward_scale=0.1, forward_loss_weight=0.2)


def _npg():
    from tianshou_b200.algorithm import NPG, AdamOptimizerFactory, DiscreteActorPolicy
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.discrete import DiscreteActor, DiscreteCritic
    actor = DiscreteActor(preprocess_net=Net(state_shape=(4,), hidden_sizes=(32,)), action_shape=(3,)).to(DEV)
    critic = DiscreteCritic(preprocess_net=Net(state_shape=(4,), hidden_sizes=(32,))).to(DEV)
    policy = DiscreteActorPolicy(actor=actor, dist_fn=torch.distributions.Categorical, action_space=Discrete(3))
    return NPG(policy=policy, critic=critic, optim=AdamOptimizerFactory(lr=1e-3))


# ------------------------------------------------------------------------------------------------------------ constructions
def test_reference_constructions_take_a_device_update():
    """test_dqn_icm.py, test_ppo_icm.py and atari_dqn.py's ``icm_lr_scale > 0`` branch build here with only their imports changed
    and run one ``update()`` each."""
    from tianshou_b200.algorithm import DQN, PPO, AdamOptimizerFactory, DiscreteActorPolicy, ICMOffPolicyWrapper, ICMOnPolicyWrapper
    from tianshou_b200.algorithm.modelfree.dqn import DiscreteQLearningPolicy
    from tianshou_b200.data import Batch, VectorReplayBuffer
    from tianshou_b200.env.atari.atari_network import DQNet, ScaledObsInputActionReprNet
    from tianshou_b200.utils import policy_within_training_step
    from tianshou_b200.utils.net.common import MLP, Net
    from tianshou_b200.utils.net.discrete import DiscreteActor, DiscreteCritic, IntrinsicCuriosityModule
    rng = np.random.default_rng(0)

    def fill(buf, E, T, obs_shape, A, u8=False):
        for _ in range(T):
            obs = rng.integers(0, 256, (E, *obs_shape), dtype=np.uint8) if u8 else rng.standard_normal((E, *obs_shape)).astype(np.float32)
            buf.add(Batch(obs=obs, act=rng.integers(0, A, E), rew=rng.standard_normal(E), terminated=rng.random(E) < 0.05,
                          truncated=np.zeros(E, bool), obs_next=obs, info=Batch()), buffer_ids=np.arange(E))

    # test_dqn_icm.py: CartPole shapes, hidden [128, 128, 128]
    hs = [128, 128, 128]
    net = Net(state_shape=(4,), action_shape=2, hidden_sizes=hs).to(DEV)
    policy = DiscreteQLearningPolicy(model=net, action_space=Discrete(2), eps_training=0.1, eps_inference=0.05)
    algorithm = DQN(policy=policy, optim=AdamOptimizerFactory(lr=1e-3), gamma=0.9, n_step_return_horizon=3, target_update_freq=320)
    feature_net = MLP(input_dim=4, output_dim=hs[-1], hidden_sizes=hs[:-1])
    icm_net = IntrinsicCuriosityModule(feature_net=feature_net, feature_dim=hs[-1], action_dim=2, hidden_sizes=hs[-1:]).to(DEV)
    icm = ICMOffPolicyWrapper(wrapped_algorithm=algorithm, model=icm_net, optim=AdamOptimizerFactory(lr=1e-3), lr_scale=1.0,
                              reward_scale=0.01, forward_loss_weight=0.2)
    buf = VectorReplayBuffer(2000, 10, device=DEV)
    fill(buf, 10, 100, (4,), 2)
    with policy_within_training_step(icm.policy):
        s = icm.update(buffer=buf, sample_size=64)
    assert np.isfinite([s.icm_loss, s.icm_forward_loss, s.icm_inverse_loss, s.loss]).all()
    # test_ppo_icm.py: one Net shared by actor and critic
    net = Net(state_shape=(4,), hidden_sizes=[64, 64])
    actor = DiscreteActor(preprocess_net=net, action_shape=(2,)).to(DEV)
    critic = DiscreteCritic(preprocess_net=net).to(DEV)
    policy = DiscreteActorPolicy(actor=actor, dist_fn=torch.distributions.Categorical, action_space=Discrete(2), deterministic_eval=True)
    algorithm = PPO(policy=policy, critic=critic, optim=AdamOptimizerFactory(lr=3e-4), gamma=0.99, max_grad_norm=0.5, eps_clip=0.2,
                    vf_coef=0.5, ent_coef=0.0, gae_lambda=0.95, return_scaling=False, dual_clip=None, value_clip=False,
                    advantage_normalization=False, recompute_advantage=False)
    icm_net = IntrinsicCuriosityModule(feature_net=MLP(input_dim=4, output_dim=64, hidden_sizes=[64]), feature_dim=64, action_dim=2,
                                       hidden_sizes=[64]).to(DEV)
    icm = ICMOnPolicyWrapper(wrapped_algorithm=algorithm, model=icm_net, optim=AdamOptimizerFactory(lr=3e-4), lr_scale=1.0,
                             reward_scale=0.01, forward_loss_weight=0.2)
    buf = VectorReplayBuffer(2000, 10, device=DEV)
    fill(buf, 10, 200, (4,), 2)
    with policy_within_training_step(icm.policy):
        s = icm.update(buffer=buf, batch_size=64, repeat=2)
    assert np.isfinite([s.icm_loss, s.loss.mean]).all()
    # atari_dqn.py with icm_lr_scale > 0
    c, h, w, A = 4, 84, 84, 6
    net = ScaledObsInputActionReprNet(DQNet(c=c, h=h, w=w, action_shape=A)).to(DEV)
    policy = DiscreteQLearningPolicy(model=net, action_space=Discrete(A), eps_training=0.1, eps_inference=0.005)
    algorithm = DQN(policy=policy, optim=AdamOptimizerFactory(lr=1e-4), gamma=0.99, n_step_return_horizon=3, target_update_freq=500)
    feat = DQNet(c=c, h=h, w=w, action_shape=A, features_only=True)
    icm_net = IntrinsicCuriosityModule(feature_net=feat.net, feature_dim=feat.output_dim, action_dim=A, hidden_sizes=[512]).to(DEV)
    icm = ICMOffPolicyWrapper(wrapped_algorithm=algorithm, model=icm_net, optim=AdamOptimizerFactory(lr=1e-4), lr_scale=0.01,
                              reward_scale=0.01, forward_loss_weight=0.2)
    buf = VectorReplayBuffer(400, 4, device=DEV, stack_num=4, ignore_obs_next=True, save_only_last_obs=True)
    for _ in range(60):
        fr = rng.integers(0, 256, (4, h, w), dtype=np.uint8)
        st = np.repeat(fr[:, None], 4, axis=1)
        buf.add(Batch(obs=st, act=rng.integers(0, A, 4), rew=rng.standard_normal(4), terminated=rng.random(4) < 0.05,
                      truncated=np.zeros(4, bool), obs_next=st, info=Batch()), buffer_ids=np.arange(4))
    with policy_within_training_step(icm.policy):
        s = icm.update(buffer=buf, sample_size=32)
    assert np.isfinite([s.icm_loss, s.loss]).all()


def test_kernels_have_no_stack_frame_or_spills(tmp_path):
    report = ptxas_report("icm.cu", tmp_path)
    ours = {k: v for k, v in report.items() if "icm" in k}
    assert len(ours) == 4
    assert_spill_free(ours)
