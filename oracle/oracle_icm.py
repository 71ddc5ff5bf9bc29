"""TEST INFRASTRUCTURE -- float64 restatement of the intrinsic curiosity module's update, and the construction of the ICM goldens'
algorithms from either the reference's modules or tianshou_b200's.

Only ``tests/`` and ``tools/`` may import this module; ``tianshou_b200`` never does.  It restates
tianshou/algorithm/modelbased/icm.py:77-109 and utils/net/discrete.py:418-428 without the framework around them:

* ``phi1 = f(s)``, ``phi2 = f(s')``; ``mse = 0.5 * sum_j (forward_model([phi1 | one_hot(a)]) - phi2)^2`` per row;
  ``act_hat = inverse_model([phi1 | phi2])``;
* intrinsic reward ``mse * reward_scale`` (fp32 in the reference, added to the float64 reward);
* ``loss = ((1 - w) CE(act_hat, a) + w mean(mse)) * lr_scale``, the gradient at phi2_hat and act_hat written out by hand, phi2
  NOT detached (the forward loss reaches the feature net through both halves), then torch's Adam on a float64 copy.

The ICM's update does not depend on the wrapped algorithm (off-policy the curiosity reward never reaches the n-step return; on-policy
the ICM reads only observations and actions), so the restatement replays the batches a golden captured.

PINNING: tests/test_oracle_icm.py replays tests/golden/icm_ref_*.npz (oracle/gen_golden_icm.py) through ``icm_update``.
"""
from __future__ import annotations

import numpy as np
import torch
from torch import nn

from oracle.oracle_discrete_sac import seeded_params


def icm_rows(phi2_hat: np.ndarray, phi2: np.ndarray, act_hat: np.ndarray, act: np.ndarray, lr_scale: float, w: float) -> dict:
    """Per-row losses, the three losses and the gradients at phi2_hat, act_hat and (directly) phi2."""
    phi2_hat, phi2, act_hat = (np.asarray(x, np.float64) for x in (phi2_hat, phi2, act_hat))
    B, A = act_hat.shape
    a = np.asarray(act).reshape(-1).astype(np.int64)
    d = phi2_hat - phi2
    mse = 0.5 * (d * d).sum(1)
    m = act_hat.max(1, keepdims=True)
    lse = m[:, 0] + np.log(np.exp(act_hat - m).sum(1))
    ce = lse - act_hat[np.arange(B), a]
    fwd, inv = mse.mean(), ce.mean()
    hit = np.zeros((B, A))
    hit[np.arange(B), a] = 1.0
    g_fwd = lr_scale * w / B * d
    g_inv = lr_scale * (1 - w) / B * (np.exp(act_hat - lse[:, None]) - hit)
    return dict(mse=mse, ce=ce, forward=fwd, inverse=inv, loss=((1 - w) * inv + w * fwd) * lr_scale, d_phi2_hat=g_fwd,
                d_act_hat=g_inv, d_phi2=-g_fwd)


class ICMState:
    """A float64 copy of the ICM module and torch's Adam over its parameters, in ``parameters()`` order."""

    def __init__(self, model: nn.Module, lr: float) -> None:
        self.model = model.double()
        self.params = list(model.parameters())
        self.opt = torch.optim.Adam(self.params, lr=lr)


def _seq(mod: nn.Module) -> nn.Module:
    """The layer chain of an ``MLP`` (its ``model``) or a plain Sequential, run in the dtype of its parameters."""
    return mod if isinstance(mod, nn.Sequential) else mod.model


def icm_update(s: ICMState, obs: np.ndarray, act: np.ndarray, obs_next: np.ndarray, lr_scale: float, reward_scale: float, w: float,
               detach_phi2: bool = False, lr_scale_as_lr: bool = False) -> dict:
    """One ICM step on a batch as the reference's buffer delivered it (uint8 frames read as their values).  ``detach_phi2`` and
    ``lr_scale_as_lr`` are the two misreadings the tests show to be measurable: phi2 as a constant, and lr_scale multiplying the
    learning rate instead of the loss."""
    m = s.model
    A = m.action_dim
    x1 = torch.as_tensor(np.asarray(obs)).double()
    x2 = torch.as_tensor(np.asarray(obs_next)).double()
    a = torch.as_tensor(np.asarray(act).reshape(-1).astype(np.int64))
    f = _seq(m.feature_net)
    phi1, phi2 = f(x1), f(x2)
    oh = torch.nn.functional.one_hot(a, A).double()
    phi2_hat = _seq(m.forward_model)(torch.cat([phi1, oh], 1))
    act_hat = _seq(m.inverse_model)(torch.cat([phi1, phi2], 1))
    scale = 1.0 if lr_scale_as_lr else lr_scale
    r = icm_rows(phi2_hat.detach().numpy(), phi2.detach().numpy(), act_hat.detach().numpy(), act, scale, w)
    s.opt.zero_grad()
    outs = [phi2_hat, act_hat] + ([] if detach_phi2 else [phi2])
    grads = [torch.as_tensor(r["d_phi2_hat"]), torch.as_tensor(r["d_act_hat"])] + ([] if detach_phi2 else [torch.as_tensor(r["d_phi2"])])
    torch.autograd.backward(outs, grads)
    if lr_scale_as_lr:
        for pg in s.opt.param_groups:
            pg["lr_saved"], pg["lr"] = pg["lr"], pg["lr"] * lr_scale
    s.opt.step()
    if lr_scale_as_lr:
        for pg in s.opt.param_groups:
            pg["lr"] = pg.pop("lr_saved")
    r["loss"] = r["loss"] if not lr_scale_as_lr else ((1 - w) * r["inverse"] + w * r["forward"]) * lr_scale
    r["intrinsic"] = (r["mse"] * reward_scale)
    return r


# ------------------------------------------------------------------------------------------------------------ constructions
def build(cfg: dict, mods: dict, device: str = "cpu"):
    """The wrapper of a golden variant built from ``mods`` (the reference's classes, or tianshou_b200's under the same names), every
    network seeded by ``seeded_params``.  Returns (wrapper, wrapped algorithm, ICM module)."""
    A = int(cfg["A"])
    space = mods["Discrete"](A)
    Adam = mods["AdamOptimizerFactory"]
    on_policy = cfg["algo"] in ("ppo", "a2c")
    if cfg["kind"] == "cnn":
        H = int(cfg["H"])
        qnet = mods["ScaledObsInputActionReprNet"](mods["DQNet"](c=4, h=H, w=H, action_shape=A))
        feat_mod = mods["DQNet"](c=4, h=H, w=H, action_shape=A, features_only=True)
        F = int(feat_mod.output_dim)
        feature_net = feat_mod.net
    else:
        obs = int(cfg["obs"])
        F = int(cfg["F"])
        feature_net = mods["MLP"](input_dim=obs, output_dim=F, hidden_sizes=tuple(cfg["feat_hidden"]))
    icm = mods["IntrinsicCuriosityModule"](feature_net=feature_net, feature_dim=F, action_dim=A, hidden_sizes=tuple(cfg["icm_hidden"]))
    seeded_params(icm, int(cfg["icm_seed"]))
    icm.to(device)
    if on_policy:
        Net = mods["Net"]
        hidden = tuple(cfg["hidden"])
        net = Net(state_shape=(obs,), hidden_sizes=hidden)
        net_c = net if bool(cfg["shared"]) else Net(state_shape=(obs,), hidden_sizes=hidden)
        actor = mods["DiscreteActor"](preprocess_net=net, action_shape=(A,))
        critic = mods["DiscreteCritic"](preprocess_net=net_c)
        seeded_params(nn.ModuleList([actor, critic]), int(cfg["init_seed"]))
        actor.to(device), critic.to(device)
        policy = mods["DiscreteActorPolicy"](actor=actor, dist_fn=torch.distributions.Categorical, action_space=space,
                                             deterministic_eval=True)
        if cfg["algo"] == "ppo":
            algo = mods["PPO"](policy=policy, critic=critic, optim=Adam(lr=float(cfg["lr"])), gamma=0.99, max_grad_norm=0.5,
                               eps_clip=0.2, vf_coef=0.5, ent_coef=0.0, gae_lambda=0.95, return_scaling=False, dual_clip=None,
                               value_clip=False, advantage_normalization=False, recompute_advantage=True)
        else:
            algo = mods["A2C"](policy=policy, critic=critic, optim=Adam(lr=float(cfg["lr"])), gamma=0.99, max_grad_norm=0.5,
                               vf_coef=0.5, ent_coef=0.01, gae_lambda=0.95, return_scaling=False)
        icm_optim = Adam(lr=float(cfg["lr"]))
        if bool(cfg.get("sched", False)):
            icm_optim = icm_optim.with_lr_scheduler_factory(mods["LRSchedulerFactoryLinear"](max_epochs=4, epoch_num_steps=64,
                                                                                              collection_step_num_env_steps=16))
        wrapper = mods["ICMOnPolicyWrapper"](wrapped_algorithm=algo, model=icm, optim=icm_optim, lr_scale=float(cfg["lr_scale"]),
                                             reward_scale=float(cfg["reward_scale"]), forward_loss_weight=float(cfg["w"]))
        return wrapper, algo, icm
    if cfg["kind"] != "cnn":
        qnet = mods["Net"](state_shape=(obs,), action_shape=A, hidden_sizes=tuple(cfg["hidden"]))
    seeded_params(qnet, int(cfg["init_seed"]))
    qnet.to(device)
    policy = mods["DiscreteQLearningPolicy"](model=qnet, action_space=space, eps_training=0.1, eps_inference=0.05)
    algo = mods["DQN"](policy=policy, optim=Adam(lr=float(cfg["lr"])), gamma=0.9, n_step_return_horizon=int(cfg["n_step"]),
                       target_update_freq=int(cfg["freq"]))
    wrapper = mods["ICMOffPolicyWrapper"](wrapped_algorithm=algo, model=icm, optim=Adam(lr=float(cfg["lr"])),
                                          lr_scale=float(cfg["lr_scale"]), reward_scale=float(cfg["reward_scale"]),
                                          forward_loss_weight=float(cfg["w"]))
    return wrapper, algo, icm


def reference_mods() -> dict:
    """The reference's classes ``build`` reads (after oracle.ref_shim.import_reference())."""
    from gymnasium.spaces import Discrete
    from tianshou.algorithm import A2C, DQN, PPO, ICMOffPolicyWrapper, ICMOnPolicyWrapper
    from tianshou.algorithm.modelfree.dqn import DiscreteQLearningPolicy
    from tianshou.algorithm.modelfree.reinforce import DiscreteActorPolicy
    from tianshou.algorithm.optim import AdamOptimizerFactory, LRSchedulerFactoryLinear
    from tianshou.env.atari.atari_network import DQNet, ScaledObsInputActionReprNet
    from tianshou.utils.net.common import MLP, Net
    from tianshou.utils.net.discrete import DiscreteActor, DiscreteCritic, IntrinsicCuriosityModule
    return dict(locals())


def b200_mods(Discrete) -> dict:
    """tianshou_b200's classes under the same names; ``Discrete`` is the test's action-space stand-in."""
    from tianshou_b200.algorithm import A2C, DQN, PPO, AdamOptimizerFactory, ICMOffPolicyWrapper, ICMOnPolicyWrapper, LRSchedulerFactoryLinear
    from tianshou_b200.algorithm.modelfree.dqn import DiscreteQLearningPolicy
    from tianshou_b200.algorithm.modelfree.reinforce import DiscreteActorPolicy
    from tianshou_b200.env.atari.atari_network import DQNet, ScaledObsInputActionReprNet
    from tianshou_b200.utils.net.common import MLP, Net
    from tianshou_b200.utils.net.discrete import DiscreteActor, DiscreteCritic, IntrinsicCuriosityModule
    return dict(locals())
