"""TD3 (arXiv:1802.09477) with the whole ``update()`` on the device.

Reference: tianshou/algorithm/modelfree/td3.py (TD3TrainingStats :25-29, dual critics :32-102, TD3 :105-226),
modelfree/ddpg.py:196-339 (n-step target, critic squared loss), utils/lagged_network.py:8-80 (Polyak).

Per ``update(buffer, sample_size)``:
  host : index draw (``buffer.sample_indices``: the reference's transitions), the target-policy noise through ``_noise_fn`` on
         EVERY update, one D2H of the losses at the end (2 floats, 3 on an actor step).
  GPU  : row gathers (device mirror or one upload); lagged actor forward -> ``ts_td3_act_rows`` (tanh, max_action, the clamped
         noise, written straight into the lagged critics' [s' | a'] input) -> both lagged critics -> ``ts_td3_target_min`` ->
         ``ts_nstep_return``; per critic forward / weighted MSE / backward + Adam; every ``update_actor_freq``-th update the actor
         step against critic 1 (``ts_td3_act_rows`` -> critic 1 -> ``ts_td3_actor_rows`` -> critic 1's input gradient over the
         action columns -> ``ts_td3_actor_head_bwd`` -> actor backward + Adam) and Polyak of all three lagged networks.
Every Linear layer's forward / input gradient / weight gradient is one wgmma GEMM launch (csrc/net_gemm.cu).  The critic pair,
the row reads, the critic step and the n-step target are ``ContinuousTwinCritic``'s (modelfree/sac.py), shared with SAC and CQL.
"""
from __future__ import annotations

from copy import deepcopy
from dataclasses import dataclass
from typing import Any

import numpy as np
import torch
from torch import nn

from ..._cabi import call, ptr, stream_ptr
from ...data import Batch, ReplayBuffer
from ..base import OffPolicyAlgorithm, TrainingStats, _space_kind
from ..flat_params import UnsupportedModelError
from ..netgraph import ACT_NONE, _Layer
from ..optim import OptimizerFactory
from ..twin_critic import _EvalModeModule, pop_batch_weight
from .ddpg import ContinuousDeterministicPolicy
from .sac import ContinuousTwinCritic, _linear_relu_chain


@dataclass(kw_only=True)
class TD3TrainingStats(TrainingStats):
    actor_loss: float
    critic1_loss: float
    critic2_loss: float


def describe_deterministic_actor(actor: Any, obs_dim: int) -> tuple[list[_Layer], list[nn.Parameter], int]:
    """ContinuousActorDeterministic(preprocess_net=Net(...), hidden_sizes=...) -> the Linear/ReLU chain of ``preprocess`` then
    ``last``, ending in a linear layer of width A (``max_action * tanh`` is applied by the kernels)."""
    if getattr(actor, "max_action", None) is None or not hasattr(actor, "last"):
        raise UnsupportedModelError("TD3 actor: a ContinuousActorDeterministic (preprocess -> last -> max_action * tanh) expected")
    trunk = _linear_relu_chain(actor.preprocess, obs_dim, "actor.preprocess")
    if getattr(actor.preprocess, "softmax", False):
        raise UnsupportedModelError("TD3 actor: softmax trunk output unsupported")
    layers = trunk + _linear_relu_chain(actor.last, trunk[-1].out_dim, "actor.last")
    if layers[-1].act != ACT_NONE:
        raise UnsupportedModelError("TD3 actor: last must end in a Linear layer")
    params: list[nn.Parameter] = []
    for L in layers:
        params += [L.weight, L.bias]
    return layers, params, layers[-1].out_dim


class TD3(ContinuousTwinCritic, OffPolicyAlgorithm):
    """Twin Delayed DDPG (arXiv:1802.09477), reference API (td3.py:105-226).

    The update reproduces what ``TD3._update_with_batch`` computes:

    * the target is ``min(Q1', Q2')(s', a')`` with ``a' = actor_old(s') + clamp(policy_noise * randn, +-noise_clip)`` (the clamp
      skipped when ``noise_clip <= 0``; the noisy action is not clipped back to the action bounds, as in the reference), through
      the n-step return; it is computed, and its noise drawn, on every update;
    * both critics take the weighted-MSE Adam step; ``batch.weight = (td1 + td2) / 2`` feeds a prioritised buffer;
    * on every ``update_actor_freq``-th update (``_cnt % update_actor_freq == 0``, ``_cnt`` counting from 0) the actor steps on
      ``-mean(Q1(s, pi(s)))`` against the UPDATED critic 1 and all three lagged networks move by Polyak; on the other updates
      they stay, and ``actor_loss`` repeats the last actor loss (0.0 before the first).  ``_cnt`` and ``_last`` are not part of
      ``state_dict()``, as in the reference.

    The update reads its losses from the device once, at its end.
    """

    def __init__(self, *, policy: ContinuousDeterministicPolicy, policy_optim: OptimizerFactory, critic: nn.Module,
                 critic_optim: OptimizerFactory, critic2: nn.Module | None = None, critic2_optim: OptimizerFactory | None = None,
                 tau: float = 0.005, gamma: float = 0.99, policy_noise: float = 0.2, update_actor_freq: int = 2,
                 noise_clip: float = 0.5, n_step_return_horizon: int = 1) -> None:
        assert 0.0 <= tau <= 1.0, f"tau should be in [0, 1] but got: {tau}"
        assert 0.0 <= gamma <= 1.0, f"gamma should be in [0, 1] but got: {gamma}"
        super().__init__(policy=policy)
        if _space_kind(policy.action_space) != "continuous":
            raise ValueError(f"TD3 only supports Box action spaces, but got {policy.action_space=}.")
        self.tau = tau
        self.gamma = gamma
        self.n_step_return_horizon = n_step_return_horizon
        self.critic = critic
        self.critic_old = _EvalModeModule(deepcopy(self.critic))
        self.critic2 = critic2 or deepcopy(critic)
        self.critic2_old = _EvalModeModule(deepcopy(self.critic2))
        self.actor_old = _EvalModeModule(deepcopy(self.policy.actor))
        self.policy_noise = policy_noise
        self.update_actor_freq = update_actor_freq
        self.noise_clip = noise_clip
        self._cnt = 0
        self._last = 0
        self._build_networks(lagged=(self.critic_old.module, self.critic2_old.module), lagged_actor=self.actor_old.module,
                             policy_optim=policy_optim, critic_optim=critic_optim, critic2_optim=critic2_optim)
        # target-policy noise: torch.randn on the networks' device, the reference's own call (td3.py:196)
        dev = self._dev
        self._noise_fn = lambda shape: torch.randn(shape, device=dev)

    def _describe_actor(self, actor: nn.Module, obs_dim: int) -> tuple[list[_Layer], list[nn.Parameter], int]:
        return describe_deterministic_actor(actor, obs_dim)

    @property
    def _max_action(self) -> float:
        return float(self.policy.actor.max_action)

    # ------------------------------------------------------------------ target
    def _target_q(self, buffer: ReplayBuffer, indices: np.ndarray) -> torch.Tensor:
        """min(Q1', Q2')(s', actor_old(s') + clamped noise)   (td3.py:94-102, :190-202)"""
        obs_next = self._obs_next_rows(buffer, indices)
        B, A, O = obs_next.shape[0], self.act_dim, self.obs_dim
        st = stream_ptr(self._dev)
        z = self._lagged_actor_forward(obs_next, B, "tq")[-1]
        noise = self._noise_fn((B, A)).to(self._dev, torch.float32).contiguous()
        x = self._buf("tq_x", (B, O + A))
        call("ts_td3_act_rows", ptr(z), ptr(noise), B, A, self._max_action, float(self.policy_noise), float(self.noise_clip),
             ptr(obs_next), O, ptr(x), st)
        q = [self._lagged_forward(k, x, B, "tq")[-1] for k in range(2)]
        out = self._buf("tq_out", (B, 1))
        call("ts_td3_target_min", ptr(q[0]), ptr(q[1]), B, ptr(out), st)
        return out

    # ------------------------------------------------------------------ update
    def _actor_step(self, obs: torch.Tensor, bc_act: torch.Tensor | None, alpha: float, out_loss: torch.Tensor) -> None:
        """The actor step against critic 1 (td3.py:214-219; with ``bc_act`` TD3+BC's, td3_bc.py:113-120): pi(s) written into
        critic 1's input, the loss rows, critic 1's input gradient over the action columns, the tanh head backward, Adam."""
        B, A, O = obs.shape[0], self.act_dim, self.obs_dim
        st = stream_ptr(self._dev)
        a_acts = self._actor.forward(obs, B, "au")
        z = a_acts[-1]
        x = self._buf("aq_x", (B, O + A))
        call("ts_td3_act_rows", ptr(z), None, B, A, self._max_action, 0.0, 0.0, ptr(obs), O, ptr(x), st)
        c_acts = self._c[0].forward(x, B, "aq")
        dq = self._buf("adq", (B, 1))
        call("ts_td3_actor_rows", ptr(c_acts[-1]), ptr(z), ptr(bc_act), B, A, self._max_action, float(alpha), ptr(dq),
             ptr(out_loss), st)
        dact = self._buf("dact", (B, A))
        self._c[0].backward(c_acts, dq, B, "aq", param_grads=False, input_grad=True, input_cols=(O, O + A), dx_out=dact)
        dz = self._buf("dz", (B, A))
        call("ts_td3_actor_head_bwd", ptr(z), ptr(dact), ptr(bc_act), B, A, self._max_action, ptr(dz), st)
        self._actor.backward(a_acts, dz, B, "au")
        self._adam(self._g_actor, self.policy_optim._optim, self.policy_optim._max_grad_norm)

    def _bc_terms(self, batch: Batch) -> tuple[torch.Tensor | None, float]:
        """The behaviour-cloning part of the actor loss: (batch actions, alpha); TD3 has none."""
        return None, 0.0

    def _device_update(self, batch: Batch) -> tuple[torch.Tensor, bool]:
        """Everything of one update after the sampling and the n-step target, with no host synchronisation: both critic steps,
        and on an actor update the actor step and Polyak.  Returns the device losses (critic 1, critic 2, actor) and whether
        the actor stepped."""
        dev = self._dev
        obs, act = batch.obs, batch.act
        B = obs.shape[0]
        returns = batch.returns.reshape(-1).to(dev, torch.float32).contiguous()
        weight = pop_batch_weight(batch, dev)
        losses = self._buf("losses", 3)
        x = self._buf("cu_x", (B, self.obs_dim + self.act_dim))
        self._concat(obs, act, x)
        td1 = self._critic_step(0, x, returns, weight, self.critic_optim, losses[0:1])
        td2 = self._critic_step(1, x, returns, weight, self.critic2_optim, losses[1:2])
        batch.weight = (td1 + td2) / 2.0       # prio-buffer
        actor_step = self._cnt % self.update_actor_freq == 0
        if actor_step:
            bc_act, alpha = self._bc_terms(batch)
            self._actor_step(obs, bc_act, alpha, losses[2:3])
            self._polyak()
        self._cnt += 1
        return losses, actor_step

    def _update_with_batch(self, batch: Batch) -> TD3TrainingStats:
        losses, actor_step = self._device_update(batch)
        l = losses[:3 if actor_step else 2].cpu().numpy()        # the only host read of the update
        if actor_step:
            self._last = float(l[2])
        return TD3TrainingStats(actor_loss=self._last, critic1_loss=float(l[0]), critic2_loss=float(l[1]))
