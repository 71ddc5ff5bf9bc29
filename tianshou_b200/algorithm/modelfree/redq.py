"""REDQ (randomized ensembled double Q-learning, arXiv:2101.05982) with the whole ``update()`` on the device.

Reference: tianshou/algorithm/modelfree/redq.py (REDQTrainingStats :26-31, REDQPolicy :37-131, REDQ :134-304),
modelfree/ddpg.py (ActorCriticOffPolicyAlgorithm: the lagged critic, the n-step target), modelfree/sac.py (Alpha),
utils/net/common.py:518-550 (EnsembleLinear), utils/lagged_network.py:8-80 (Polyak).

Per ``update(buffer, sample_size)``:
  host : index draw (``buffer.sample_indices``), the rsample noise of pi(.|s') (torch, ``_noise_fn``), the subset draw with the
         reference's own ``np.random.choice(E, M, replace=False)`` at the reference's point in the sequence (so numpy's global
         stream, and a prioritised buffer's next draw, stay the reference's), the actor step's rsample noise, one D2H of the
         losses at the end.
  GPU  : row gathers (device mirror or one upload); actor forward + ``ts_squashed_gaussian`` on s' -> the lagged ensemble on
         [s' | a'] -> ``ts_redq_target`` (the subset travels as a launch argument, a member bitmask) -> ``ts_nstep_return``;
         the ensemble forward -> ``ts_redq_critic_rows`` -> backward -> one Adam step over the whole ensemble; every
         ``actor_delay``-th update the actor step against the UPDATED ensemble (``ts_redq_actor_rows``, the ensemble's input
         gradient over the action columns summed over its members, ``ts_squashed_gaussian_bwd``, actor backward + Adam) and
         ``alpha.update``; Polyak of the lagged ensemble on every update.
Every ensemble layer's forward, weight gradient and input gradient is ONE batched wgmma launch over all members
(``ts_net_gemm_batched``); the actor's layers are ``ts_net_gemm`` launches.
"""
from __future__ import annotations

from copy import deepcopy
from dataclasses import dataclass
from typing import Any, Literal

import numpy as np
import torch
from torch import nn
from torch.distributions import Independent, Normal

from ..._cabi import ABI, call, ptr, stream_ptr
from ...data import Batch, ReplayBuffer
from ...exploration import BaseNoise
from ..base import OffPolicyAlgorithm, TrainingStats, _space_kind
from ..flat_params import DeviceScratch, FlatGroup, UnsupportedModelError, bind_optimizer
from ..netgraph import ACT_NONE, FusedStack, _Layer, compile_sequential, layer_params, module_layers, polyak_update
from ..optim import OptimizerFactory
from ..twin_critic import _EvalModeModule, _group_adam_step, cuda_device_of, per_weight, pop_batch_weight
from .ddpg import ContinuousPolicyWithExplorationNoise
from .sac import _F32_EPS, SIGMA_MAX, SIGMA_MIN, Alpha, correct_log_prob_gaussian_tanh, describe_gaussian_actor

TARGET_MODES = {"min": ABI.consts["TS_REDQ_MIN"], "mean": ABI.consts["TS_REDQ_MEAN"]}
MAX_ENSEMBLE = 64          # the subset travels to ts_redq_target as a 64-bit member mask


@dataclass(kw_only=True)
class REDQTrainingStats(TrainingStats):
    actor_loss: float
    critic_loss: float
    alpha: float | None = None
    alpha_loss: float | None = None


class REDQPolicy(ContinuousPolicyWithExplorationNoise):
    """Tanh-squashed Gaussian policy of REDQ (redq.py:37-131).  ``forward`` is the torch-module path the Collector runs."""

    def __init__(self, *, actor: nn.Module, exploration_noise: BaseNoise | Literal["default"] | None = None, action_space: Any,
                 deterministic_eval: bool = True, action_scaling: bool = True,
                 action_bound_method: Literal["clip"] | None = "clip", observation_space: Any | None = None) -> None:
        super().__init__(exploration_noise=exploration_noise, action_space=action_space, observation_space=observation_space,
                         action_scaling=action_scaling, action_bound_method=action_bound_method)
        self.actor = actor
        self.deterministic_eval = deterministic_eval
        self._eps = np.finfo(np.float32).eps.item()

    def forward(self, batch: Batch, state: Any = None, **kwargs: Any) -> Batch:
        (loc, scale), hidden = self.actor(batch.obs, state=state, info=batch.get("info"))
        dist = Independent(Normal(loc, scale), 1)
        act = dist.mode if (self.deterministic_eval and not self.is_within_training_step) else dist.rsample()
        log_prob = dist.log_prob(act).unsqueeze(-1)
        squashed = torch.tanh(act)
        log_prob = correct_log_prob_gaussian_tanh(log_prob, squashed, self._eps)
        return Batch(logits=(loc, scale), act=squashed, state=hidden, dist=dist, log_prob=log_prob)


def describe_ensemble_critic(critic: Any, obs_dim: int, act_dim: int, ensemble_size: int
                             ) -> tuple[list[_Layer], list[nn.Parameter]]:
    """ContinuousCritic(preprocess_net=Net(concat=True, linear_layer=EnsembleLinear), linear_layer=EnsembleLinear,
    flatten_input=False) (test/continuous/test_redq.py:95-109) -> one ensemble chain on concat(obs, act) ending in one output per
    member."""
    if getattr(critic, "apply_preprocess_net_to_obs_only", False):
        raise UnsupportedModelError("REDQ critic: apply_preprocess_net_to_obs_only unsupported")
    if getattr(critic.preprocess, "softmax", False):
        raise UnsupportedModelError("REDQ critic: softmax trunk output unsupported")
    try:
        layers = compile_sequential(module_layers(critic.preprocess) + module_layers(critic.last), (obs_dim + act_dim,),
                                    ensemble=True)
    except UnsupportedModelError as e:
        raise UnsupportedModelError(f"REDQ critic: {e}") from e
    if any(L.kind != "ensemble" for L in layers):
        raise UnsupportedModelError("REDQ critic: every layer must be an EnsembleLinear (linear_layer=EnsembleLinear)")
    if layers[0].E != ensemble_size:
        raise UnsupportedModelError(f"REDQ critic: ensemble of {layers[0].E} members, but ensemble_size={ensemble_size}")
    if layers[-1].out_dim != 1 or layers[-1].act != ACT_NONE:
        raise UnsupportedModelError("REDQ critic must end in a single linear Q output per member")
    return layers, layer_params(layers)


class REDQ(OffPolicyAlgorithm):
    """REDQ, reference API (redq.py:134-304).

    The update reproduces what ``REDQ._update_with_batch`` computes:

    * the target is ``{min | mean}`` over a random ``subset_size`` members of the lagged ensemble at (s', a'), a' ~ pi(.|s'),
      minus ``alpha * log pi(a'|s')``, through the n-step return;
    * the ensemble takes one Adam step on ``mean(td^2 * w)`` over all members and rows; ``batch.weight = mean_e td`` feeds a
      prioritised buffer;
    * on every ``actor_delay``-th update (``critic_gradient_step % actor_delay == 0``, counting from 1) the actor steps on
      ``mean(alpha * log pi - mean_e Q_e(s, a))`` against the updated ensemble, then ``alpha.update``; ``actor_loss`` reports the
      last actor loss (0.0 before the first) and ``alpha_loss`` is None on the other updates;
    * the lagged ensemble moves by Polyak on every update.

    With a fixed alpha the update reads the device once, at its end (the losses).  The critic parameter gradients the
    reference computes in the actor step and then discards are not computed.
    """

    def __init__(self, *, policy: REDQPolicy, policy_optim: OptimizerFactory, critic: nn.Module, critic_optim: OptimizerFactory,
                 ensemble_size: int = 10, subset_size: int = 2, tau: float = 0.005, gamma: float = 0.99,
                 alpha: float | Alpha = 0.2, n_step_return_horizon: int = 1, actor_delay: int = 20,
                 deterministic_eval: bool = True, target_mode: Literal["mean", "min"] = "min") -> None:
        if target_mode not in ("min", "mean"):
            raise ValueError(f"Unsupported target_mode: {target_mode}")
        if not 0 < subset_size <= ensemble_size:
            raise ValueError(f"Invalid choice of ensemble size or subset size. Should be 0 < {subset_size=} <= {ensemble_size=}")
        assert 0.0 <= tau <= 1.0, f"tau should be in [0, 1] but got: {tau}"
        assert 0.0 <= gamma <= 1.0, f"gamma should be in [0, 1] but got: {gamma}"
        super().__init__(policy=policy)
        if _space_kind(policy.action_space) != "continuous":
            raise ValueError(f"REDQ only supports Box action spaces, but got {policy.action_space=}.")
        if ensemble_size > MAX_ENSEMBLE:
            raise UnsupportedModelError(f"REDQ: ensemble_size {ensemble_size} > {MAX_ENSEMBLE} (the subset's member mask)")
        self.tau = tau
        self.gamma = gamma
        self.n_step_return_horizon = n_step_return_horizon
        self.critic = critic
        self.critic_old = _EvalModeModule(deepcopy(self.critic))
        self.ensemble_size = ensemble_size
        self.subset_size = subset_size
        self.target_mode = target_mode
        self.critic_gradient_step = 0
        self.actor_delay = actor_delay
        self.deterministic_eval = deterministic_eval
        self._last_actor_loss = 0.0
        self.alpha = Alpha.from_float_or_instance(alpha)

        dev = self._dev = cuda_device_of(policy.actor, critic)
        actor = policy.actor
        self.obs_dim = int(module_layers(actor.preprocess)[0].in_features)
        a_layers, a_params, self.act_dim = describe_gaussian_actor(actor, self.obs_dim)
        c_layers, c_params = describe_ensemble_critic(critic, self.obs_dim, self.act_dim, ensemble_size)
        _, t_params = describe_ensemble_critic(self.critic_old.module, self.obs_dim, self.act_dim, ensemble_size)
        self._g_actor = FlatGroup(a_params, dev)
        self._actor = FusedStack(a_layers, self._g_actor, "actor")
        self._g_c = FlatGroup(c_params, dev)
        self._c = FusedStack(c_layers, self._g_c, "critic")
        self._g_ct = FlatGroup(t_params, dev)
        self.policy_optim = self._create_optimizer(self.policy, policy_optim)
        self.critic_optim = self._create_optimizer(self.critic, critic_optim)
        bind_optimizer(self.policy_optim, self._g_actor)
        bind_optimizer(self.critic_optim, self._g_c)
        self._scratch = DeviceScratch(dev)
        self._buf = self._scratch.tensor
        self._adam = _group_adam_step           # every Adam step of the update: ``self._adam(group, torch_optimizer, max_grad_norm)``
        # rsample noise source: Normal.rsample's own draw on the networks' device (torch.distributions.utils._standard_normal)
        self._noise_fn = lambda shape: torch.empty(shape, device=dev).normal_()

    # ------------------------------------------------------------------ rows
    def _rows(self, buffer: ReplayBuffer, key: str, indices: np.ndarray) -> torch.Tensor:
        from ... import ops
        return ops.buffer_rows(buffer, key, indices, self._dev).contiguous()

    def _sample(self, buffer: ReplayBuffer, sample_size: int | None) -> tuple[Batch, Any]:
        """Indices from the buffer's host RNG streams (the reference's draws); rows stay on the device."""
        indices = buffer.sample_indices(sample_size)
        batch = Batch()
        batch.__dict__["obs"] = self._rows(buffer, "obs", indices)
        batch.__dict__["act"] = self._rows(buffer, "act", indices)
        weight = per_weight(buffer, indices, self._dev)
        if weight is not None:
            batch.__dict__["weight"] = weight
        batch.__dict__["info"] = Batch()
        return batch, indices

    def _preprocess_batch(self, batch: Batch, buffer: ReplayBuffer, indices: np.ndarray) -> Batch:
        """The n-step return of ``_target_q`` into ``batch.returns`` (ddpg.py:287-302)."""
        return self.compute_nstep_return(batch=batch, buffer=buffer, indices=indices, target_q_fn=self._target_q,
                                         gamma=self.gamma, n_step=self.n_step_return_horizon)

    def _critic_input(self, obs: torch.Tensor, act: torch.Tensor, tag: str) -> torch.Tensor:
        x = self._buf(f"{tag}_x", (obs.shape[0], self.obs_dim + self.act_dim))
        call("ts_concat2", ptr(obs), self.obs_dim, ptr(act), self.act_dim, obs.shape[0], ptr(x), stream_ptr(self._dev))
        return x

    def _actor_forward(self, obs: torch.Tensor, tag: str) -> tuple[list[torch.Tensor], torch.Tensor, torch.Tensor, torch.Tensor,
                                                                  torch.Tensor]:
        """policy(batch) in a training step on the device (redq.py:103-131): (activations, act, log_prob, sigma, noise)."""
        B, A = obs.shape[0], self.act_dim
        acts = self._actor.forward(obs, B, tag)
        noise = self._noise_fn((B, A)).to(self._dev, torch.float32).contiguous()
        act, logp, sigma = self._buf(tag + "_act", (B, A)), self._buf(tag + "_logp", B), self._buf(tag + "_sigma", (B, A))
        call("ts_squashed_gaussian", ptr(acts[-1]), 2 * A, ptr(noise), B, A, SIGMA_MIN, SIGMA_MAX, _F32_EPS, ptr(act), ptr(logp),
             ptr(sigma), stream_ptr(self._dev))
        return acts, act, logp, sigma, noise

    # ------------------------------------------------------------------ target
    def _target_q(self, buffer: ReplayBuffer, indices: np.ndarray) -> torch.Tensor:
        """``_target_q_compute_value`` (redq.py:254-269) on a' ~ pi(.|s')."""
        if buffer._save_obs_next:
            obs_next = self._rows(buffer, "obs_next", indices)
        else:
            obs_next = self._rows(buffer, "obs", buffer.next(indices))
        B = obs_next.shape[0]
        _, act, logp, _, _ = self._actor_forward(obs_next, "tq")
        subset = np.random.choice(self.ensemble_size, self.subset_size, replace=False)    # the reference's call, in its place
        mask = 0
        for e in subset:
            mask |= 1 << int(e)
        x = self._critic_input(obs_next, act, "tq")
        self._g_ct.ensure_adopted()
        q = self._c.forward(x, B, "tq", params=self._g_ct.flat)[-1]
        out = self._buf("tq_out", (B, 1))
        call("ts_redq_target", ptr(q), self.ensemble_size, B, mask, TARGET_MODES[self.target_mode], float(self.alpha.value),
             ptr(logp), ptr(out), stream_ptr(self._dev))
        return out

    # ------------------------------------------------------------------ update
    def _actor_step(self, obs: torch.Tensor, alpha: float, out_loss: torch.Tensor) -> torch.Tensor:
        """The actor step against the ensemble (redq.py:285-289): L = mean(alpha * log pi(a|s) - mean_e Q_e(s, a)) into
        ``out_loss``, the ensemble's input gradient over the action columns (summed over the members), the tanh-Gaussian head
        backward, Adam.  Returns log pi(a|s)."""
        B, A, E = obs.shape[0], self.act_dim, self.ensemble_size
        st = stream_ptr(self._dev)
        a_acts, act, logp, sigma, noise = self._actor_forward(obs, "au")
        c_acts = self._c.forward(self._critic_input(obs, act, "aq"), B, "aq")
        dq, rows = self._buf("adq", (E, B, 1)), self._buf("actor_rows", B)
        call("ts_redq_actor_rows", ptr(c_acts[-1]), ptr(logp), E, B, alpha, ptr(dq), ptr(rows), ptr(out_loss), st)
        dact = self._buf("dact", (B, A))
        self._c.backward(c_acts, dq, B, "aq", param_grads=False, input_grad=True, input_cols=(self.obs_dim, self.obs_dim + A),
                         dx_out=dact)
        dhead = self._buf("dhead", (B, 2 * A))
        call("ts_squashed_gaussian_bwd", ptr(a_acts[-1]), 2 * A, ptr(noise), ptr(act), ptr(sigma), ptr(dact), B, A,
             SIGMA_MIN, SIGMA_MAX, _F32_EPS, alpha / B, ptr(dhead), st)
        self._actor.backward(a_acts, dhead, B, "au")
        self._adam(self._g_actor, self.policy_optim._optim, self.policy_optim._max_grad_norm)
        return logp

    def _update_with_batch(self, batch: Batch) -> REDQTrainingStats:
        dev = self._dev
        obs, act = batch.obs, batch.act
        B, E = obs.shape[0], self.ensemble_size
        returns = batch.returns.reshape(-1).to(dev, torch.float32).contiguous()
        weight = pop_batch_weight(batch, dev)
        losses = self._buf("losses", 2)
        acts = self._c.forward(self._critic_input(obs, act, "cu"), B, "cu")
        td, dq = self._buf("td", (E, B)), self._buf("dq", (E, B, 1))
        row_mean, rows = self._buf("td_mean", B), self._buf("loss_rows", B)
        call("ts_redq_critic_rows", ptr(acts[-1]), ptr(returns), ptr(weight), E, B, ptr(td), ptr(dq), ptr(row_mean), ptr(rows),
             ptr(losses[0:1]), stream_ptr(dev))
        self._c.backward(acts, dq, B, "cu")
        self._adam(self._g_c, self.critic_optim._optim, self.critic_optim._max_grad_norm)
        batch.weight = row_mean.clone()         # prio-buffer
        self.critic_gradient_step += 1

        alpha_loss = None
        actor_step = self.critic_gradient_step % self.actor_delay == 0
        if actor_step:
            logp = self._actor_step(obs, float(self.alpha.value), losses[1:2])
            alpha_loss = self.alpha.update(-logp.detach().unsqueeze(-1))
        polyak_update(self._g_ct, self._g_c, self.tau)
        l = losses[: 2 if actor_step else 1].cpu().numpy()        # the only host read of the update (fixed alpha)
        if actor_step:
            self._last_actor_loss = float(l[1])
        return REDQTrainingStats(actor_loss=self._last_actor_loss, critic_loss=float(l[0]), alpha=float(self.alpha.value),
                                 alpha_loss=alpha_loss)
