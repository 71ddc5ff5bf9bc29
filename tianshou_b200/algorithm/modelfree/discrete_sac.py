"""Discrete soft actor-critic (arXiv:1910.07207) with the whole ``update()`` on the device.

Reference: tianshou/algorithm/modelfree/discrete_sac.py (DiscreteSACPolicy :31-80, DiscreteSAC :83-196), modelfree/td3.py:40-92
(dual critics, ``critic2=None`` deep-copies the critic), modelfree/ddpg.py:267-339 (n-step target, critic squared loss),
utils/lagged_network.py:8-80 (Polyak).

Per ``update(buffer, sample_size)``:
  host : index draw (uniform: numpy RandomState streams; prioritised: ``np.random.rand`` scalars -- the reference's
         transitions), the two discarded ``Categorical.sample()`` draws of the reference's policy calls (torch generator on
         the device, so it stays in step with a reference run there), one D2H of the three loss scalars.
  GPU  : observation source (dense rows, or uint8 frames + frame slots for the first convolution) of s and s'; actor and both
         lagged critics forward on s' -> ``ts_discrete_sac_rows`` (V(s')) -> value mask + ``ts_nstep_return``; per critic
         forward -> ``ts_dqn_loss`` (gathered weighted MSE) -> backward GEMMs -> Adam; actor forward, both critics forward ->
         ``ts_discrete_sac_rows`` (V(s), H, d loss / d logits) -> actor backward -> Adam; alpha update; Polyak.
Every Linear / Conv2d layer's forward, input gradient and weight gradient is one wgmma GEMM launch (csrc/net_gemm.cu).  The
networks, optimisers, lagged forward and Polyak are the twin-critic core's (twin_critic.py), as for SAC and CQL.
"""
from __future__ import annotations

from copy import deepcopy
from dataclasses import dataclass
from typing import Any

import numpy as np
import torch
from torch import nn
from torch.distributions import Categorical

from ..._cabi import call, ptr, stream_ptr
from ...data import Batch, ReplayBuffer
from ..base import OffPolicyAlgorithm, Policy
from ..discrete_q import describe_discrete_head, sample_discrete
from ..flat_params import UnsupportedModelError
from ..netgraph import ACT_NONE, _Layer, compile_sequential, layer_params, module_layers
from ..obs_source import DeviceObsSource, device_obs_source
from ..optim import OptimizerFactory
from ..twin_critic import TwinCriticAlgorithm, pop_batch_weight
from .sac import Alpha, SACTrainingStats


@dataclass(kw_only=True)
class DiscreteSACTrainingStats(SACTrainingStats):
    pass


def _is_discrete(space: Any) -> bool:
    return getattr(space, "n", None) is not None and type(space).__name__ not in ("MultiBinary", "MultiDiscrete")


class DiscreteSACPolicy(Policy):
    """Categorical policy on the actor's logits (discrete_sac.py:31-80).  ``forward`` is the torch-module path the Collector
    runs: the mode outside a training step with ``deterministic_eval``, a sample otherwise."""

    def __init__(self, *, actor: nn.Module, deterministic_eval: bool = True, action_space: Any,
                 observation_space: Any | None = None) -> None:
        assert _is_discrete(action_space), f"DiscreteSACPolicy needs a Discrete action space, got {action_space}"
        super().__init__(action_space=action_space, observation_space=observation_space)
        self.actor = actor
        self.deterministic_eval = deterministic_eval

    def forward(self, batch: Batch, state: Any = None, **kwargs: Any) -> Batch:
        logits, hidden = self.actor(batch.obs, state=state, info=batch.get("info"))
        dist = Categorical(logits=logits)
        act = dist.mode if (self.deterministic_eval and not self.is_within_training_step) else dist.sample()
        return Batch(logits=logits, act=act, state=hidden, dist=dist)


def _head_chain(net: Any, role: str) -> tuple[list[_Layer], tuple[int, ...], float]:
    """(layer chain ``module_layers(preprocess) + module_layers(last)``, input shape, input denominator) of a
    ``DiscreteActor`` / ``DiscreteCritic`` over the actions."""
    inner, last, shape, scale = describe_discrete_head(net, role)
    try:
        layers = compile_sequential(module_layers(inner) + module_layers(last), shape)
    except UnsupportedModelError as e:
        raise UnsupportedModelError(f"{role}: {e}") from e
    if layers[-1].kind != "linear" or layers[-1].act != ACT_NONE:
        raise UnsupportedModelError(f"{role}: must end in a linear layer over the actions")
    return layers, shape, scale


class DiscreteSAC(TwinCriticAlgorithm, OffPolicyAlgorithm):
    """Soft actor-critic for discrete actions (arXiv:1910.07207), reference API (discrete_sac.py:83-196)."""

    def __init__(self, *, policy: DiscreteSACPolicy, policy_optim: OptimizerFactory, critic: nn.Module,
                 critic_optim: OptimizerFactory, critic2: nn.Module | None = None, critic2_optim: OptimizerFactory | None = None,
                 tau: float = 0.005, gamma: float = 0.99, alpha: float | Alpha = 0.2, n_step_return_horizon: int = 1) -> None:
        assert 0.0 <= tau <= 1.0, f"tau should be in [0, 1] but got: {tau}"
        assert 0.0 <= gamma <= 1.0, f"gamma should be in [0, 1] but got: {gamma}"
        super().__init__(policy=policy)
        actor = policy.actor
        if getattr(actor, "softmax_output", False):
            raise UnsupportedModelError("DiscreteActor(softmax_output=True): discrete SAC reads the actor output as logits, "
                                        "probabilities would be treated as logits; build the actor with softmax_output=False")
        self.tau = tau
        self.gamma = gamma
        self.n_step_return_horizon = n_step_return_horizon
        self.critic = critic
        self.critic_old = deepcopy(critic).eval()
        self.critic2 = critic2 or deepcopy(critic)
        self.critic2_old = deepcopy(self.critic2).eval()
        self.alpha = Alpha.from_float_or_instance(alpha)
        nets = (("actor", actor), ("critic", self.critic), ("critic2", self.critic2))
        # each parameter has one flat storage and one optimiser state: a trunk shared between the networks (atari_sac.py:95-107
        # steps it with three Adam states in turn) cannot be expressed
        owner: dict[int, str] = {}
        for name, net in nets:
            for p in net.parameters():
                if id(p) in owner and owner[id(p)] != name:
                    raise UnsupportedModelError(f"{owner[id(p)]} and {name} share parameters (a common preprocess trunk, as in "
                                                "examples/atari/atari_sac.py); give each network its own trunk")
                owner[id(p)] = name
        self._build_twin_critic(describe_actor=self._describe_actor, describe_critic=self._describe_critic,
                                lagged=(self.critic_old, self.critic2_old), policy_optim=policy_optim, critic_optim=critic_optim,
                                critic2_optim=critic2_optim)

    def _describe_actor(self, actor: nn.Module) -> tuple[list[_Layer], list[nn.Parameter]]:
        layers, self._in_shape, self._in_scale = _head_chain(actor, "actor")
        self.n_actions = layers[-1].out_dim
        if self.n_actions != int(self.policy.action_space.n):
            raise UnsupportedModelError(f"actor has {self.n_actions} outputs for {int(self.policy.action_space.n)} actions")
        return layers, layer_params(layers)

    def _describe_critic(self, net: nn.Module, name: str) -> tuple[list[_Layer], list[nn.Parameter]]:
        """A critic read as the actor reads the observation, one output per action."""
        layers, shape, scale = _head_chain(net, name)
        if (shape, scale) != (self._in_shape, self._in_scale):
            raise UnsupportedModelError(f"{name} reads the observation as shape {shape} / denominator {scale}, the actor as "
                                        f"{self._in_shape} / {self._in_scale}: the networks must read it the same way")
        if layers[-1].out_dim != self.n_actions:
            raise UnsupportedModelError(f"{name} has {layers[-1].out_dim} outputs for {self.n_actions} actions")
        return layers, layer_params(layers)

    # ------------------------------------------------------------------ helpers
    def _obs_source(self, buffer: ReplayBuffer, indices: np.ndarray | torch.Tensor, key: str = "obs") -> DeviceObsSource:
        return device_obs_source(buffer, indices, key, self._in_shape, self._in_scale, self._dev, self._buf)

    def _categorical_rows(self, logits: torch.Tensor, q1: torch.Tensor, q2: torch.Tensor, alpha: float, tag: str,
                          with_grad: bool) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor | None]:
        """(V rows, entropy rows, d(-mean V) / d logits or None) of ``Categorical(logits)`` against min(q1, q2); then the
        reference's discarded ``dist.sample()`` of the same distribution, drawn with torch as ``Categorical.sample`` does."""
        B, A = logits.shape
        v, ent, probs = self._buf(tag + "_v", B), self._buf(tag + "_ent", B), self._buf(tag + "_probs", (B, A))
        dlogits = self._buf(tag + "_dlogits", (B, A)) if with_grad else None
        call("ts_discrete_sac_rows", ptr(logits), ptr(q1), ptr(q2), alpha, B, A, ptr(v), ptr(ent), ptr(probs), ptr(dlogits),
             1.0 / B, stream_ptr(self._dev))
        torch.multinomial(probs, 1, True)
        return v, ent, dlogits

    # ------------------------------------------------------------------ target
    def _target_q(self, buffer: ReplayBuffer, indices: np.ndarray) -> torch.Tensor:
        """sum_a pi(a|s') min(Q1', Q2')(s', a) + alpha H(pi(.|s'))   (discrete_sac.py:147-155, ddpg.py:327-339)"""
        src = self._obs_source(buffer, indices, "obs_next")
        B = src.rows
        logits = self._actor.forward(src.x, B, "tq", frames=src.frames)[-1]
        q = [self._lagged_forward(k, src.x, B, "tq", frames=src.frames)[-1] for k in range(2)]
        v, _, _ = self._categorical_rows(logits, q[0], q[1], float(self.alpha.value), "tq", with_grad=False)
        return v

    def _preprocess_batch(self, batch: Batch, buffer: ReplayBuffer, indices: np.ndarray) -> Batch:
        return self.compute_nstep_return(batch=batch, buffer=buffer, indices=indices, target_q_fn=self._target_q,
                                         gamma=self.gamma, n_step=self.n_step_return_horizon)

    def _sample(self, buffer: ReplayBuffer, sample_size: int | None) -> tuple[Batch, Any]:
        return sample_discrete(buffer, sample_size, self._obs_source, self._dev, self.n_actions)

    # ------------------------------------------------------------------ update
    def _critic_step(self, k: int, src: DeviceObsSource, act: torch.Tensor, returns: torch.Tensor, weight: torch.Tensor | None,
                     optim: Any, out_loss: torch.Tensor) -> torch.Tensor:
        """Q_k(s).gather(act), weighted squared error, backward, Adam (discrete_sac.py:162-172).  ``ts_dqn_loss`` returns
        td = returns - q, the negative of the reference's td."""
        B, A = src.rows, self.n_actions
        st = stream_ptr(self._dev)
        acts = self._c[k].forward(src.x, B, "cu", frames=src.frames)
        td = self._buf(f"td{k}", B)
        dq = self._buf("dq", (B, A))
        rows = self._buf("loss_rows", B)
        call("ts_dqn_loss", ptr(acts[-1]), ptr(act), ptr(returns), ptr(weight), B, A, 0.0, ptr(td), ptr(dq), ptr(rows), st)
        call("ts_mean", ptr(rows), B, ptr(out_loss), st)
        self._c[k].backward(acts, dq, B, "cu")
        self._adam(self._g_c[k], optim._optim, optim._max_grad_norm)
        return td

    def _update_with_batch(self, batch: Batch) -> DiscreteSACTrainingStats:
        dev, st = self._dev, stream_ptr(self._dev)
        src = batch.obs
        B = src.rows
        weight = pop_batch_weight(batch, dev)
        returns = batch.returns.reshape(-1).to(dev, torch.float32).contiguous()
        losses = self._buf("losses", 3)
        td1 = self._critic_step(0, src, batch.act, returns, weight, self.critic_optim, losses[0:1])
        td2 = self._critic_step(1, src, batch.act, returns, weight, self.critic2_optim, losses[1:2])
        batch.weight = -(td1 + td2) / 2.0       # prio-buffer: (td1 + td2) / 2 with the reference's td = q - returns

        # actor: loss = -mean(alpha H + sum_a pi(a|s) min(Q1, Q2)(s, a)), the critics after their steps, no gradient into them
        alpha = float(self.alpha.value)
        a_acts = self._actor.forward(src.x, B, "au", frames=src.frames)
        q1 = self._c[0].forward(src.x, B, "aq", frames=src.frames)[-1]
        q2 = self._c[1].forward(src.x, B, "aq", frames=src.frames)[-1]
        v, entropy, dlogits = self._categorical_rows(a_acts[-1], q1, q2, alpha, "au", with_grad=True)
        call("ts_mean", ptr(v), B, ptr(losses[2:3]), st)
        self._actor.backward(a_acts, dlogits, B, "au")
        self._adam(self._g_actor, self.policy_optim._optim, self.policy_optim._max_grad_norm)

        alpha_loss = self.alpha.update(entropy)
        self._polyak()
        l = losses.cpu().numpy()                # the only host read of the losses
        return DiscreteSACTrainingStats(actor_loss=-float(l[2]), critic1_loss=float(l[0]), critic2_loss=float(l[1]),
                                        alpha=float(self.alpha.value), alpha_loss=alpha_loss)
