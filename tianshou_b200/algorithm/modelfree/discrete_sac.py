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
Every Linear / Conv2d layer's forward, input gradient and weight gradient is one wgmma GEMM launch (csrc/net_gemm.cu).
"""
from __future__ import annotations

from copy import deepcopy
from dataclasses import dataclass
from typing import Any

import numpy as np
import torch
from torch import nn
from torch.distributions import Categorical

from ..._cabi import call, ptr, stream_ptr, to_device
from ...data import Batch, ReplayBuffer
from ..base import OffPolicyAlgorithm, Policy
from ..flat_params import FlatGroup, UnsupportedModelError, bind_optimizer
from ..netgraph import ACT_NONE, FusedStack, _Layer, compile_sequential, module_layers, polyak_update
from ..obs_source import DeviceObsSource, device_obs_source
from ..optim import OptimizerFactory
from .dqn import describe_q_network
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


def describe_discrete_head_network(net: Any, role: str) -> tuple[list[_Layer], list[nn.Parameter], tuple[int, ...], float]:
    """``DiscreteActor`` / ``DiscreteCritic`` -> (layer chain ``module_layers(preprocess) + module_layers(last)``, its
    parameters, input shape, input denominator).  The preprocess net is anything DQN reads: an MLP ``Net`` on flat
    observations or ``DQNet``, optionally behind ``ScaledObsInputActionReprNet``."""
    pre, last = getattr(net, "preprocess", None), getattr(net, "last", None)
    if pre is None or last is None:
        raise UnsupportedModelError(f"{role}: expected a DiscreteActor / DiscreteCritic (preprocess net + last MLP), got "
                                    f"{type(net).__name__}")
    if getattr(pre, "softmax", False):
        raise UnsupportedModelError(f"{role}: a softmax preprocess output is not supported")
    try:
        inner, shape, scale = describe_q_network(pre)
        layers = compile_sequential(module_layers(inner) + module_layers(last), shape)
    except UnsupportedModelError as e:
        raise UnsupportedModelError(f"{role}: {e}") from e
    if layers[-1].kind != "linear" or layers[-1].act != ACT_NONE:
        raise UnsupportedModelError(f"{role}: must end in a linear layer over the actions")
    params = [p for L in layers if L.weight is not None for p in (L.weight, L.bias)]
    return layers, params, shape, scale


class DiscreteSAC(OffPolicyAlgorithm):
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
        devs = {p.device for _, net in nets for p in net.parameters()}
        if len(devs) != 1 or next(iter(devs)).type != "cuda":
            raise UnsupportedModelError(f"networks live on {sorted(map(str, devs))}; tianshou_b200 has no CPU path -- move them to "
                                        "one CUDA device")
        dev = self._dev = next(iter(devs))
        a_layers, a_params, self._in_shape, self._in_scale = describe_discrete_head_network(actor, "actor")
        self.n_actions = a_layers[-1].out_dim
        if self.n_actions != int(policy.action_space.n):
            raise UnsupportedModelError(f"actor has {self.n_actions} outputs for {int(policy.action_space.n)} actions")
        self._g_actor = FlatGroup(a_params, dev)
        self._actor_net = FusedStack(a_layers, self._g_actor, "actor")
        self._g_c, self._c, self._g_ct = [], [], []
        for name, src, tgt in (("critic", self.critic, self.critic_old), ("critic2", self.critic2, self.critic2_old)):
            layers, params, shape, scale = describe_discrete_head_network(src, name)
            if (shape, scale) != (self._in_shape, self._in_scale):
                raise UnsupportedModelError(f"{name} reads the observation as shape {shape} / denominator {scale}, the actor as "
                                            f"{self._in_shape} / {self._in_scale}: the networks must read it the same way")
            if layers[-1].out_dim != self.n_actions:
                raise UnsupportedModelError(f"{name} has {layers[-1].out_dim} outputs for {self.n_actions} actions")
            _, tparams, _, _ = describe_discrete_head_network(tgt, name)
            g = FlatGroup(params, dev)
            self._g_c.append(g)
            self._c.append(FusedStack(layers, g, name))
            self._g_ct.append(FlatGroup(tparams, dev))
        self.policy_optim = self._create_optimizer(policy, policy_optim)
        self.critic_optim = self._create_optimizer(self.critic, critic_optim)
        self.critic2_optim = self._create_optimizer(self.critic2, critic2_optim or critic_optim)
        for o, g in ((self.policy_optim, self._g_actor), (self.critic_optim, self._g_c[0]), (self.critic2_optim, self._g_c[1])):
            bind_optimizer(o, g)
        self._scratch: dict[str, torch.Tensor] = {}

    # ------------------------------------------------------------------ helpers
    def _buf(self, name: str, shape: tuple[int, ...] | int, dtype: torch.dtype = torch.float32) -> torch.Tensor:
        shape = (shape,) if isinstance(shape, int) else tuple(shape)
        t = self._scratch.get(name)
        if t is None or t.shape != shape or t.dtype != dtype:
            t = self._scratch[name] = torch.empty(shape, dtype=dtype, device=self._dev)
        return t

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
        logits = self._actor_net.forward(src.x, B, "tq", frames=src.frames)[-1]
        q = []
        for k in range(2):
            self._g_ct[k].ensure_adopted()
            q.append(self._c[k].forward(src.x, B, "tq", frames=src.frames, params=self._g_ct[k].flat)[-1])
        v, _, _ = self._categorical_rows(logits, q[0], q[1], float(self.alpha.value), "tq", with_grad=False)
        return v

    def _preprocess_batch(self, batch: Batch, buffer: ReplayBuffer, indices: np.ndarray) -> Batch:
        return self.compute_nstep_return(batch=batch, buffer=buffer, indices=indices, target_q_fn=self._target_q,
                                         gamma=self.gamma, n_step=self.n_step_return_horizon)

    def _sample(self, buffer: ReplayBuffer, sample_size: int | None) -> tuple[Batch, Any]:
        """Indices from the buffer's host RNG streams (identical to the reference's draws); observations stay on the device."""
        indices = buffer.sample_indices(sample_size)
        batch = Batch()
        batch.__dict__["obs"] = self._obs_source(buffer, indices, "obs")
        act = np.asarray(buffer.act)[indices]
        batch.__dict__["act"] = to_device(np.ascontiguousarray(act.reshape(-1)).astype(np.int64), self._dev)
        if hasattr(buffer, "get_weight"):          # PrioritizedReplayBuffer.__getitem__ adds the IS weight (prio.py:104-106)
            w = buffer.get_weight(indices)
            batch.__dict__["weight"] = to_device(np.asarray(w / np.max(w) if buffer._weight_norm else w, dtype=np.float32), self._dev)
        batch.__dict__["info"] = Batch()
        return batch, indices

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
        self._g_c[k].adam_step(optim._optim, optim._max_grad_norm)
        return td

    def _update_with_batch(self, batch: Batch) -> DiscreteSACTrainingStats:
        dev, st = self._dev, stream_ptr(self._dev)
        src = batch.obs
        B = src.rows
        weight = batch.__dict__.pop("weight", None)
        if weight is not None:
            if not isinstance(weight, torch.Tensor):
                weight = to_device(np.asarray(weight, dtype=np.float32), dev)
            weight = weight.reshape(-1).to(dev, torch.float32).contiguous()
        returns = batch.returns.reshape(-1).to(dev, torch.float32).contiguous()
        losses = self._buf("losses", 3)
        td1 = self._critic_step(0, src, batch.act, returns, weight, self.critic_optim, losses[0:1])
        td2 = self._critic_step(1, src, batch.act, returns, weight, self.critic2_optim, losses[1:2])
        batch.weight = -(td1 + td2) / 2.0       # prio-buffer: (td1 + td2) / 2 with the reference's td = q - returns

        # actor: loss = -mean(alpha H + sum_a pi(a|s) min(Q1, Q2)(s, a)), the critics after their steps, no gradient into them
        alpha = float(self.alpha.value)
        a_acts = self._actor_net.forward(src.x, B, "au", frames=src.frames)
        q1 = self._c[0].forward(src.x, B, "aq", frames=src.frames)[-1]
        q2 = self._c[1].forward(src.x, B, "aq", frames=src.frames)[-1]
        v, entropy, dlogits = self._categorical_rows(a_acts[-1], q1, q2, alpha, "au", with_grad=True)
        call("ts_mean", ptr(v), B, ptr(losses[2:3]), st)
        self._actor_net.backward(a_acts, dlogits, B, "au")
        self._g_actor.adam_step(self.policy_optim._optim, self.policy_optim._max_grad_norm)

        alpha_loss = self.alpha.update(entropy)
        for k in range(2):                      # _update_lagged_network_weights
            polyak_update(self._g_ct[k], self._g_c[k], self.tau)
        l = losses.cpu().numpy()                # the only host read of the losses
        return DiscreteSACTrainingStats(actor_loss=-float(l[2]), critic1_loss=float(l[0]), critic2_loss=float(l[1]),
                                        alpha=float(self.alpha.value), alpha_loss=alpha_loss)
