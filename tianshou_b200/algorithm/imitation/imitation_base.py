"""Imitation learning (behavioural cloning) with the whole ``update()`` on the device.

Reference: tianshou/algorithm/imitation/imitation_base.py:32-183 (ImitationTrainingStats, ImitationPolicy, the
``_imitation_update`` of OffPolicyImitationLearning and OfflineImitationLearning), utils/net/continuous.py
(ContinuousActorDeterministic), utils/net/discrete.py:29-90 (DiscreteActor, ``softmax_output=True`` by default),
algorithm_base.py:562-584 (a prioritised buffer's ``batch.weight`` written back as the new priorities).

Per ``update(buffer, sample_size)``:
  host : index draw (``buffer.sample_indices``: the reference's draws), the range check of drawn discrete actions, one D2H of
         the loss.
  GPU  : the observation rows (continuous: ``ops.buffer_rows``; discrete: ``device_obs_source``, dense rows or the uint8 frames
         the first convolution reads) and the action rows -> the actor's GEMM chain -> ``ts_imitation_mse_rows`` /
         ``ts_imitation_nll_rows`` (loss, gradient at the last Linear's output) -> the backward GEMMs of the parameter gradients
         -> one Adam step over the flat group.
There is no lagged network, no n-step return and no importance weight in the loss.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Any, Literal

import numpy as np
from torch import nn

from ... import ops
from ..._cabi import call, ptr, stream_ptr
from ...data import Batch, ReplayBuffer
from ..base import OfflineAlgorithm, OffPolicyAlgorithm, Policy, TrainingStats
from ..discrete_q import describe_discrete_head, describe_q_network, sample_discrete
from ..flat_params import DeviceScratch, FlatGroup, UnsupportedModelError, bind_optimizer
from ..modelfree.td3 import describe_deterministic_actor
from ..netgraph import ACT_NONE, FusedStack, compile_sequential, layer_params, module_layers
from ..obs_source import DeviceObsSource, device_obs_source
from ..optim import OptimizerFactory
from ..twin_critic import cuda_device_of, per_weight


@dataclass(kw_only=True)
class ImitationTrainingStats(TrainingStats):
    loss: float = 0.0


class ImitationPolicy(Policy):
    """The actor's output as the action (imitation_base.py:37-105).  ``forward`` is the torch-module path the Collector runs:
    discrete, the arg-max of the output; continuous, the output itself."""

    def __init__(self, *, actor: nn.Module, action_space: Any, observation_space: Any | None = None, action_scaling: bool = False,
                 action_bound_method: Literal["clip", "tanh"] | None = "clip") -> None:
        super().__init__(action_space=action_space, observation_space=observation_space, action_scaling=action_scaling,
                         action_bound_method=action_bound_method)
        self.actor = actor

    def forward(self, batch: Batch, state: Any = None, **kwargs: Any) -> Batch:
        out, hidden = self.actor(batch.obs, state=state, info=batch.get("info"))
        if self.action_type == "discrete":
            return Batch(logits=out, act=out.argmax(dim=1), state=hidden)
        return Batch(logits=out, act=out, state=hidden)


def _continuous_actor(actor: Any, act_dim: int) -> tuple[list, list[nn.Parameter], float]:
    """A ContinuousActorDeterministic over an MLP ``Net``: (layer chain ending in the Linear of width ``act_dim``, parameters in
    flat order, max_action)."""
    if hasattr(actor, "mu"):
        raise UnsupportedModelError("imitation actor: a probabilistic actor (mu, sigma) is not supported; the reference's "
                                    "regression loss takes the actor's output as the action")
    pre = getattr(actor, "preprocess", None)
    first = module_layers(pre)[0] if pre is not None else None
    if not isinstance(first, nn.Linear):
        raise UnsupportedModelError(f"imitation actor: a ContinuousActorDeterministic over an MLP Net expected, got "
                                    f"{type(actor).__name__}")
    try:
        layers, params, A = describe_deterministic_actor(actor, int(first.in_features))
    except UnsupportedModelError as e:
        raise UnsupportedModelError(f"imitation actor: {e}") from e
    if A != act_dim:
        raise UnsupportedModelError(f"imitation actor: {A} outputs for an action of dimension {act_dim}")
    return layers, params, float(actor.max_action)


def _discrete_actor(actor: Any, n_actions: int) -> tuple[list, tuple[int, ...], float, bool]:
    """A ``DiscreteActor`` (either ``softmax_output``), or a plain chain ending in ``Linear(., n_actions)`` without activation
    (``Net(action_shape=n)``, ``DQNet``, optionally behind ``ScaledObsInputActionReprNet``): (layer chain, input shape, input
    denominator, whether the network's output is the softmax of the chain's)."""
    if hasattr(actor, "preprocess") and hasattr(actor, "last"):
        inner, last, shape, scale = describe_discrete_head(actor, "imitation actor")
        mods, softmax_output = module_layers(inner) + module_layers(last), bool(getattr(actor, "softmax_output", False))
    else:
        inner, shape, scale = describe_q_network(actor)
        if getattr(inner, "softmax", False):
            raise UnsupportedModelError("imitation actor: a Net with softmax=True is not supported; use DiscreteActor for "
                                        "probabilities")
        mods, softmax_output = module_layers(inner), False
    layers = compile_sequential(mods, shape)
    if layers[-1].kind != "linear" or layers[-1].act != ACT_NONE:
        raise UnsupportedModelError("imitation actor: the network must end in a linear layer over the actions")
    if layers[-1].out_dim != n_actions:
        raise UnsupportedModelError(f"imitation actor: {layers[-1].out_dim} outputs for {n_actions} actions")
    return layers, shape, scale, softmax_output


class ImitationLearningAlgorithmMixin:
    """The device update of both trainer bases (imitation_base.py:108-127): the subclass creates ``self.optim`` over the policy,
    then calls ``_build_device_update``."""

    policy: ImitationPolicy
    optim: Any

    def _build_device_update(self) -> None:
        actor = self.policy.actor
        dev = self._dev = cuda_device_of(actor)
        self._continuous = self.policy.action_type == "continuous"
        if self._continuous:
            self.n_out = int(np.prod(self.policy.action_space.shape))
            layers, params, self._max_action = _continuous_actor(actor, self.n_out)
            self._obs_dim = layers[0].in_dim
        else:
            self.n_out = int(self.policy.action_space.n)
            layers, self._in_shape, self._in_scale, self._softmax_output = _discrete_actor(actor, self.n_out)
            params = layer_params(layers)
        self._group = FlatGroup(params, dev)
        self._net = FusedStack(layers, self._group, "actor")
        bind_optimizer(self.optim, self._group)
        self._scratch = DeviceScratch(dev)
        self._buf = self._scratch.tensor

    # ------------------------------------------------------------------ sampling
    def _obs_source(self, buffer: ReplayBuffer, indices: np.ndarray, key: str) -> DeviceObsSource:
        return device_obs_source(buffer, indices, key, self._in_shape, self._in_scale, self._dev, self._buf)

    def _sample(self, buffer: ReplayBuffer, sample_size: int | None) -> tuple[Batch, Any]:
        """The buffer's index draw; observations and actions as device rows, a prioritised sample's importance weight as
        ``batch.weight`` (it stays on the batch and becomes the new priorities, as in the reference)."""
        if not self._continuous:
            return sample_discrete(buffer, sample_size, self._obs_source, self._dev, self.n_out)
        indices = buffer.sample_indices(sample_size)
        obs = ops.buffer_rows(buffer, "obs", indices, self._dev).contiguous()
        act = ops.buffer_rows(buffer, "act", indices, self._dev).contiguous()
        if obs.shape[1] != self._obs_dim:
            raise UnsupportedModelError(f"the buffer holds observation rows of width {obs.shape[1]}, the actor reads {self._obs_dim}")
        if act.shape[1] != self.n_out:
            raise UnsupportedModelError(f"the buffer holds action rows of width {act.shape[1]}, the actor has {self.n_out} outputs")
        batch = Batch()
        batch.__dict__["obs"], batch.__dict__["act"] = obs, act
        weight = per_weight(buffer, indices, self._dev)
        if weight is not None:
            batch.__dict__["weight"] = weight
        batch.__dict__["info"] = Batch()
        return batch, indices

    # ------------------------------------------------------------------ update
    def _update_with_batch(self, batch: Batch) -> ImitationTrainingStats:
        st = stream_ptr(self._dev)
        A = self.n_out
        loss = self._buf("loss", 1)
        if self._continuous:
            B = batch.obs.shape[0]
            acts = self._net.forward(batch.obs, B, "up")
            dz = self._buf("dz", (B, A))
            call("ts_imitation_mse_rows", ptr(acts[-1]), ptr(batch.act), B, A, self._max_action, ptr(dz), ptr(loss), st)
        else:
            src = batch.obs
            B = src.rows
            acts = self._net.forward(src.x, B, "up", frames=src.frames)
            dz, rows = self._buf("dz", (B, A)), self._buf("loss_rows", B)
            call("ts_imitation_nll_rows", ptr(acts[-1]), ptr(batch.act), B, A, int(self._softmax_output), ptr(dz), ptr(rows), ptr(loss),
                 st)
        self._net.backward(acts, dz, B, "up")
        self._group.adam_step(self.optim._optim, self.optim._max_grad_norm)
        return ImitationTrainingStats(loss=float(loss.item()))       # the only host read of the update


class OffPolicyImitationLearning(ImitationLearningAlgorithmMixin, OffPolicyAlgorithm):
    """Off-policy vanilla imitation learning (imitation_base.py:130-155)."""

    def __init__(self, *, policy: ImitationPolicy, optim: OptimizerFactory) -> None:
        super().__init__(policy=policy)
        self.optim = self._create_optimizer(self.policy, optim)
        self._build_device_update()


class OfflineImitationLearning(ImitationLearningAlgorithmMixin, OfflineAlgorithm):
    """Offline vanilla imitation learning (imitation_base.py:158-183)."""

    def __init__(self, *, policy: ImitationPolicy, optim: OptimizerFactory) -> None:
        super().__init__(policy=policy)
        self.optim = self._create_optimizer(self.policy, optim)
        self._build_device_update()
