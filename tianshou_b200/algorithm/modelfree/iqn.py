"""Implicit quantile networks (arXiv:1806.06923) with ``update()`` on the device.

Reference: tianshou/algorithm/modelfree/iqn.py (IQNPolicy :21-100, IQN :103-183), modelfree/qrdqn.py:94-106 (the target at the
online arg-max of the quantile means), utils/net/discrete.py:126-216 (CosineEmbeddingNetwork, ImplicitQuantileNetwork).

The network is a trunk (the preprocess net) on B rows, the cosine embedding of S fractions per row, and the ``last`` MLP on the
B * S rows ``h[b * S + s] = feat[b] * e[b * S + s]`` (sample-major, so the head's output is q[B][S][A]).  Per
``update(buffer, sample_size)``:
  host : index draw from the buffer's RNG streams (prioritised: the importance weight), the range check of the drawn actions,
         one D2H of the loss.
  GPU  : observation source of s_{t+n} -> online network on ``online_sample_size`` fractions (+ the lagged network, on the lagged
         flat buffer, on ``target_sample_size`` fractions of its own) -> ``ts_iqn_target`` (sample means, first arg-max, the
         chosen action's quantiles) -> value mask + ``ts_nstep_return`` over those columns; observation source of s -> network on
         a third draw of ``online_sample_size`` fractions -> ``ts_iqn_rows`` (quantile-Huber loss with a fraction per row and
         sample, d loss / d q, the priorities) -> head backward -> ``ts_iqn_mix_backward`` -> the embedding's weight and bias
         gradients -> trunk backward -> Adam; the lagged copy is one device memcpy.
One network forward is the trunk's GEMMs, ``ts_iqn_cos``, the embedding's ``Linear + ReLU`` GEMM, ``ts_iqn_mix`` and the head's
GEMMs.  Every fraction draw is ``IQN._draw_taus``, the reference's own ``torch.rand`` call, in the reference's order.
"""
from __future__ import annotations

from typing import Any, NamedTuple

import numpy as np
import torch
from torch import nn

from ..._cabi import call, ptr, stream_ptr
from ...data import Batch, ReplayBuffer, to_numpy
from ..discrete_q import describe_discrete_head
from ..flat_params import FlatGroup, UnsupportedModelError
from ..netgraph import ACT_NONE, ACT_RELU, FusedStack, _out_shape, compile_sequential, layer_params, module_layers
from ..obs_source import DeviceObsSource
from ..optim import OptimizerFactory
from ..twin_critic import pop_batch_weight
from .dqn import SimpleLossTrainingStats
from .qrdqn import QRDQN, QRDQNPolicy


class IQNPolicy(QRDQNPolicy):
    """The arg-max of the sample means (iqn.py:21-100).  The sample size is ``target_sample_size`` for the lagged network
    (``model=``), ``online_sample_size`` in train mode and ``sample_size`` in eval mode.  ``forward`` is the torch-module path
    the Collector runs; it returns the logits ``[B, actions, S]`` and the fractions ``taus [B, S]``."""

    def __init__(self, *, model: nn.Module, action_space: Any, sample_size: int = 32, online_sample_size: int = 8,
                 target_sample_size: int = 8, observation_space: Any | None = None, eps_training: float = 0.0,
                 eps_inference: float = 0.0) -> None:
        assert sample_size > 1, f"sample_size should be greater than 1 but got: {sample_size}"
        assert online_sample_size > 1, f"online_sample_size should be greater than 1 but got: {online_sample_size}"
        assert target_sample_size > 1, f"target_sample_size should be greater than 1 but got: {target_sample_size}"
        super().__init__(model=model, action_space=action_space, observation_space=observation_space, eps_training=eps_training,
                         eps_inference=eps_inference)
        self.sample_size = sample_size
        self.online_sample_size = online_sample_size
        self.target_sample_size = target_sample_size

    def forward(self, batch: Batch, state: Any = None, model: nn.Module | None = None, **kwargs: Any) -> Batch:
        if model is not None:
            sample_size = self.target_sample_size
        elif self.training:
            sample_size = self.online_sample_size
        else:
            sample_size = self.sample_size
        if model is None:
            model = self.model
        obs = batch.obs
        obs_arr = obs.obs if hasattr(obs, "obs") else obs
        (logits, taus), hidden = model(obs_arr, sample_size=sample_size, state=state, info=batch.get("info"))
        q = self.compute_q_value(logits, getattr(obs, "mask", None))
        return Batch(logits=logits, act=to_numpy(q.argmax(dim=1)), state=hidden, taus=taus)


class _IqnActs(NamedTuple):
    """One device forward: the trunk's, the embedding's and the head's activation lists and the fractions it drew.
    ``trunk[-1]`` is feat [B, D], ``embed[0]`` the cosines [B * S, C], ``embed[-1]`` e [B * S, D], ``head[0]`` h, ``head[-1]`` q."""

    trunk: list[torch.Tensor]
    taus: torch.Tensor
    embed: list[torch.Tensor]
    head: list[torch.Tensor]


class IQN(QRDQN):
    """IQN, reference API and semantics (iqn.py:103-183): QR-DQN's target rule and loss shape with sampled fractions.

    ``policy.model`` is an ``ImplicitQuantileNetwork`` whose preprocess net is a ``Net`` or a ``DQNet(features_only=True)``
    (optionally behind ``ScaledObsInputActionReprNet``) and whose ``last`` MLP ends in ``Linear(., actions)``.  The target takes
    the arg-max of the online network's sample means at s_{t+n} and the lagged network's ``target_sample_size`` quantiles of
    that action, on fractions of its own; with ``target_update_freq == 0`` both come from one online forward, and the returns
    have ``online_sample_size`` columns.  The loss pairs each of the step's ``online_sample_size`` quantiles, with its own
    fraction, against every return column.  ``num_quantiles`` only becomes ``tau_hat`` in ``state_dict()``, as in the reference.
    """

    def __init__(self, *, policy: IQNPolicy, optim: OptimizerFactory, gamma: float = 0.99, num_quantiles: int = 200,
                 n_step_return_horizon: int = 1, target_update_freq: int = 0) -> None:
        super().__init__(policy=policy, optim=optim, gamma=gamma, num_quantiles=num_quantiles,
                         n_step_return_horizon=n_step_return_horizon, target_update_freq=target_update_freq)

    def _build_network(self, policy: QRDQNPolicy, dev: torch.device) -> None:
        """The trunk, the embedding and the head of an ``ImplicitQuantileNetwork`` in one flat group, in the model's parameter
        order (``preprocess.*``, ``last.*``, ``embed_model.net.0.*``)."""
        model = policy.model
        inner, last, in_shape, in_scale = describe_discrete_head(model, "model")
        embed_model = getattr(model, "embed_model", None)
        if embed_model is None:
            raise UnsupportedModelError(f"model: expected an ImplicitQuantileNetwork (preprocess net, last MLP, embed_model), got "
                                        f"{type(model).__name__}")
        trunk = compile_sequential(module_layers(inner), in_shape)
        if not trunk:
            raise UnsupportedModelError("model: the preprocess network has no layers")
        feat = _out_shape(trunk, in_shape)
        head = compile_sequential(module_layers(last), feat)
        if not head or head[-1].kind != "linear" or head[-1].act != ACT_NONE:
            raise UnsupportedModelError("the quantile network must end in a linear layer over the actions")
        n_actions = int(policy.action_space.n)
        if head[-1].out_dim != n_actions:
            raise UnsupportedModelError(f"the network has {head[-1].out_dim} outputs, not {n_actions} actions")
        C = int(embed_model.num_cosines)
        embed = compile_sequential(module_layers(embed_model), (C,))
        if len(embed) != 1 or embed[0].out_dim != feat[0] or embed[0].act != ACT_RELU:
            raise UnsupportedModelError(f"model: the embedding must be Linear({C}, {feat[0]}) + ReLU")
        params = layer_params(trunk) + layer_params(head) + layer_params(embed)
        if [id(p) for p in params] != [id(p) for p in model.parameters()]:
            raise UnsupportedModelError("the compiled layers' parameters differ from the model's parameters")
        self._init_discrete(dev, in_shape, in_scale, n_actions)
        self._group = FlatGroup(params, dev)
        self._trunk = FusedStack(trunk, self._group, "trunk")
        self._embed = FusedStack(embed, self._group, "embed")
        self._head = FusedStack(head, self._group, "head")
        self.num_cosines, self._feat_dim = C, int(feat[0])
        # the derivative of the trunk's last activation, folded into its feature gradient by ts_iqn_mix_backward; a trunk ending
        # in Flatten applies its producer's ReLU mask in its own backward
        self._trunk_act = trunk[-1].act if trunk[-1].kind != "flatten" else ACT_NONE

    # ------------------------------------------------------------------ network
    def _draw_taus(self, rows: int, sample_size: int) -> torch.Tensor:
        """The fractions of one forward: ``torch.rand(rows, sample_size)`` in fp32 on the device, the call the reference's
        ``ImplicitQuantileNetwork.forward`` makes (discrete.py:210).  Every draw of an update goes through here, in the
        reference's order: the target's online forward, the lagged forward (when there is one), the step's forward."""
        return torch.rand(rows, sample_size, dtype=torch.float32, device=self._dev)

    def _quantiles(self, src: DeviceObsSource, S: int, tag: str, params: torch.Tensor | None = None) -> _IqnActs:
        """q[B][S][A] of the network (``params``: the lagged flat buffer) on ``S`` fresh fractions per row."""
        B, R, C, D = src.rows, src.rows * S, self.num_cosines, self._feat_dim
        st = stream_ptr(self._dev)
        trunk = self._trunk.forward(src.x, B, tag, frames=src.frames, params=params)
        taus = self._draw_taus(B, S)
        assert taus.shape == (B, S) and taus.dtype == torch.float32 and taus.is_contiguous() and taus.device == self._dev
        cos = self._buf(f"{tag}_cos", (R, C))
        call("ts_iqn_cos", ptr(taus), R, C, ptr(cos), st)
        embed = self._embed.forward(cos, R, tag, params=params)
        h = self._buf(f"{tag}_h", (R, D))
        call("ts_iqn_mix", ptr(trunk[-1]), ptr(embed[-1]), B, S, D, ptr(h), st)
        head = self._head.forward(h, R, tag, params=params)
        return _IqnActs(trunk, taus, embed, head)

    def _backward(self, f: _IqnActs, dq: torch.Tensor, S: int, tag: str) -> None:
        """Every parameter's gradient of the loss whose gradient w.r.t. q is ``dq [B * S, A]``, stored into the group's gradient
        buffer: head (with its input gradient dh), ``ts_iqn_mix_backward`` (dfeat and the embedding's pre-activation gradient),
        the embedding's weight and bias gradients, then the trunk."""
        feat = f.trunk[-1]
        B, D = feat.shape[0], self._feat_dim
        R = B * S
        dh = self._head.backward(f.head, dq, R, tag, input_grad=True)
        dfeat, de_pre = self._buf(f"{tag}_dfeat", (B, D)), self._buf(f"{tag}_de_pre", (R, D))
        call("ts_iqn_mix_backward", ptr(dh), ptr(feat), ptr(f.embed[-1]), B, S, D, int(self._trunk_act),
             ptr(feat) if self._trunk_act != ACT_NONE else None, ptr(dfeat), ptr(de_pre), stream_ptr(self._dev))
        self._embed.backward(f.embed, de_pre, R, tag, dy_preact=True)
        self._trunk.backward(f.trunk, dfeat, B, tag, dy_preact=True)

    # ------------------------------------------------------------------ target
    def _target_q(self, buffer: ReplayBuffer, indices: np.ndarray) -> torch.Tensor:
        """The quantiles of Q_old(s', argmax_a mean_s Q(s', a, s)) on the lagged network's own fractions   (qrdqn.py:94-106)."""
        src = self._obs_source(buffer, indices, "obs_next")
        B, S_on = src.rows, self.policy.online_sample_size
        q_online = self._quantiles(src, S_on, "tq_on").head[-1]
        q_next, S_next = q_online, S_on
        if self.use_target_network:
            self._g_old.ensure_adopted()
            S_next = self.policy.target_sample_size
            q_next = self._quantiles(src, S_next, "tq_old", params=self._g_old.flat).head[-1]
        out = self._buf("tq_out", (B, S_next))
        call("ts_iqn_target", ptr(q_online), ptr(q_next), B, self.n_actions, S_on, S_next, ptr(out), None, stream_ptr(self._dev))
        return out

    # ------------------------------------------------------------------ update
    def _update_with_batch(self, batch: Batch) -> SimpleLossTrainingStats:
        self._tick_lagged(self.target_update_freq)
        src = batch.obs
        B, A, S_on = src.rows, self.n_actions, self.policy.online_sample_size
        weight = pop_batch_weight(batch, self._dev)
        f = self._quantiles(src, S_on, "up")
        returns = batch.returns.reshape(B, -1).to(self._dev, torch.float32).contiguous()
        S_t = returns.shape[1]
        dq, prio = self._buf("dq", (B * S_on, A)), self._buf("prio", B)
        rows, losses = self._buf("loss_rows", (3, B)), self._buf("losses", 4)
        call("ts_iqn_rows", ptr(f.head[-1]), ptr(batch.act), ptr(returns), ptr(f.taus), ptr(weight), B, A, S_on, S_t, ptr(dq),
             ptr(prio), ptr(rows), ptr(losses), stream_ptr(self._dev))
        batch.weight = prio                     # prio-buffer
        self._backward(f, dq, S_on, "up")
        self._group.adam_step(self.optim._optim, self.optim._max_grad_norm)
        return SimpleLossTrainingStats(loss=float(losses[0].item()))      # the only host read of the loss
