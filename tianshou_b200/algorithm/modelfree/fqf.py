"""Fully parameterized quantile functions (arXiv:1911.02140) with ``update()`` on the device.

Reference: tianshou/algorithm/modelfree/fqf.py (FQFTrainingStats :20-24, FQFPolicy :27-106, FQF :109-255),
utils/net/discrete.py:219-314 (FractionProposalNetwork, FullQuantileFunction).

The network is IQN's (iqn.py ``QuantileNetworkCore``) at fractions a one-layer fraction net proposes from the trunk's features:
z = Linear(D, N)(feat) -> ``ts_fqf_fractions`` (softmax, cumulative sum ``taus [B, N + 1]``, midpoints ``tau_hats [B, N]``, the
inner fractions ``taus[:, 1:-1]``, the entropy) -> the quantiles at ``tau_hats`` (and, for the fraction loss, at the inner
fractions).  Per ``update(buffer, sample_size)``:
  host : index draw from the buffer's RNG streams (prioritised: the importance weight), the range check of the drawn actions,
         one D2H of the four loss statistics.
  GPU  : observation source of s_{t+n} -> trunk -> fraction net -> ``ts_fqf_fractions`` -> the cosines of ``tau_hats`` once ->
         online embedding + head (+ the lagged trunk, embedding and head on the lagged flat buffer, at the same cosines) ->
         ``ts_fqf_target`` (fraction-weighted means, first arg-max, the chosen action's N quantiles) -> value mask +
         ``ts_nstep_return``; observation source of s -> trunk -> fraction net -> ``ts_fqf_fractions`` -> quantiles at ``tau_hats``
         and at the inner fractions -> ``ts_iqn_rows`` (quantile-Huber loss with ``tau_hats``, d loss / d q, the priorities) and
         ``ts_fqf_fraction_rows`` (the W1 fraction loss, the entropy, d loss / d z) -> the fraction net's weight and bias
         gradients -> its Adam / RMSprop step; head, embedding and trunk backward -> Adam; the lagged copy is one device memcpy.
Nothing in the update draws a random number besides the buffer's index draw.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Any

import numpy as np
import torch
from torch import nn

from ..._cabi import call, ptr, stream_ptr
from ...data import Batch, ReplayBuffer, to_numpy
from ..flat_params import FlatGroup, UnsupportedModelError, bind_optimizer
from ..netgraph import ACT_NONE, FusedStack, compile_sequential, layer_params
from ..optim import OptimizerFactory
from ..twin_critic import pop_batch_weight
from .dqn import DiscreteQLearningPolicy, SimpleLossTrainingStats
from .iqn import QuantileNetworkCore
from .qrdqn import QRDQN, QRDQNPolicy


@dataclass(kw_only=True)
class FQFTrainingStats(SimpleLossTrainingStats):
    quantile_loss: float
    fraction_loss: float
    entropy_loss: float


class FQFPolicy(QRDQNPolicy):
    """The first arg-max of the fraction-weighted quantile mean (fqf.py:27-106).  ``forward`` is the torch-module path the
    Collector runs; it returns the quantiles ``logits [B, actions, N]`` at ``tau_hats``, the ``fractions`` Batch(taus, tau_hats,
    entropies) (the ones passed in, when given) and, in training mode, ``quantiles_tau [B, actions, N - 1]``."""

    def __init__(self, *, model: nn.Module, fraction_model: nn.Module, action_space: Any, observation_space: Any | None = None,
                 eps_training: float = 0.0, eps_inference: float = 0.0) -> None:
        assert hasattr(action_space, "n"), "FQF needs a discrete action space"
        super().__init__(model=model, action_space=action_space, observation_space=observation_space, eps_training=eps_training,
                         eps_inference=eps_inference)
        self.fraction_model = fraction_model

    def forward(self, batch: Batch, state: Any = None, model: nn.Module | None = None, fractions: Batch | None = None,
                **kwargs: Any) -> Batch:
        if model is None:
            model = self.model
        obs = batch.obs
        obs_arr = obs.obs if hasattr(obs, "obs") else obs
        if fractions is None:
            (logits, fractions, quantiles_tau), hidden = model(obs_arr, propose_model=self.fraction_model, state=state,
                                                               info=batch.get("info"))
        else:
            (logits, _, quantiles_tau), hidden = model(obs_arr, propose_model=self.fraction_model, fractions=fractions,
                                                       state=state, info=batch.get("info"))
        weighted_logits = (fractions.taus[:, 1:] - fractions.taus[:, :-1]).unsqueeze(1) * logits
        q = DiscreteQLearningPolicy.compute_q_value(self, weighted_logits.sum(2), getattr(obs, "mask", None))
        return Batch(logits=logits, act=to_numpy(q.max(dim=1)[1]), state=hidden, fractions=fractions, quantiles_tau=quantiles_tau)


class FQF(QuantileNetworkCore, QRDQN):
    """FQF, reference API and semantics (fqf.py:109-255).

    ``policy.model`` is a ``FullQuantileFunction`` that IQN's update would take (a ``Net`` or ``DQNet(features_only=True)`` trunk,
    optionally behind ``ScaledObsInputActionReprNet``, a ``Linear(C, D) + ReLU`` embedding, a ``last`` MLP ending in
    ``Linear(., actions)``); ``policy.fraction_model`` is a ``FractionProposalNetwork``: one ``Linear(D, N)`` on the trunk's width,
    sharing no parameter with the model.  ``optim`` steps ``policy.model`` (Adam), ``fraction_optim`` steps
    ``policy.fraction_model`` (Adam or RMSprop) and is created second.  The target takes the first arg-max of the online
    network's fraction-weighted quantile mean at s_{t+n} and the lagged network's quantiles of that action at the online
    ``tau_hats`` (the online quantiles when ``target_update_freq == 0``).  The lagged copy is of ``policy.model`` only.  A
    prioritised buffer's importance weight scales the quantile loss only.  ``num_fractions`` only becomes ``tau_hat`` in
    ``state_dict()``, as in QR-DQN; the network's N is the fraction model's ``num_fractions``.
    """

    def __init__(self, *, policy: FQFPolicy, optim: OptimizerFactory, fraction_optim: OptimizerFactory, gamma: float = 0.99,
                 num_fractions: int = 32, ent_coef: float = 0.0, n_step_return_horizon: int = 1,
                 target_update_freq: int = 0) -> None:
        super().__init__(policy=policy, optim=optim, gamma=gamma, num_quantiles=num_fractions,
                         n_step_return_horizon=n_step_return_horizon, target_update_freq=target_update_freq)
        if not np.isfinite(ent_coef):
            raise ValueError(f"ent_coef must be finite, got {ent_coef}")
        self.ent_coef = ent_coef
        self.fraction_optim = self._create_optimizer(policy.fraction_model, fraction_optim)
        bind_optimizer(self.fraction_optim, self._fgroup, rmsprop=True)

    def _create_policy_optimizer(self, policy: QRDQNPolicy, optim: OptimizerFactory) -> QRDQN.Optimizer:
        return self._create_optimizer(policy.model, optim)

    def _build_network(self, policy: QRDQNPolicy, dev: torch.device) -> None:
        """IQN's network over ``policy.model``, then the fraction net as a one-layer ``FusedStack`` in a flat group of its own."""
        self._build_quantile_network(policy, dev)
        fm = getattr(policy, "fraction_model", None)
        lin = getattr(fm, "net", None)
        D = self._feat_dim
        if not isinstance(lin, nn.Linear) or lin.bias is None or lin.in_features != D:
            raise UnsupportedModelError(f"fraction_model: expected a FractionProposalNetwork, Linear({D}, N) with a bias on the "
                                        f"trunk's {D} features, got {type(fm).__name__}")
        if [id(p) for p in fm.parameters()] != [id(lin.weight), id(lin.bias)]:
            raise UnsupportedModelError("fraction_model: its parameters must be exactly its Linear layer's weight and bias")
        if {id(p) for p in fm.parameters()} & {id(p) for p in policy.model.parameters()}:
            raise UnsupportedModelError("fraction_model shares parameters with model: each needs its own optimiser")
        if lin.weight.device != dev:
            raise UnsupportedModelError(f"fraction_model lives on {lin.weight.device}, the model on {dev}")
        self._n_fractions = int(lin.out_features)
        if self._n_fractions < 2:
            raise UnsupportedModelError(f"fraction_model proposes {self._n_fractions} fraction; FQF needs at least 2")
        layers = compile_sequential([lin], (D,))
        assert len(layers) == 1 and layers[0].act == ACT_NONE
        self._fgroup = FlatGroup(layer_params(layers), dev)
        self._frac = FusedStack(layers, self._fgroup, "frac")

    # ------------------------------------------------------------------ network
    def _propose(self, feat: torch.Tensor, tag: str) -> dict[str, Any]:
        """The fraction net on ``feat [B, D]`` and ``ts_fqf_fractions``: z, taus, tau_hats, inner fractions, p, log p, H."""
        B, N = feat.shape[0], self._n_fractions
        z = self._frac.forward(feat, B, tag)
        out = dict(z=z, taus=self._buf(f"{tag}_taus", (B, N + 1)), tau_hats=self._buf(f"{tag}_tau_hats", (B, N)),
                   inner=self._buf(f"{tag}_inner", (B, N - 1)), p=self._buf(f"{tag}_p", (B, N)),
                   logp=self._buf(f"{tag}_logp", (B, N)), H=self._buf(f"{tag}_H", B))
        call("ts_fqf_fractions", ptr(z[-1]), B, N, ptr(out["taus"]), ptr(out["tau_hats"]), ptr(out["inner"]), ptr(out["p"]),
             ptr(out["logp"]), ptr(out["H"]), stream_ptr(self._dev))
        return out

    # ------------------------------------------------------------------ target
    def _target_q(self, buffer: ReplayBuffer, indices: np.ndarray) -> torch.Tensor:
        """The quantiles of Q_old(s', a*) at the online ``tau_hats``, a* the first arg-max of the online fraction-weighted
        quantile mean   (fqf.py:178-193)."""
        src = self._obs_source(buffer, indices, "obs_next")
        B, N = src.rows, self._n_fractions
        trunk = self._trunk.forward(src.x, B, "tq_on", frames=src.frames)
        fr = self._propose(trunk[-1], "tq_on")
        cos, _, head = self._quantiles_at(trunk[-1], fr["tau_hats"], N, "tq_on")
        q_online = head[-1]
        q_next = q_online
        if self.use_target_network:
            self._g_old.ensure_adopted()
            old = self._g_old.flat
            trunk_old = self._trunk.forward(src.x, B, "tq_old", frames=src.frames, params=old)
            q_next = self._quantiles_at(trunk_old[-1], None, N, "tq_old", params=old, cos=cos)[2][-1]
        out = self._buf("tq_out", (B, N))
        call("ts_fqf_target", ptr(q_online), ptr(fr["taus"]), ptr(q_next), B, self.n_actions, N, ptr(out), None,
             stream_ptr(self._dev))
        return out

    # ------------------------------------------------------------------ update
    def _update_with_batch(self, batch: Batch) -> FQFTrainingStats:
        self._tick_lagged(self.target_update_freq)
        src = batch.obs
        B, A, N = src.rows, self.n_actions, self._n_fractions
        st = stream_ptr(self._dev)
        weight = pop_batch_weight(batch, self._dev)
        trunk = self._trunk.forward(src.x, B, "up", frames=src.frames)
        fr = self._propose(trunk[-1], "up")
        _, embed, head = self._quantiles_at(trunk[-1], fr["tau_hats"], N, "up")
        q_tau = self._quantiles_at(trunk[-1], fr["inner"], N - 1, "up_tau")[2][-1]
        returns = batch.returns.reshape(B, -1).to(self._dev, torch.float32).contiguous()
        dq, prio = self._buf("dq", (B * N, A)), self._buf("prio", B)
        dz, rows = self._buf("dz", (B, N)), self._buf("loss_rows", (3, B))
        losses = self._buf("losses", 8)          # ts_iqn_rows' four, then ts_fqf_fraction_rows' four: one read
        call("ts_iqn_rows", ptr(head[-1]), ptr(batch.act), ptr(returns), ptr(fr["tau_hats"]), ptr(weight), B, A, N,
             returns.shape[1], ptr(dq), ptr(prio), ptr(rows), ptr(losses), st)
        call("ts_fqf_fraction_rows", ptr(head[-1]), ptr(q_tau), ptr(batch.act), ptr(fr["taus"]), ptr(fr["p"]), ptr(fr["logp"]),
             ptr(fr["H"]), B, A, N, float(self.ent_coef), ptr(dz), ptr(rows), losses.data_ptr() + 16, st)
        batch.weight = prio                     # prio-buffer
        self._frac.backward(fr["z"], dz, B, "up")
        self._fgroup.optimizer_step(self.fraction_optim._optim, self.fraction_optim._max_grad_norm)
        self._quantile_backward(trunk, embed, head, dq, N, "up")
        self._group.adam_step(self.optim._optim, self.optim._max_grad_norm)
        l = losses.cpu().numpy()                # the only host read of the losses
        return FQFTrainingStats(loss=float(l[0]) + float(l[4]), quantile_loss=float(l[0]), fraction_loss=float(l[5]),
                                entropy_loss=float(l[6]))
