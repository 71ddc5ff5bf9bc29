"""Quantile-regression DQN (arXiv:1710.10044) with ``update()`` on the device.

Reference: tianshou/algorithm/modelfree/qrdqn.py (QRDQNPolicy :18-20, QRDQN :26-131), modelfree/dqn.py:170-283
(QLearningOffPolicyAlgorithm: n-step return, the lagged network), utils/lagged_network.py:83-103 (the full lagged copy),
utils/net/common.py:298-369 (``Net(num_atoms)``), env/atari/atari_network.py:211-235 (``QRDQNet``).

Per ``update(buffer, sample_size)``:
  host : index draw from the buffer's RNG streams (prioritised: the importance weight), the range check of the drawn actions,
         one D2H of the loss scalars.
  GPU  : observation source of s_{t+n} -> online chain (+ the lagged chain on the lagged flat buffer) -> ``ts_qrdqn_target``
         (quantile means, first arg-max, the chosen action's N quantiles) -> value mask + ``ts_nstep_return`` over N columns;
         observation source of s -> chain -> ``ts_qrdqn_rows`` (quantile-Huber loss, d loss / d q, the priorities) -> backward
         GEMMs -> Adam; the lagged copy is one device memcpy.
The network is read as a plain layer chain ending in ``Linear(., actions * num_quantiles)``: ``Net(num_atoms=N)`` and ``QRDQNet``
only view that output as ``[B, actions, N]``, which is the kernels' row layout.
"""
from __future__ import annotations

from copy import deepcopy

import numpy as np
import torch
from torch import nn

from ..._cabi import call, ptr, stream_ptr
from ...data import Batch, ReplayBuffer
from ..base import OffPolicyAlgorithm
from ..discrete_q import DiscreteQCore, describe_q_network, lagged_group
from ..flat_params import FlatGroup, UnsupportedModelError, bind_optimizer
from ..netgraph import ACT_NONE, FusedStack, compile_sequential, layer_params, module_layers
from ..optim import OptimizerFactory
from ..twin_critic import _EvalModeModule, cuda_device_of, pop_batch_weight
from .dqn import DiscreteQLearningPolicy, SimpleLossTrainingStats


class QRDQNPolicy(DiscreteQLearningPolicy):
    """The arg-max of the quantile means (qrdqn.py:18-20).  ``forward`` is the torch-module path the Collector runs."""

    def compute_q_value(self, logits: torch.Tensor, mask: np.ndarray | None) -> torch.Tensor:
        return super().compute_q_value(logits.mean(2), mask)


class QRDQN(DiscreteQCore, OffPolicyAlgorithm):
    """QR-DQN, reference API and semantics (qrdqn.py:26-131).

    ``policy.model`` is a ``Net(num_atoms=num_quantiles)`` on flat observations or a ``QRDQNet`` (optionally behind
    ``ScaledObsInputActionReprNet``) with ``actions * num_quantiles`` outputs.  The target takes the arg-max of the online
    network's quantile means at s_{t+n} and the lagged network's quantiles of that action (the online ones when
    ``target_update_freq == 0``); there is no double-Q switch.  The lagged copy is refreshed when ``_iter % target_update_freq
    == 0``, before the step.  A prioritised buffer's importance weight scales each row's loss, and ``batch.weight`` leaves the
    update as the rows' mean summed Huber term, the priority the buffer is updated with.
    """

    def __init__(self, *, policy: QRDQNPolicy, optim: OptimizerFactory, gamma: float = 0.99, num_quantiles: int = 200,
                 n_step_return_horizon: int = 1, target_update_freq: int = 0) -> None:
        assert num_quantiles > 1, f"num_quantiles should be greater than 1 but got: {num_quantiles}"
        super().__init__(policy=policy)
        assert 0.0 <= gamma <= 1.0, f"discount factor should be in [0, 1] but got: {gamma}"
        assert n_step_return_horizon > 0, f"n_step_return_horizon should be greater than 0 but got: {n_step_return_horizon}"
        self.gamma = gamma
        self.n_step = n_step_return_horizon
        self.target_update_freq = target_update_freq
        self.num_quantiles = num_quantiles
        dev = cuda_device_of(policy.model)
        self._build_network(policy, dev)
        self.optim = self._create_optimizer(policy, optim)
        bind_optimizer(self.optim, self._group)
        # the midpoints exactly as the reference forms them in fp32 on the CPU (not (k + 0.5) / N, which differs in the last bit)
        tau = torch.linspace(0, 1, num_quantiles + 1)
        self.tau_hat = nn.Parameter(((tau[:-1] + tau[1:]) / 2).view(1, -1, 1).to(dev), requires_grad=False)
        self.model_old: _EvalModeModule | None = None
        self._g_old: FlatGroup | None = None
        if self.use_target_network:
            self.model_old = _EvalModeModule(deepcopy(policy.model))
            self._g_old = lagged_group(self._group, list(self.model_old.parameters()))

    def _build_network(self, policy: QRDQNPolicy, dev: torch.device) -> None:
        """Read ``policy.model`` as a plain layer chain ending in ``Linear(., actions * num_quantiles)``, refuse anything else,
        and set up the core (``_init_discrete``), the flat group over the model's parameters and the device network."""
        inner, in_shape, in_scale = describe_q_network(policy.model)
        if getattr(inner, "softmax", False):
            raise UnsupportedModelError("Net(softmax=True): QR-DQN reads the network output as quantiles; build it with "
                                        "softmax=False")
        layers = compile_sequential(module_layers(inner), in_shape)
        if layers[-1].kind != "linear" or layers[-1].act != ACT_NONE:
            raise UnsupportedModelError("the quantile network must end in a linear layer over actions * num_quantiles")
        n_actions = int(policy.action_space.n)
        if layers[-1].out_dim != n_actions * self.num_quantiles:
            raise UnsupportedModelError(f"the network has {layers[-1].out_dim} outputs, not {n_actions} actions x "
                                        f"{self.num_quantiles} quantiles")
        self._init_discrete(dev, in_shape, in_scale, n_actions)
        self._group = FlatGroup(layer_params(layers), dev)
        self._net = FusedStack(layers, self._group, "qr")

    @property
    def use_target_network(self) -> bool:
        return self.target_update_freq > 0

    # ------------------------------------------------------------------ target
    def _target_q(self, buffer: ReplayBuffer, indices: np.ndarray) -> torch.Tensor:
        """The quantiles of Q_old(s', argmax_a mean_k Q(s', a, k))   (qrdqn.py:94-106)."""
        src = self._obs_source(buffer, indices, "obs_next")
        B = src.rows
        q_online = self._net.forward(src.x, B, "tq_on", frames=src.frames)[-1]
        q_next = q_online
        if self.use_target_network:
            self._g_old.ensure_adopted()
            q_next = self._net.forward(src.x, B, "tq_old", frames=src.frames, params=self._g_old.flat)[-1]
        out = self._buf("tq_out", (B, self.num_quantiles))
        call("ts_qrdqn_target", ptr(q_online), ptr(q_next), B, self.n_actions, self.num_quantiles, ptr(out), None,
             stream_ptr(self._dev))
        return out

    # ------------------------------------------------------------------ update
    def _quantile_step(self, batch: Batch, min_q_weight: float) -> np.ndarray:
        """One step on the quantile-Huber loss (+ ``min_q_weight`` times the CQL penalty): (loss, qr_loss, cql_loss)."""
        self._tick_lagged(self.target_update_freq)
        src = batch.obs
        B, A, N = src.rows, self.n_actions, self.num_quantiles
        weight = pop_batch_weight(batch, self._dev)
        acts = self._net.forward(src.x, B, "up", frames=src.frames)
        returns = batch.returns.reshape(B, N).to(self._dev, torch.float32).contiguous()
        dq, prio = self._buf("dq", (B, A * N)), self._buf("prio", B)
        rows, losses = self._buf("loss_rows", (3, B)), self._buf("losses", 4)
        call("ts_qrdqn_rows", ptr(acts[-1]), ptr(batch.act), ptr(returns), ptr(self.tau_hat), ptr(weight), B, A, N,
             float(min_q_weight), ptr(dq), ptr(prio), ptr(rows), ptr(losses), stream_ptr(self._dev))
        batch.weight = prio                     # prio-buffer
        self._net.backward(acts, dq, B, "up")
        self._group.adam_step(self.optim._optim, self.optim._max_grad_norm)
        return losses[:3].cpu().numpy()         # the only host read of the losses

    def _update_with_batch(self, batch: Batch) -> SimpleLossTrainingStats:
        return SimpleLossTrainingStats(loss=float(self._quantile_step(batch, 0.0)[0]))
