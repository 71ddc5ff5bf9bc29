"""Categorical DQN (C51, arXiv:1707.06887) with ``update()`` on the device.

Reference: tianshou/algorithm/modelfree/c51.py (C51Policy :16-66, C51 :69-160), modelfree/dqn.py:170-283
(QLearningOffPolicyAlgorithm: n-step return, the lagged network), utils/lagged_network.py:83-103 (the full lagged copy),
utils/net/common.py:298-369 (``Net(softmax=True, num_atoms)``), env/atari/atari_network.py:125-151 (``C51Net``).

Per ``update(buffer, sample_size)``:
  host : index draw from the buffer's RNG streams (prioritised: the importance weight), the range check of the drawn actions,
         one D2H of the loss.
  GPU  : value mask + ``ts_nstep_return`` over the N atoms of the support; the lagged copy (one device memcpy, before the
         target, as the reference refreshes it first); observation source of s_{t+n} -> online chain (+ the lagged chain on the
         lagged flat buffer) -> ``ts_c51_target`` (per-action softmax, expected values, first arg-max, the chosen action's
         distribution); observation source of s -> chain -> ``ts_c51_rows`` (clamp, dense projection, cross-entropy, d loss /
         d logits, the priorities) -> backward GEMMs -> Adam.
The network is read as a plain layer chain ending in ``Linear(., actions * num_atoms)``; the softmax that ``Net(softmax=True)``
and ``C51Net`` apply over each action's atoms is taken inside the kernels, on the raw ``[B, actions, num_atoms]`` logits.
"""
from __future__ import annotations

from copy import deepcopy
from typing import Any

import numpy as np
import torch
from torch import nn

from ..._cabi import call, ptr, stream_ptr
from ...data import Batch, ReplayBuffer
from ...env.atari.atari_network import C51Net
from ..base import OffPolicyAlgorithm
from ..discrete_q import DiscreteQCore, atom_chain, describe_q_network, lagged_group
from ..flat_params import FlatGroup, UnsupportedModelError, bind_optimizer
from ..netgraph import FusedStack, layer_params
from ..optim import OptimizerFactory
from ..twin_critic import _EvalModeModule, cuda_device_of, pop_batch_weight
from .dqn import DiscreteQLearningPolicy
from .reinforce import LossSequenceTrainingStats


class C51Policy(DiscreteQLearningPolicy):
    """The arg-max of the expected values ``(p * support).sum(2)`` (c51.py:16-66).  ``support`` is a frozen parameter, so it is
    in ``state_dict()`` and in the optimiser's parameter list, as in the reference; it lives on the model's device.
    ``forward`` is the torch-module path the Collector runs: ``logits`` are the model's probabilities ``[B, A, num_atoms]``."""

    def __init__(self, model: nn.Module, action_space: Any, observation_space: Any | None = None, num_atoms: int = 51,
                 v_min: float = -10.0, v_max: float = 10.0, eps_training: float = 0.0, eps_inference: float = 0.0) -> None:
        assert hasattr(action_space, "n"), f"C51Policy needs a Discrete action space, got {action_space}"
        super().__init__(model=model, action_space=action_space, observation_space=observation_space, eps_training=eps_training,
                         eps_inference=eps_inference)
        assert num_atoms > 1, f"num_atoms should be greater than 1 but got: {num_atoms}"
        assert v_min < v_max, f"v_max should be larger than v_min, but got {v_min=} and {v_max=}"
        self.num_atoms = num_atoms
        self.v_min = v_min
        self.v_max = v_max
        dev = next((p.device for p in model.parameters()), torch.device("cpu"))
        # formed on the CPU as the reference forms it, then moved: a device linspace may differ in the last bit
        self.support = nn.Parameter(torch.linspace(self.v_min, self.v_max, self.num_atoms).to(dev), requires_grad=False)

    def compute_q_value(self, logits: torch.Tensor, mask: np.ndarray | None) -> torch.Tensor:
        return super().compute_q_value((logits * self.support).sum(2), mask)


class C51(DiscreteQCore, OffPolicyAlgorithm):
    """C51, reference API and semantics (c51.py:69-160).

    ``policy.model`` is a ``Net(softmax=True, num_atoms=N)`` on flat observations or a ``C51Net`` (optionally behind
    ``ScaledObsInputActionReprNet``) with ``actions * N`` outputs, N = ``policy.num_atoms``.  The lagged copy is refreshed when
    ``_iter % target_update_freq == 0``, before the target is formed.  The target takes the online network's first arg-max
    of the expected values at s_{t+n} and the lagged network's distribution of that action (the online one when
    ``target_update_freq == 0``), projected onto the support from the clamped n-step returns.  A prioritised buffer's
    importance weight scales each row's cross-entropy in the loss; ``batch.weight`` leaves the update as the unweighted
    cross-entropy, the priority the buffer is updated with.
    """

    def __init__(self, *, policy: C51Policy, optim: OptimizerFactory, gamma: float = 0.99, n_step_return_horizon: int = 1,
                 target_update_freq: int = 0) -> None:
        super().__init__(policy=policy)
        assert 0.0 <= gamma <= 1.0, f"discount factor should be in [0, 1] but got: {gamma}"
        assert n_step_return_horizon > 0, f"n_step_return_horizon should be greater than 0 but got: {n_step_return_horizon}"
        self.gamma = gamma
        self.n_step = n_step_return_horizon
        self.target_update_freq = target_update_freq
        self.delta_z = (policy.v_max - policy.v_min) / (policy.num_atoms - 1)
        dev = cuda_device_of(policy.model)
        self._build_network(policy, dev)
        self.optim = self._create_optimizer(policy, optim)
        bind_optimizer(self.optim, self._group, frozen=(policy.support, *self._frozen_params()))
        self.model_old: nn.Module | None = None
        self._g_old: FlatGroup | None = None
        if self.use_target_network:
            self._build_lagged(policy)

    def _build_network(self, policy: C51Policy, dev: torch.device) -> None:
        """Read ``policy.model`` as a layer chain over ``actions * num_atoms`` logits whose module applies a softmax over each
        action's atoms; refuse anything else."""
        N = policy.num_atoms
        inner, in_shape, in_scale = describe_q_network(policy.model)
        n_actions = int(policy.action_space.n)
        layers = atom_chain(inner, in_shape, n_actions, N, "categorical", "atoms")
        per_action_softmax = (isinstance(inner, C51Net) and inner.num_atoms == N) or \
            (getattr(inner, "softmax", False) and getattr(inner, "num_atoms", 1) == N)
        if not per_action_softmax:
            raise UnsupportedModelError(f"C51 reads the network output as probabilities over {N} atoms per action: build "
                                        f"Net(softmax=True, num_atoms={N}) or C51Net, got {type(inner).__name__} without that "
                                        "softmax")
        self._init_discrete(dev, in_shape, in_scale, n_actions)
        self._group = FlatGroup(layer_params(layers), dev)
        self._net = FusedStack(layers, self._group, "c51")

    def _frozen_params(self) -> tuple[nn.Parameter, ...]:
        """Parameters of ``policy.model`` that the optimiser lists but never steps."""
        return ()

    def _build_lagged(self, policy: C51Policy) -> None:
        self.model_old = _EvalModeModule(deepcopy(policy.model))
        self._g_old = lagged_group(self._group, list(self.model_old.parameters()))

    def _logits(self, src: Any, tag: str, lagged: bool = False) -> tuple[torch.Tensor, Any]:
        """The raw ``[B, A * N]`` logits of the online (``lagged``: the lagged) network at the observation source ``src``, and
        what ``_backward`` needs of that pass."""
        params = None
        if lagged:
            self._g_old.ensure_adopted()
            params = self._g_old.flat
        acts = self._net.forward(src.x, src.rows, tag, frames=src.frames, params=params)
        return acts[-1], acts

    def _backward(self, acts: Any, dlogits: torch.Tensor, rows: int) -> None:
        """Store d loss / d parameters in the group's gradient from d loss / d logits of the ``"up"`` pass."""
        self._net.backward(acts, dlogits, rows, "up")

    @property
    def use_target_network(self) -> bool:
        return self.target_update_freq > 0

    # ------------------------------------------------------------------ target
    def _target_q(self, buffer: ReplayBuffer, indices: np.ndarray) -> torch.Tensor:
        """The support repeated per row (c51.py:110-111): ``returns`` becomes ``r_n + gamma^n * support * mask``."""
        return self.policy.support.repeat(len(indices), 1)

    def _preprocess_batch(self, batch: Batch, buffer: ReplayBuffer, indices: np.ndarray) -> Batch:
        batch = super()._preprocess_batch(batch, buffer, indices)
        batch.__dict__["obs_next"] = self._obs_source(buffer, indices, "obs_next")
        return batch

    def _target_dist(self, batch: Batch) -> torch.Tensor:
        """The distribution of Q_old(s', argmax_a sum_k p_ak z_k) over the atoms, ``[B, N]``   (c51.py:113-124)."""
        src = batch.obs_next
        B = src.rows
        logits_on = self._logits(src, "tq_on")[0]
        logits_next = logits_on
        if self.use_target_network:
            logits_next = self._logits(src, "tq_old", lagged=True)[0]
        out = self._buf("next_dist", (B, self.policy.num_atoms))
        call("ts_c51_target", ptr(logits_on), ptr(logits_next), ptr(self.policy.support), B, self.n_actions, self.policy.num_atoms,
             ptr(out), None, stream_ptr(self._dev))
        return out

    # ------------------------------------------------------------------ update
    def _update_with_batch(self, batch: Batch) -> LossSequenceTrainingStats:
        self._tick_lagged(self.target_update_freq)
        next_dist = self._target_dist(batch)
        pol = self.policy
        src = batch.obs
        B, A, N = src.rows, self.n_actions, pol.num_atoms
        weight = pop_batch_weight(batch, self._dev)
        logits, acts = self._logits(src, "up")
        returns = batch.returns.reshape(B, N).to(self._dev, torch.float32).contiguous()
        dlogits, prio = self._buf("dlogits", (B, A * N)), self._buf("prio", B)
        rows, losses = self._buf("loss_rows", (3, B)), self._buf("losses", 4)
        call("ts_c51_rows", ptr(logits), ptr(batch.act), ptr(returns), ptr(pol.support), float(pol.v_min), float(pol.v_max),
             float(self.delta_z), ptr(next_dist), ptr(weight), B, A, N, ptr(dlogits), ptr(prio), ptr(rows), ptr(losses),
             stream_ptr(self._dev))
        batch.weight = prio                     # prio-buffer
        self._backward(acts, dlogits, B)
        self._group.adam_step(self.optim._optim, self.optim._max_grad_norm)
        return LossSequenceTrainingStats(loss=float(losses[0].item()))      # the only host read of the loss
