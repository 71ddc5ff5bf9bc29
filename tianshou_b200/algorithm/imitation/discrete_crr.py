"""Discrete critic-regularised regression (arXiv:2006.15134) with the whole ``update()`` on the device.

Reference: tianshou/algorithm/imitation/discrete_crr.py (DiscreteCRR :33-167), modelfree/reinforce.py:249-312
(``DiscountedReturnComputation``), utils/lagged_network.py:81-87 (the full lagged copy), examples/offline/atari_crr.py:105-124
and test/offline/test_discrete_crr.py:69-84 (the actor and the critic on ONE preprocess network).

Per ``update(buffer, sample_size)``:
  host : index draw from the buffer's RNG streams, the drawn rows' reward / done / action upload, one D2H of the four loss scalars.
  GPU  : observation sources of s and s' -> trunk + actor and critic heads on s, lagged trunk + heads on s' ->
         ``ts_discrete_crr_rows`` (one-step target, the three losses, d loss / d q, d loss / d logits) -> both heads' backward GEMMs
         into one trunk gradient -> trunk backward -> one Adam step over the whole flat group; the lagged copy is one memcpy.
Every Linear / Conv2d layer's forward, input gradient and weight gradient is one wgmma GEMM launch (csrc/net_gemm.cu); the two
heads on one trunk are shared_trunk.py's.
"""
from __future__ import annotations

from copy import deepcopy
from dataclasses import dataclass
from typing import Any, Literal

import numpy as np
import torch
from torch import nn

from ..._cabi import ABI, call, ptr, stream_ptr, to_device
from ...data import Batch, ReplayBuffer
from ..base import OfflineAlgorithm
from ..discrete_q import DiscreteQCore, lagged_group
from ..flat_params import FlatGroup, UnsupportedModelError, bind_optimizer
from ..modelfree.dqn import SimpleLossTrainingStats
from ..modelfree.reinforce import DiscreteActorPolicy
from ..optim import OptimizerFactory
from ..shared_trunk import TwoHeadNetwork, two_head_parameters
from ..twin_critic import _EvalModeModule, cuda_device_of

_MODES = {"exp": ABI.consts["TS_CRR_EXP"], "binary": ABI.consts["TS_CRR_BINARY"], "all": ABI.consts["TS_CRR_ALL"]}


@dataclass(kw_only=True)
class DiscreteCRRTrainingStats(SimpleLossTrainingStats):
    actor_loss: float
    critic_loss: float
    cql_loss: float


@dataclass
class DiscountedReturnComputation:
    """The settings of the reference's Monte-Carlo return computation (reinforce.py:249-312).  Discrete CRR reads ``gamma``
    from it and nothing else."""

    gamma: float = 0.99
    return_standardization: bool = False

    def __post_init__(self) -> None:
        assert 0.0 <= self.gamma <= 1.0, "discount factor gamma should be in [0, 1]"


class DiscreteCRR(DiscreteQCore, OfflineAlgorithm):
    """Discrete CRR, reference API and semantics (discrete_crr.py:33-167).

    The policy's actor (``DiscreteActor(softmax_output=False)``) and ``critic`` (``DiscreteCritic(last_size=n_actions)``) sit on
    the same preprocess network or on one each; one optimiser steps both over ``actor_loss + critic_loss + min_q_weight *
    cql_loss``.  Loss and gradient are the reference's as its code computes them, not the paper's: the advantage is not
    detached, so in ``"exp"`` mode the improvement coefficient carries gradient into the critic and the actor; and the product
    of ``-log_prob`` ``[B]`` with the coefficient ``[B, 1]`` broadcasts to ``[B, B]``, so ``actor_loss`` is
    ``mean(-log_prob) * mean(coefficient)``.  The target is one-step, on ``batch.done``.

    ``target_update_freq > 0``: the lagged actor and critic are copied when ``_iter % target_update_freq == 0``, before the
    step; both copies are taken at the same moment, so on the device they are one lagged flat buffer of the whole group, and
    ``critic_old``'s own copy of a shared trunk is kept equal to ``actor_old``'s.  ``0``: the lagged networks are the online
    ones.  ``_iter`` advances in the copy's tick, before the step, where the reference advances it after the step: after every
    completed update it holds the same count, and the copies fall on the same updates.

    ``batch.returns`` is not produced: the reference computes Monte-Carlo returns in ``_preprocess_batch`` and its loss never
    reads them, so parameters and statistics are the same with ``return_standardization`` on and off; the running return
    statistics that option would maintain are not kept.
    """

    def __init__(self, *, policy: DiscreteActorPolicy, critic: nn.Module, optim: OptimizerFactory, gamma: float = 0.99,
                 policy_improvement_mode: Literal["exp", "binary", "all"] = "exp", ratio_upper_bound: float = 20.0,
                 beta: float = 1.0, min_q_weight: float = 10.0, target_update_freq: int = 0,
                 return_standardization: bool = False) -> None:
        super().__init__(policy=policy)
        self.discounted_return_computation = DiscountedReturnComputation(gamma=gamma, return_standardization=return_standardization)
        if policy_improvement_mode not in _MODES:
            raise ValueError(f"policy_improvement_mode must be one of {sorted(_MODES)}, got {policy_improvement_mode!r}")
        self.critic = critic
        actor = policy.actor
        if getattr(actor, "softmax_output", False):
            raise UnsupportedModelError("DiscreteActor(softmax_output=True): discrete CRR reads the actor output as logits, "
                                        "probabilities would be treated as logits; build the actor with softmax_output=False")
        dev = cuda_device_of(actor, critic)
        self._group = FlatGroup(two_head_parameters(actor, critic), dev)
        self._net = TwoHeadNetwork(actor, critic, self._group, roles=("actor", "critic"))
        n_actions = int(policy.action_space.n)
        for name, n in zip(("actor", "critic"), self._net.n_out):
            if n != n_actions:
                raise UnsupportedModelError(f"{name} has {n} outputs for {n_actions} actions")
        self._init_discrete(dev, self._net.in_shape, self._net.in_scale, n_actions)
        self.optim = self._create_optimizer(nn.ModuleList([policy, critic]), optim)
        bind_optimizer(self.optim, self._group)
        self._target = target_update_freq > 0
        self._freq = target_update_freq
        self._g_old: FlatGroup | None = None
        if self._target:
            self.actor_old = _EvalModeModule(deepcopy(actor))
            self.critic_old = _EvalModeModule(deepcopy(critic))
            a_old, c_old = self.actor_old.module, self.critic_old.module
            # the online flat order with the lagged modules' parameters; of a shared trunk actor_old's copy is the one in it
            tail = c_old.last.parameters() if self._net.shared else c_old.parameters()
            self._g_old = lagged_group(self._group, [*a_old.parameters(), *tail])
        else:
            self.actor_old = actor
            self.critic_old = critic
        self._policy_improvement_mode = policy_improvement_mode
        self._ratio_upper_bound = ratio_upper_bound
        self._beta = beta
        self._min_q_weight = min_q_weight

    # ------------------------------------------------------------------ sampling
    def _sample(self, buffer: ReplayBuffer, sample_size: int | None) -> tuple[Batch, Any]:
        """The core's sample plus what the one-step target needs of the drawn rows: ``obs_next`` as a device observation
        source, ``rew`` and ``done`` as fp32 rows (``to_torch_as(batch.rew, q)``, ``batch.done > 0``)."""
        batch, indices = super()._sample(buffer, sample_size)
        batch.__dict__["obs_next"] = self._obs_source(buffer, indices, "obs_next")
        batch.__dict__["rew"] = to_device(np.asarray(buffer.rew)[indices].astype(np.float32).reshape(-1), self._dev)
        batch.__dict__["done"] = to_device(np.asarray(buffer.done)[indices].astype(np.float32).reshape(-1), self._dev)
        return batch, indices

    def _preprocess_batch(self, batch: Batch, buffer: ReplayBuffer, indices: np.ndarray) -> Batch:
        return batch

    # ------------------------------------------------------------------ update
    def _refresh_lagged(self) -> None:
        super()._refresh_lagged()
        if self._net.shared:
            with torch.no_grad():
                for tp, sp in zip(self.critic_old.module.preprocess.parameters(), self.actor_old.module.preprocess.parameters(),
                                  strict=True):
                    tp.copy_(sp)

    def _update_with_batch(self, batch: Batch) -> DiscreteCRRTrainingStats:
        self._tick_lagged(self._freq)
        src, src_next = batch.obs, batch.obs_next
        B, A = src.rows, self.n_actions
        on = self._net.forward(src, "up")
        if self._target:
            self._g_old.ensure_adopted()
        old = self._net.forward(src_next, "old", params=self._g_old.flat if self._target else None)
        dq, dlogits = self._buf("dq", (B, A)), self._buf("dlogits", (B, A))
        rows, losses = self._buf("loss_rows", 4 * B + 2), self._buf("losses", 4)
        call("ts_discrete_crr_rows", ptr(on.b[-1]), ptr(on.a[-1]), ptr(batch.act), ptr(old.b[-1]), ptr(old.a[-1]), ptr(batch.rew),
             ptr(batch.done), B, A, float(self.discounted_return_computation.gamma), _MODES[self._policy_improvement_mode],
             float(self._beta), float(self._ratio_upper_bound), float(self._min_q_weight), ptr(dq), ptr(dlogits), ptr(rows),
             ptr(losses), stream_ptr(self._dev))
        self._net.backward(on, dlogits, dq, "up")
        self._group.adam_step(self.optim._optim, self.optim._max_grad_norm)
        l = losses.cpu().numpy()                # the only host read of the losses
        return DiscreteCRRTrainingStats(loss=float(l[0]), actor_loss=float(l[1]), critic_loss=float(l[2]), cql_loss=float(l[3]))
