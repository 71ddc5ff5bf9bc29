"""Trust Region Policy Optimization with the whole ``update()`` on the device.

Reference: tianshou/algorithm/modelfree/trpo.py (TRPOTrainingStats :19-21, constructor :27-129, minibatch loop :131-200).
Same device pipeline as NPG (npg.py here), with the ratio surrogate, the step size ``sqrt(2 max_kl / (s . MVP(s)))`` from one
more Fisher-vector product, and the backtracking line search: per candidate one actor forward pass at ``theta + step * s``,
the KL / surrogate rows, and ``ts_trpo_decide`` (acceptance, step shrink or failure in device memory).  The host reads one
4-byte flag per evaluated candidate -- the reference compares on the host at the same point -- and nothing else until the
statistics table.
"""
from __future__ import annotations

import warnings
from dataclasses import dataclass

import numpy as np
import torch

from ..._cabi import call, ptr, stream_ptr
from ...data import SequenceSummaryStats
from ..optim import OptimizerFactory
from .npg import COL_ACCEPTED, COL_FAILED, COL_STEP_SIZE, NPG, NPGTrainingStats
from .reinforce import ProbabilisticActorPolicy


@dataclass(kw_only=True)
class TRPOTrainingStats(NPGTrainingStats):
    step_size: SequenceSummaryStats


class TRPO(NPG):
    """Trust Region Policy Optimization (arXiv:1502.05477)."""

    _ratio_surrogate = True

    def __init__(self, *, policy: ProbabilisticActorPolicy, critic: torch.nn.Module, optim: OptimizerFactory, max_kl: float = 0.01,
                 backtrack_coeff: float = 0.8, max_backtracks: int = 10, optim_critic_iters: int = 5, trust_region_size: float = 0.5,
                 advantage_normalization: bool = True, gae_lambda: float = 0.95, max_batchsize: int = 256, gamma: float = 0.99,
                 return_scaling: bool = False) -> None:
        super().__init__(policy=policy, critic=critic, optim=optim, optim_critic_iters=optim_critic_iters,
                         trust_region_size=trust_region_size, advantage_normalization=advantage_normalization, gae_lambda=gae_lambda,
                         max_batchsize=max_batchsize, gamma=gamma, return_scaling=return_scaling)
        self.max_backtracks = max_backtracks
        self.max_kl = max_kl
        self.backtrack_coeff = backtrack_coeff

    def _actor_step(self, at: list[torch.Tensor], ah: list[torch.Tensor], x: torch.Tensor, obs: torch.Tensor, act: torch.Tensor,
                    adv: torch.Tensor, lpo: torch.Tensor, B: int, row: torch.Tensor) -> None:
        """trpo.py:152-186 with the search direction s = -x (s . MVP(s) = x . MVP(x))."""
        L = self._layered
        g, st = L.group, stream_ptr(self.device)
        step = L._buf("trpo_step", 1)
        self._fvp(at, ah, x, B)
        call("ts_trpo_step_size", ptr(x), ptr(g.grad), g.n, self._damping, float(self.max_kl), ptr(step), ptr(row), st)
        cand = L._buf("cand", g.n)
        loss_rows = L._buf("cand_loss", B)
        flag = L._buf("trpo_flag", 1, torch.int32)
        for i in range(self.max_backtracks):
            call("ts_npg_axpy", ptr(cand), ptr(g.flat), ptr(x), -1.0, ptr(step), g.n, st)
            kl_rows, head = self._candidate_kl(ah[-1], cand, obs, B)
            call("ts_npg_rows", ptr(head), L._logstd_ptr(cand), ptr(act), ptr(adv), ptr(lpo), B, L.act_dim, int(L.categorical), 1,
                 ptr(loss_rows), None, None, st)
            call("ts_trpo_decide", ptr(loss_rows), ptr(kl_rows), B, i, self.max_backtracks, float(self.max_kl),
                 float(self.backtrack_coeff), ptr(step), ptr(row), ptr(flag), st)
            decision = self._read_flag(flag)
            if decision == 1:
                g.flat.copy_(cand)
            if decision != 0:
                break

    @staticmethod
    def _read_flag(flag: torch.Tensor) -> int:
        """The line search's one host read per candidate (trpo.py:180 compares on the host as well)."""
        return int(flag.item())

    def _training_stats(self, table: np.ndarray) -> TRPOTrainingStats:
        for row in table:                 # the reference's warnings, in minibatch order (trpo.py:181-190)
            if row[COL_ACCEPTED] > 0:
                warnings.warn(f"Backtracking to step {int(row[COL_ACCEPTED])}.")
            if row[COL_FAILED] != 0:
                warnings.warn("Line search failed! It seems hyperparamters are poor and need to be changed.")
        base = super()._training_stats(table)
        return TRPOTrainingStats(actor_loss=base.actor_loss, vf_loss=base.vf_loss, kl=base.kl,
                                 step_size=SequenceSummaryStats.from_sequence(table[:, COL_STEP_SIZE]))
