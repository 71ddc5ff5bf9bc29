"""Natural Policy Gradient with the whole ``update()`` on the device.

Reference: tianshou/algorithm/modelfree/npg.py (NPGTrainingStats :20-24, constructor :33-121, preprocessing :123-138,
minibatch loop :140-187, MVP :189-200, conjugate gradient :202-224).

Per minibatch, with no host round trip: actor forward (once, reused by every Fisher-vector product), surrogate rows and the
vanilla gradient (backward GEMMs), 10 conjugate-gradient iterations -- each one Fisher-vector product ``J^T H J v`` (a tangent
pass ``FusedStack.jvp``, the KL-Hessian rows ``ts_npg_fvp_rows``, a backward pass) and one ``ts_cg_step`` whose scalars and
early-exit flag stay in device memory -- then the natural step, the KL statistic and ``optim_critic_iters`` Adam steps on the
critic.  One D2H of the per-minibatch statistics table ends the update.  The actor and the critic are layer-wise networks
(algorithm/layered.py) with one parameter group each: the torch optimiser covers ``critic.parameters()`` only, as in the
reference.  Single GPU; shared actor / critic trunks are refused.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Any

import numpy as np
import torch

from ... import ops
from ..._cabi import call, ptr, stream_ptr
from ...data import Batch, ReplayBuffer, SequenceSummaryStats
from ...data.batch import minibatch_bounds
from ..base import TrainingStats
from ..flat_params import UnsupportedModelError
from ..netgraph import ACT_NONE
from ..optim import OptimizerFactory
from .a2c import ActorCriticOnPolicyAlgorithm
from .reinforce import ProbabilisticActorPolicy

# columns of the per-minibatch statistics table
COL_ACTOR_LOSS, COL_VF_LOSS, COL_KL, COL_STEP_SIZE, COL_CG_ITERS, COL_ACCEPTED, COL_FAILED = range(7)
CG_ITERS = 10                   # npg.py:160 nsteps
CG_RESIDUAL_TOL = 1e-10         # npg.py:207


@dataclass(kw_only=True)
class NPGTrainingStats(TrainingStats):
    actor_loss: SequenceSummaryStats
    vf_loss: SequenceSummaryStats
    kl: SequenceSummaryStats


class NPG(ActorCriticOnPolicyAlgorithm):
    """Natural Policy Gradient (https://proceedings.neurips.cc/paper/2001/file/4b86abe48d358ecf194c56c69108433e-Paper.pdf)."""

    _ratio_surrogate = False

    def __init__(self, *, policy: ProbabilisticActorPolicy, critic: torch.nn.Module, optim: OptimizerFactory,
                 optim_critic_iters: int = 5, trust_region_size: float = 0.5, advantage_normalization: bool = True,
                 gae_lambda: float = 0.95, max_batchsize: int = 256, gamma: float = 0.99, return_scaling: bool = False) -> None:
        super().__init__(policy=policy, critic=critic, optim=optim, optim_include_actor=False, gae_lambda=gae_lambda,
                         max_batchsize=max_batchsize, gamma=gamma, return_scaling=return_scaling)
        self.advantage_normalization = advantage_normalization
        self.optim_critic_iters = optim_critic_iters
        self.trust_region_size = trust_region_size
        self._damping = 0.1      # npg.py:121
        self.last_stats_table: np.ndarray | None = None

    # ------------------------------------------------------------------ preprocess
    def _preprocess_batch(self, batch: Batch, buffer: ReplayBuffer, indices: Any) -> Batch:
        """returns / advantages, logp_old and the whole-batch advantage normalisation on the device (npg.py:123-138)."""
        self._rms_begin()
        batch = self._add_returns_and_advantages(batch, buffer, indices)
        n = batch.obs.shape[0]
        logp_old = self._buf("logp_old", n, torch.float32)
        self._layered.actor_logp(batch.obs, batch.act, logp_old, self._hparams())
        batch.__dict__["logp_old"] = logp_old
        if self.advantage_normalization:
            call("ts_npg_normalize_adv", ptr(batch.adv), n, stream_ptr(self.device))
        return batch

    # ------------------------------------------------------------------ update
    def _update_with_batch(self, batch: Batch, batch_size: int | None, repeat: int) -> NPGTrainingStats:
        """The repeat x minibatch loop of npg.py:140-187 / trpo.py:99-200; the statistics table is the one host read."""
        if self.minibatch_shuffle != "numpy":
            raise UnsupportedModelError("NPG / TRPO draw the reference's minibatch order (numpy's global stream) only; "
                                        "the device-generated order is unsupported")
        N = batch.obs.shape[0]
        bounds = minibatch_bounds(N, batch_size or N, merge_last=True)
        n_mb = len(bounds)
        stats = self._alloc_stats(repeat * n_mb)
        with self._minibatch_order(repeat, N) as order:
            for r in range(repeat):
                order.ready(r)
                for m, (lo, hi) in enumerate(bounds):
                    self._minibatch(batch, order.rows[r, lo:hi].to(torch.int64), stats[r * n_mb + m])
            table = stats.cpu().numpy().astype(np.float64)      # the only host sync
        self._rms_end()
        self._flat.export_state(self.optim._optim)
        self.last_stats_table = table
        return self._training_stats(table)

    def _training_stats(self, table: np.ndarray) -> NPGTrainingStats:
        return NPGTrainingStats(actor_loss=SequenceSummaryStats.from_sequence(table[:, COL_ACTOR_LOSS]),
                                vf_loss=SequenceSummaryStats.from_sequence(table[:, COL_VF_LOSS]),
                                kl=SequenceSummaryStats.from_sequence(table[:, COL_KL]))

    # ------------------------------------------------------------------ one minibatch
    def _minibatch(self, batch: Batch, idx: torch.Tensor, row: torch.Tensor) -> None:
        L = self._layered
        g = L.group
        st = stream_ptr(self.device)
        B, A, n = int(idx.numel()), L.act_dim, g.n
        cat = int(L.categorical)
        obs = ops.gather_rows(batch.obs, idx)
        act = ops.gather_rows(L._act_rows(batch.act), idx)
        adv, ret, lpo = ops.gather_rows(batch.adv, idx), ops.gather_rows(batch.returns, idx), ops.gather_rows(batch.logp_old, idx)
        at = L.a_trunk.forward(obs, B, "up")
        ah = L.a_head.forward(at[-1], B, "up")
        head = ah[-1]
        # vanilla gradient of the surrogate (npg.py:150-157, trpo.py:132-141)
        loss_rows = L._buf("npg_loss", B)
        dhead = L._buf("dhead", (B, A))
        dls = None if cat else L._buf("dls", (B, A))
        call("ts_npg_rows", ptr(head), L._logstd_ptr(g.flat), ptr(act), ptr(adv), ptr(lpo), B, A, cat, int(self._ratio_surrogate),
             ptr(loss_rows), ptr(dhead), ptr(dls), st)
        call("ts_npg_mean_rows", ptr(loss_rows), B, row.data_ptr() + 4 * COL_ACTOR_LOSS, st)
        self._actor_backward(at, ah, dhead, B)
        if dls is not None:
            call("ts_net_colsum", ptr(dls), A, B, A, L._logstd_ptr(g.grad), 0, st)
        # natural direction: conjugate gradient on MVP(v) = F v + damping v (npg.py:158-162, 202-224)
        x, r, p = L._buf("cg_x", n), L._buf("cg_r", n), L._buf("cg_p", n)
        state = L._buf("cg_state", 3, torch.float64)
        call("ts_cg_init", ptr(g.grad), ptr(x), ptr(r), ptr(p), n, ptr(state), st)
        for _ in range(CG_ITERS):
            self._fvp(at, ah, p, B)
            call("ts_cg_step", ptr(x), ptr(r), ptr(p), ptr(g.grad), n, self._damping, CG_RESIDUAL_TOL, ptr(state),
                 row.data_ptr() + 4 * COL_CG_ITERS, st)
        self._actor_step(at, ah, x, obs, act, adv, lpo, B, row)          # search direction s = -x
        self._critic_steps(obs, ret, B, row)

    def _actor_step(self, at: list[torch.Tensor], ah: list[torch.Tensor], x: torch.Tensor, obs: torch.Tensor, act: torch.Tensor,
                    adv: torch.Tensor, lpo: torch.Tensor, B: int, row: torch.Tensor) -> None:
        """npg.py:164-172: theta += trust_region_size * s, kl = KL(old || new) at the new parameters."""
        g, st = self._layered.group, stream_ptr(self.device)
        cand = self._layered._buf("cand", g.n)
        call("ts_npg_axpy", ptr(cand), ptr(g.flat), ptr(x), -float(self.trust_region_size), None, g.n, st)
        kl_rows, _ = self._candidate_kl(ah[-1], cand, obs, B)
        call("ts_npg_mean_rows", ptr(kl_rows), B, row.data_ptr() + 4 * COL_KL, st)
        g.flat.copy_(cand)

    def _candidate_kl(self, head_old: torch.Tensor, cand: torch.Tensor, obs: torch.Tensor, B: int
                      ) -> tuple[torch.Tensor, torch.Tensor]:
        """Forward pass at the candidate parameters ``cand``: (KL(old || candidate) rows, the candidate's head outputs)."""
        L, st = self._layered, stream_ptr(self.device)
        t = L.a_trunk.forward(obs, B, "cand", params=cand)
        head = L.a_head.forward(t[-1], B, "cand", params=cand)[-1]
        kl_rows = L._buf("kl_rows", B)
        call("ts_npg_kl_rows", ptr(head_old), L._logstd_ptr(L.group.flat), ptr(head), L._logstd_ptr(cand), B, L.act_dim,
             int(L.categorical), ptr(kl_rows), st)
        return kl_rows, head

    def _actor_backward(self, at: list[torch.Tensor], ah: list[torch.Tensor], dhead: torch.Tensor, B: int) -> None:
        """Head-output gradient -> actor weight / bias gradients (stored into the actor group's gradient buffer)."""
        L = self._layered
        dz = L._buf("dz_a", (B, L.a_trunk.layers[-1].out_dim))
        L.a_head.backward(ah, dhead, B, "up", input_grad=True, input_act=(L._a_act, at[-1]) if L._a_act != ACT_NONE else None,
                          dx_out=dz)
        L.a_trunk.backward(at, dz, B, "up", dy_preact=True)

    def _fvp(self, at: list[torch.Tensor], ah: list[torch.Tensor], v: torch.Tensor, B: int) -> None:
        """Actor group gradient buffer <- F v = J^T H J v (without damping): tangent pass, KL-Hessian rows, backward pass."""
        L = self._layered
        tt = L.a_trunk.jvp(at, v, B, "up")
        ht = L.a_head.jvp(ah, v, B, "up", x_dot=tt[-1])
        rows = L._buf("fvp_rows", (B, L.act_dim))
        call("ts_npg_fvp_rows", ptr(ah[-1]), ptr(ht[-1]), L._logstd_ptr(L.group.flat), L._logstd_ptr(v), B, L.act_dim,
             int(L.categorical), ptr(rows), L._logstd_ptr(L.group.grad), stream_ptr(self.device))
        self._actor_backward(at, ah, rows, B)

    def _critic_steps(self, obs: torch.Tensor, ret: torch.Tensor, B: int, row: torch.Tensor) -> None:
        """optim_critic_iters x (F.mse_loss(returns, critic(obs)), optimiser step) (npg.py:175-179); vf_loss = the last one."""
        L, st = self._layered, stream_ptr(self.device)
        td, dval, vrows = L._buf("vf_td", B), L._buf("dval", (B, 1)), L._buf("vf_rows", B)
        dz = L._buf("dz_c", (B, L.c_trunk.layers[-1].out_dim))
        for _ in range(self.optim_critic_iters):
            ct = L.c_trunk.forward(obs, B, "up")
            ch = L.c_head.forward(ct[-1], B, "up")
            call("ts_critic_mse", ptr(ch[-1]), ptr(ret), None, B, ptr(td), ptr(dval), ptr(vrows), st)
            call("ts_mean", ptr(vrows), B, row.data_ptr() + 4 * COL_VF_LOSS, st)
            L.c_head.backward(ch, dval, B, "up", input_grad=True, input_act=(L._c_act, ct[-1]) if L._c_act != ACT_NONE else None,
                              dx_out=dz)
            L.c_trunk.backward(ct, dz, B, "up", dy_preact=True)
            L.critic_group.optimizer_step(self.optim._optim, None)
