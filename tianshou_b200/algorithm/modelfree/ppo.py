"""PPO with the whole ``update()`` on the device.

Reference: tianshou/algorithm/modelfree/ppo.py:16-224 (constructor kwargs :19-37, logp_old
:146-162, minibatch loop :164-224).

Per ``update(buffer, batch_size, repeat)``:
  host : bulk H2D of the rollout (``_sample``), ``np.random.permutation`` per repeat (the
         reference's *global numpy RNG* draw of ``Batch.split``, batch.py:1209, kept so that
         minibatch composition is bit-identical), one D2H of the per-step loss table.
  GPU  : critic x2 -> GAE scan (+ return scaling + RunningMeanStd) -> actor log-prob, then for
         every minibatch: fused forward/backward + loss (``ts_ppo_grad``), global-norm clip +
         Adam (``ts_clip_adam_step``).  With >1 ranks each rank processes its slice of the
         minibatch and one all-reduce of (gradient, loss sums) precedes the Adam step.

``minibatch_shuffle="device"`` replaces the host permutation by a keyed bijection generated on
the GPU (algorithm/minibatch_order.py).  The index stream then differs from the reference's (same
distribution, different RNG) -- opt-in.
"""
from __future__ import annotations

import ctypes as C
from typing import Any, Literal

import torch

from ... import ops
from ..._cabi import LOSS_A2C, call, ptr, stream_ptr
from ...data import Batch, ReplayBuffer
from ...data.batch import minibatch_bounds
from ...parallel import allreduce_sum_
from ..minibatch_order import shared_slice
from ..optim import OptimizerFactory
from .a2c import A2CTrainingStats, ActorCriticOnPolicyAlgorithm
from .reinforce import ProbabilisticActorPolicy


class FusedActorCriticUpdate(ActorCriticOnPolicyAlgorithm):
    """The repeat x minibatch loop shared by PPO and A2C as device work: per pass ONE persistent launch covering every
    optimiser step (single GPU), the same launch with the gradient all-reduce fused in (multi GPU, NVLink peer memory),
    or the per-step NCCL fallback.  Subclasses provide ``_preprocess_batch`` and ``_loss_hparams``."""

    recompute_adv: bool = False
    advantage_normalization: bool = False

    def _loss_hparams(self) -> Any:
        raise NotImplementedError

    def _one_pass(self, batch: Batch, perm_r: torch.Tensor, bounds: list[tuple[int, int]], hp: Any, stats: torch.Tensor,
                  r: int, rank: int, wsize: int) -> None:
        """Pass r over the minibatches in the order ``perm_r`` (optional advantage recompute first, ppo.py:174-178)."""
        if self.recompute_adv and r > 0:
            self._add_returns_and_advantages(batch, None, None)
        if self.rollout_partition == "shared":
            perm_r, bounds = shared_slice(perm_r, bounds, rank, wsize)
        if self._peer_exchange(bounds) is not None:
            self._fused_distributed_pass(batch, perm_r, bounds, hp, stats, rank, wsize)
        else:
            self._distributed_repeat(batch, perm_r, bounds, hp, stats, rank, wsize)

    # ------------------------------------------------------------------ update
    def _update_with_batch(self, batch: Batch, batch_size: int | None, repeat: int) -> A2CTrainingStats:
        """The repeat x minibatch loop of ppo.py:164-224 as device work."""
        N = batch.obs.shape[0]
        with self._minibatch_order(repeat, N) as order:
            if self._layered is not None:    # networks outside the fused kernels' envelope: layer-wise tensor-core path
                from ..layered import layered_update
                stats = layered_update(self, batch, batch_size, repeat, order)
            else:
                bounds = minibatch_bounds(N, batch_size or N, merge_last=True)
                n_mb = len(bounds)
                hp = self._loss_hparams()
                stats = self._alloc_stats(repeat * n_mb)
                rank, wsize = self._ranks()
                if wsize == 1:       # every pass of the update in ONE asynchronous C call
                    self._device_passes(batch, order.rows, bounds, hp, stats, repeat, self.recompute_adv, feed=order.feed)
                else:                # pass by pass: the exchange set-up is host-driven
                    for r in range(repeat):
                        order.ready(r)
                        self._one_pass(batch, order.rows[r], bounds, hp, stats[r * n_mb:], r, rank, wsize)
            result = self._stats_from_device(stats)   # the only host sync of the update
        self._rms_end()
        self._flat.export_state(self.optim._optim)
        return result

    def _minibatch_adv_moments(self, batch: Batch, perm: torch.Tensor, lo: int, hi: int, world: int) -> torch.Tensor:
        """Advantage mean / std of minibatch ``perm[lo:hi]`` over every rank's slice (rows hi - lo per rank)."""
        st = stream_ptr(self.device)
        sums = self._buf("adv_sums", 2, torch.float64)
        call("ts_minibatch_adv_sums", ptr(batch.adv), ptr(perm), lo, hi, ptr(sums), st)
        if world > 1:
            allreduce_sum_(sums)
        adv_mom = self._buf("adv_mom", 2, torch.float32)
        call("ts_adv_moments_finalize", ptr(sums), (hi - lo) * world, ptr(adv_mom), st)
        return adv_mom

    def _device_passes(self, batch: Batch, perm_rows: torch.Tensor | None, bounds: list[tuple[int, int]], hp: Any,
                       stats: torch.Tensor, nrep: int, recompute: bool, feed: Any = None) -> None:
        """``nrep`` passes over the minibatches as ONE asynchronous C call (``ts_ppo_update_dedup``): per pass an
        optional critic + GAE recompute (with the alias map of the preprocess call, when the batch is still the one it was
        built from) and one persistent launch covering every optimiser step."""
        f, dev = self._flat, self.device
        N, n_mb = batch.obs.shape[0], len(bounds)
        adv_tmp = self._buf("adv_tmp", 32 + 8 * n_mb, torch.uint8)
        adv_tmp.zero_()
        bounds_c = (C.c_int64 * (2 * n_mb))(*[x for b in bounds for x in b])
        amap = self._next_alias_map(batch) if recompute else None
        call("ts_ppo_update_dedup", ptr(f.flat), ptr(f.grad), ptr(f.partials), ptr(f.exp_avg), ptr(f.exp_avg_sq), ptr(f.step_dev),
             C.byref(self._desc), C.byref(hp), ptr(batch.obs), ptr(batch.obs_next), ptr(batch.act),
             ptr(batch.rew), ptr(batch.terminated), ptr(batch.truncated), ptr(batch.get("_unfinished")),
             ptr(batch.v_s), ptr(batch.returns), ptr(batch.adv), ptr(batch.logp_old),
             ptr(self._buf("v_next", N, torch.float32)), N, ptr(perm_rows), nrep, bounds_c, n_mb,
             int(recompute), float(self.gamma), float(self.gae_lambda),
             ptr(self._rms_device()) if self.return_scaling else None, float(self._eps),
             ptr(self._gae_workspace(N)), ptr(adv_tmp), ptr(f.weight_image), ptr(stats), feed,
             *((ptr(amap.alias), ptr(amap.extra), ptr(amap.count)) if amap is not None else (None, None, None)), stream_ptr(dev))

    # ------------------------------------------------------------------ multi-GPU, fused (NVLink peer memory)
    def _peer_exchange(self, bounds: list[tuple[int, int]]):
        """The exchange buffers of the in-kernel all-reduce, created collectively on first use.  None ->
        NCCL path (``TS_B200_NO_P2P=1``, irregular minibatch bounds, a network the tensor-core kernels do
        not cover, or peer mapping unavailable)."""
        import os

        from ...parallel import PeerExchange
        if "peer_exchange" not in self._scratch:
            size = bounds[0][1] - bounds[0][0]
            regular = all(lo == bounds[0][0] + m * size and (m == len(bounds) - 1 or hi == lo + size)
                          for m, (lo, hi) in enumerate(bounds))
            # (decided once per algorithm instance from the first pass's bounds; "shared" slices are regular by construction)
            usable = (os.environ.get("TS_B200_NO_P2P", "0") != "1" and regular
                      and self._flat.weight_image is not None and os.environ.get("TS_B200_FORCE_SIMT", "0") != "1")
            # the decision must be identical on every rank: all inputs above are (shapes, env) -- replicas agree
            self._scratch["peer_exchange"] = PeerExchange.create(self._desc, self.device) if usable else None
        return self._scratch["peer_exchange"]

    def _fused_distributed_pass(self, batch: Batch, perm: torch.Tensor | None, bounds: list[tuple[int, int]], hp: Any,
                                stats: torch.Tensor, rank: int, wsize: int) -> None:
        """One pass over the minibatches of this rank's shard as ONE persistent launch; the gradient sum over
        the ranks happens inside the kernel (8-byte packets over NVLink, ``ts_ppo_epoch_multi``).  The only
        collective on the host side is the all-reduce of the per-minibatch advantage sums when
        ``advantage_normalization`` is on (2 * n_minibatch doubles per pass)."""
        f, st = self._flat, stream_ptr(self.device)
        ex = self._scratch["peer_exchange"]
        n_mb = len(bounds)
        lo0, size, end = bounds[0][0], bounds[0][1] - bounds[0][0], bounds[-1][1]
        adv_mom = None
        if self.advantage_normalization:
            sums = self._buf("epoch_adv_sums", 2 * n_mb, torch.float64)
            call("ts_epoch_adv_sums", ptr(batch.adv), ptr(perm), lo0, size, end, n_mb, ptr(sums), st)
            allreduce_sum_(sums)
            adv_mom = self._buf("epoch_adv_mom", 2 * n_mb, torch.float32)
            call("ts_epoch_adv_finalize", ptr(sums), lo0, size, end, n_mb, wsize, ptr(adv_mom), st)
        call("ts_ppo_epoch_multi", ptr(f.flat), ptr(f.grad), ptr(f.partials), ptr(f.exp_avg), ptr(f.exp_avg_sq), ptr(f.step_dev),
             C.byref(self._desc), C.byref(hp), ptr(batch.obs), ptr(batch.act), ptr(batch.adv), ptr(batch.returns),
             ptr(batch.logp_old), ptr(batch.v_s), ptr(perm), lo0, size, end, n_mb, ptr(adv_mom), ptr(f.weight_image),
             ptr(stats), rank, wsize, ex.ptrs, st)

    def _distributed_repeat(self, batch: Batch, perm: torch.Tensor, bounds: list[tuple[int, int]], hp: Any,
                            stats: torch.Tensor, rank: int, wsize: int) -> None:
        """One pass over the minibatches with the gradient all-reduce between backward and Adam.
        Every rank owns ITS OWN rollout shard (weak scaling): the global minibatch is the union of
        the ranks' local minibatches, so the mean's denominator is wsize * local rows."""
        f, dev = self._flat, self.device
        st = stream_ptr(dev)
        for m, (lo, hi) in enumerate(bounds):
            global_rows = (hi - lo) * wsize
            adv_mom = self._minibatch_adv_moments(batch, perm, lo, hi, wsize) if self.advantage_normalization else None
            n_part = C.c_int32(0)
            call("ts_ppo_grad", ptr(f.flat), C.byref(self._desc), C.byref(hp), ptr(batch.obs), ptr(batch.act),
                 ptr(batch.adv), ptr(batch.returns), ptr(batch.logp_old), ptr(batch.v_s), ptr(perm), lo, hi,
                 global_rows, ptr(adv_mom), ptr(f.partials), C.byref(n_part), st)
            call("ts_grad_reduce", ptr(f.partials), n_part.value, C.byref(self._desc), ptr(f.grad), st)
            allreduce_sum_(f.grad)   # ONE collective per optimiser step: grads + loss sums
            call("ts_clip_adam_step", ptr(f.flat), ptr(f.grad), None, 0, ptr(f.exp_avg), ptr(f.exp_avg_sq), ptr(f.step_dev),
                 C.byref(self._desc), C.byref(hp), ptr(stats[m]), st)



class PPO(FusedActorCriticUpdate):
    """Proximal Policy Optimization (arXiv:1707.06347), clip variant with optional dual clip,
    value clip, advantage normalisation and per-repeat advantage recomputation."""

    def __init__(
        self,
        *,
        policy: ProbabilisticActorPolicy,
        critic: torch.nn.Module,
        optim: OptimizerFactory,
        eps_clip: float = 0.2,
        dual_clip: float | None = None,
        value_clip: bool = False,
        advantage_normalization: bool = True,
        recompute_advantage: bool = False,
        vf_coef: float = 0.5,
        ent_coef: float = 0.01,
        max_grad_norm: float | None = None,
        gae_lambda: float = 0.95,
        max_batchsize: int = 256,
        gamma: float = 0.99,
        return_scaling: bool = False,
        minibatch_shuffle: Literal["numpy", "device"] = "numpy",
        shuffle_seed: int = 0,
        rollout_partition: Literal["per_rank", "shared"] = "per_rank",
        data_parallel: bool = True,
    ) -> None:
        assert dual_clip is None or dual_clip > 1.0, (
            f"Dual-clip PPO parameter should greater than 1.0 but got {dual_clip}")
        super().__init__(policy=policy, critic=critic, optim=optim, optim_include_actor=True,
                         max_grad_norm=max_grad_norm, gae_lambda=gae_lambda, max_batchsize=max_batchsize,
                         gamma=gamma, return_scaling=return_scaling, rollout_partition=rollout_partition,
                         data_parallel=data_parallel)
        self.vf_coef = vf_coef
        self.ent_coef = ent_coef
        self.eps_clip = eps_clip
        self.dual_clip = dual_clip
        self.value_clip = value_clip
        self.advantage_normalization = advantage_normalization
        self.recompute_adv = recompute_advantage
        if minibatch_shuffle not in ("numpy", "device"):
            raise ValueError(f"minibatch_shuffle must be 'numpy' or 'device', got {minibatch_shuffle!r}")
        self.minibatch_shuffle = minibatch_shuffle
        self._shuffle_seed = shuffle_seed

    # ------------------------------------------------------------------ preprocess
    def _preprocess_batch(self, batch: Batch, buffer: ReplayBuffer, indices: Any) -> Batch:
        """returns / advantages / logp_old on the device (ppo.py:146-162)."""
        self._rms_begin()
        if self.recompute_adv:
            self._buffer, self._indices = buffer, indices
        batch = self._add_returns_and_advantages(batch, buffer, indices)
        n = batch.obs.shape[0]
        logp_old = self._buf("logp_old", n, torch.float32)
        if self._layered is not None:
            self._layered.actor_logp(batch.obs, batch.act, logp_old, self._loss_hparams())
        else:
            ops.actor_logp(self._flat.flat, self._desc, batch.obs, batch.act, out=logp_old)
        batch.__dict__["logp_old"] = logp_old
        return batch

    def _ppo_hparams(self):
        return self._hparams(
            eps_clip=float(self.eps_clip), dual_clip=float(self.dual_clip or 0.0), vf_coef=float(self.vf_coef),
            ent_coef=float(self.ent_coef), value_clip=int(bool(self.value_clip)),
            advantage_normalization=int(bool(self.advantage_normalization)))

    _loss_hparams = _ppo_hparams


class A2C(FusedActorCriticUpdate):
    """Synchronous Advantage Actor-Critic (arXiv:1602.01783); reference: a2c.py:156-299.  Same device path as PPO with
    the actor loss ``-(log_prob * adv).mean()`` (``TS_LOSS_A2C``), plain MSE value loss, no clipping."""

    def __init__(self, *, policy: ProbabilisticActorPolicy, critic: torch.nn.Module, optim: OptimizerFactory,
                 vf_coef: float = 0.5, ent_coef: float = 0.01, max_grad_norm: float | None = None,
                 gae_lambda: float = 0.95, max_batchsize: int = 256, gamma: float = 0.99, return_scaling: bool = False,
                 minibatch_shuffle: Literal["numpy", "device"] = "numpy", shuffle_seed: int = 0) -> None:
        super().__init__(policy=policy, critic=critic, optim=optim, optim_include_actor=True,
                         max_grad_norm=max_grad_norm, gae_lambda=gae_lambda, max_batchsize=max_batchsize,
                         gamma=gamma, return_scaling=return_scaling)
        self.vf_coef = vf_coef
        self.ent_coef = ent_coef
        if minibatch_shuffle not in ("numpy", "device"):
            raise ValueError(f"minibatch_shuffle must be 'numpy' or 'device', got {minibatch_shuffle!r}")
        self.minibatch_shuffle = minibatch_shuffle
        self._shuffle_seed = shuffle_seed

    def _preprocess_batch(self, batch: Batch, buffer: ReplayBuffer, indices: Any) -> Batch:
        """returns / advantages on the device (a2c.py:239-247); the A2C loss needs no behaviour log-prob."""
        self._rms_begin()
        batch = self._add_returns_and_advantages(batch, buffer, indices)
        n = batch.obs.shape[0]
        batch.__dict__["logp_old"] = self._buf("logp_old", n, torch.float32).zero_()     # unused by TS_LOSS_A2C
        return batch

    def _loss_hparams(self) -> Any:
        return self._hparams(eps_clip=0.0, dual_clip=0.0, vf_coef=float(self.vf_coef), ent_coef=float(self.ent_coef),
                             value_clip=0, advantage_normalization=0, loss_kind=LOSS_A2C)
