"""Actor-critic on-policy base: device-resident rollout, fused value pass + GAE.

Reference: tianshou/algorithm/modelfree/a2c.py (A2CTrainingStats :23-29,
ActorCriticOnPolicyAlgorithm :32-153, A2C :156-290).

What changes (same signatures, same 3-phase structure as ``Algorithm._update``):
  * ``_sample``: instead of a host fancy-index copy of every key (buffer_base.py:605-649,
    ~95 MB at 4096x128) the buffer's pinned numpy storage is uploaded once and, if the valid slots
    are not simply ``arange(N)``, gathered on the device by the ``sample_indices(0)`` kernel order.
    The returned ``Batch`` holds CUDA tensors.
  * ``_add_returns_and_advantages``: ONE fused critic kernel for v_s and v_s_ (replacing
    2*N/256 chunked forwards + H2D per chunk), then ``ts_gae`` with the return-scaling arithmetic
    and the RunningMeanStd merge folded in; nothing returns to the host.
"""
from __future__ import annotations

import contextlib
import ctypes as C
import os
import weakref
from abc import ABC
from dataclasses import dataclass
from typing import Any

import numpy as np
import torch

from ... import ops
from ..._cabi import GRAD_EXTRA, STATS_STRIDE, PPOHParams, load_library, to_device
from ...data import Batch, ReplayBuffer, SequenceSummaryStats
from ...parallel import world
from ...utils import RunningMeanStd
from ...utils.net.common import ActorCritic
from ..base import OnPolicyAlgorithm, TrainingStats
from ..flat_params import (
    DeviceScratch,
    FlatGroup,
    UnsupportedModelError,
    bind_optimizer,
    check_categorical_dist_fn,
    check_gaussian_dist_fn,
    optimizer_hyperparams,
)
from ..layered import LayeredActorCritic, fused_descriptor, parse_actor_critic
from ..minibatch_order import MinibatchOrder
from ..optim import OptimizerFactory
from .reinforce import ProbabilisticActorPolicy


@dataclass(kw_only=True)
class A2CTrainingStats(TrainingStats):
    loss: SequenceSummaryStats
    actor_loss: SequenceSummaryStats
    vf_loss: SequenceSummaryStats
    ent_loss: SequenceSummaryStats
    gradient_steps: int


def _upload(arr: np.ndarray, dev: torch.device, dtype: torch.dtype | None = None) -> torch.Tensor:
    t = to_device(arr, dev, non_blocking=True)
    if dtype is not None and t.dtype != dtype:
        t = t.to(dtype)
    return t


class ActorCriticOnPolicyAlgorithm(OnPolicyAlgorithm, ABC):
    """GAE-based actor-critic base (a2c.py:32-153) on the fused device path.

    Multi-GPU data parallelism (one process per GPU).  ``rollout_partition="per_rank"``: every rank's buffer is ITS OWN shard
    of the rollout (weak scaling: the global minibatch is the union of the ranks' local minibatches).  ``"shared"``: every
    rank holds the SAME rollout and draws the SAME permutation; each minibatch of B rows is split into world_size contiguous
    slices of B / world_size (SURVEY 8(e): a fixed problem, results comparable with a single-GPU / reference run on the same
    inputs).  ``data_parallel=False`` ignores an initialised process group (single-rank execution)."""

    minibatch_shuffle: str = "numpy"
    _shuffle_seed: int = 0
    _shuffle_epoch: int = 0

    def __init__(self, *, policy: ProbabilisticActorPolicy, critic: torch.nn.Module, optim: OptimizerFactory,
                 optim_include_actor: bool, max_grad_norm: float | None = None, gae_lambda: float = 0.95,
                 max_batchsize: int = 256, gamma: float = 0.99, return_scaling: bool = False,
                 rollout_partition: str = "per_rank", data_parallel: bool = True) -> None:
        super().__init__(policy=policy)
        if rollout_partition not in ("per_rank", "shared"):
            raise ValueError(f"rollout_partition must be 'per_rank' or 'shared', got {rollout_partition!r}")
        self.rollout_partition = rollout_partition
        self.data_parallel = bool(data_parallel)
        self._active_order: MinibatchOrder | None = None
        self._next_alias: tuple[Any, Any, ops.NextAliasMap] | None = None
        self.critic = critic
        assert 0.0 <= gae_lambda <= 1.0, f"GAE lambda should be in [0, 1] but got: {gae_lambda}"
        assert 0.0 <= gamma <= 1.0, f"discount factor gamma should be in [0, 1] but got: {gamma}"
        self.gae_lambda = gae_lambda
        self.max_batchsize = max_batchsize  # kept for API parity; the fused pass needs no chunking
        self._actor_critic = ActorCritic(self.policy.actor, self.critic)
        # kernel-side view of the networks.  Shapes outside the fused kernels' envelope (two 64-wide layers, obs <= 64) run
        # layer by layer on the tensor-core GEMM (algorithm/layered.py), and so does a critic-only optimiser (NPG / TRPO,
        # a2c.py:102-109: the actor moves along the natural gradient, while the fused kernels take one Adam step over both
        # networks); anything that is not a Linear / ReLU | Tanh actor-critic raises -- there is no eager-PyTorch path.
        self._spec = parse_actor_critic(self.policy.actor, self.critic, split=not optim_include_actor)
        dev = next(self.policy.actor.parameters()).device
        if dev.type != "cuda":
            raise UnsupportedModelError(
                f"actor/critic live on {dev}; tianshou_b200 has no CPU path -- move them to a CUDA device first")
        if self._spec.categorical:
            check_categorical_dist_fn(self.policy.dist_fn, self._spec.act_dim, dev)
        else:
            check_gaussian_dist_fn(self.policy.dist_fn, self._spec.act_dim, dev)
        force_layered = os.environ.get("TS_B200_FORCE_LAYERED", "0") == "1"      # tests: the layer-wise path on any shape
        fused = fused_descriptor(self._spec) if optim_include_actor and not force_layered else None
        if fused is None:
            self._desc, self._layered = None, LayeredActorCritic(self._spec, dev)
            if self._ranks()[1] > 1:
                raise UnsupportedModelError("the layer-wise actor-critic path is single-GPU")
            self._flat = self._layered.critic_group        # the optimiser's parameters (``group`` unless split)
        else:
            self._desc, plist = fused
            self._layered = None
            self._flat = FlatGroup(plist, dev, grad_extra=GRAD_EXTRA, device_step=True)
            lib = load_library()
            # per-CTA partial gradient rows written by ts_ppo_grad (folded by ts_clip_adam_step)
            self._flat.partials = torch.zeros((int(lib.ts_ppo_partial_rows()), self._flat.n + GRAD_EXTRA), dtype=torch.float32,
                                              device=dev)
            # scratch for the pre-split (bf16x3) weight image of the tensor-core update kernel; None -> the
            # kernels gather + split the weights themselves (networks the tensor-core path does not cover)
            nbytes = int(lib.ts_ppo_weight_image_bytes(C.byref(self._desc)))
            self._flat.weight_image = torch.zeros(nbytes, dtype=torch.uint8, device=dev) if nbytes > 0 else None
            if hasattr(self.policy, "_fused_inference"):      # Collector-side inference through the same forward kernel
                self.policy._fused_inference = (self._flat, self._desc)
            if self._ranks()[1] > 1:      # replicas start bit-identical
                from ...parallel import broadcast_params_
                broadcast_params_(self._flat.flat)
        # a real torch Adam / RMSprop (+ scheduler) keeps lr schedules and state_dict round trips unchanged
        self.optim = self._create_optimizer(self._actor_critic if optim_include_actor else self.critic, optim,
                                            max_grad_norm=max_grad_norm)
        bind_optimizer(self.optim, self._flat, rmsprop=True)
        self.max_grad_norm = max_grad_norm
        self.gamma = gamma
        self.return_scaling = return_scaling
        self.ret_rms = RunningMeanStd()
        self._eps = 1e-8
        self._scratch = DeviceScratch(dev)
        self._buf = self._scratch.tensor

    @property
    def device(self) -> torch.device:
        return self._flat.device

    def _ranks(self) -> tuple[int, int]:
        """(rank, world size) of the data-parallel update; (0, 1) without a process group or with ``data_parallel=False``."""
        return world() if self.data_parallel else (0, 1)

    # ------------------------------------------------------------------ update
    def update(self, buffer: ReplayBuffer, batch_size: int | None, repeat: int) -> TrainingStats:
        """``OnPolicyAlgorithm.update`` (algorithm_base.py:854-865).  The ``repeat`` minibatch orders are started here, so that
        the reference-exact draws of ``Batch.split`` (batch.py:1209) overlap the upload / value pass / GAE that precede the
        first pass (nothing in between touches numpy's global stream: ``sample(0)`` draws nothing)."""
        with self._minibatch_order_job(buffer, repeat):
            return super().update(buffer=buffer, batch_size=batch_size, repeat=repeat)

    @contextlib.contextmanager
    def _minibatch_order_job(self, buffer: Any, repeat: int) -> Any:
        """Open (and on exit close) this update's ``MinibatchOrder``; ``_update_with_batch`` picks it up."""
        if buffer is None or not self.policy.is_within_training_step or len(buffer) == 0 or repeat <= 0:
            yield None        # update() raises or returns before any pass: no draw
            return
        with self._minibatch_order(repeat, len(buffer)) as order:
            self._active_order = order
            try:
                yield order
            finally:
                self._active_order = None

    @contextlib.contextmanager
    def _minibatch_order(self, repeat: int, n: int) -> Any:
        """The running order if it covers (repeat, n), else one opened for the duration of the block (direct calls)."""
        order = self._active_order
        if order is not None and order.shape == (repeat, n):
            yield order
            return
        order = MinibatchOrder(self, repeat, n)
        completed = False
        try:
            yield order
            completed = True
        finally:
            order.close(completed)

    # ------------------------------------------------------------------ rollout -> device
    def _sample(self, buffer: ReplayBuffer, sample_size: int | None) -> tuple[Batch, Any]:
        """Device-resident equivalent of ``buffer.sample(0)`` (manager.py:200-234 order)."""
        if sample_size not in (0, None):
            return super()._sample(buffer, sample_size)
        dev = self.device
        meta_host = buffer._meta
        for k in ("obs", "act", "rew", "terminated", "truncated", "done"):
            if k not in meta_host.get_keys() or isinstance(meta_host[k], Batch):
                raise UnsupportedModelError(f"fused update needs a dense '{k}' array in the buffer")
        # the kernels stride the columns by the network descriptor: refuse layouts they would mis-read (the reference
        # would stack frames, buffer_base.py:557-603, or fail with a shape error in the first Linear)
        if getattr(buffer, "stack_num", 1) != 1 or getattr(buffer, "_save_only_last_obs", False):
            raise UnsupportedModelError("fused update: frame stacking (stack_num > 1 / save_only_last_obs) is not supported "
                                        "by the MLP actor-critic kernels")
        obs_w = int(np.prod(meta_host.obs.shape[1:], dtype=np.int64))
        act_w = int(np.prod(meta_host.act.shape[1:], dtype=np.int64))
        net_obs, want_act = self._spec.obs_dim, (1 if self._spec.categorical else self._spec.act_dim)
        if obs_w != net_obs or act_w != want_act:
            raise ValueError(f"buffer rows (obs width {obs_w}, act width {act_w}) do not match the networks "
                             f"(obs_dim {net_obs}, action width {want_act})")
        n = len(buffer)
        full = n == buffer.maxsize and bool(np.all(buffer._ins == 0))
        need = ("obs", "act", "rew", "terminated", "truncated", "done") + (("obs_next",) if buffer._save_obs_next else ())
        mirrored = buffer.device_columns()      # kept up to date by add(): no bulk transfer (data/buffer/mirror.py)
        if mirrored is not None and all(k in mirrored for k in need) and mirrored["obs"].device == dev:
            up = {k: mirrored[k] for k in need if k != "done"}
            done_dev = mirrored["done"]
        else:       # one DMA per key from the (pinned) host arrays
            up = {"obs": _upload(meta_host.obs, dev, torch.float32), "act": _upload(meta_host.act, dev, torch.float32),
                  "rew": _upload(meta_host.rew, dev, torch.float64), "terminated": _upload(meta_host.terminated, dev),
                  "truncated": _upload(meta_host.truncated, dev)}
            if buffer._save_obs_next:
                up["obs_next"] = _upload(meta_host.obs_next, dev, torch.float32)
            done_dev = _upload(meta_host.done, dev)
        for k in ("obs", "act", "obs_next"):
            if k in up:
                up[k] = up[k].reshape(buffer.maxsize, -1)
        meta = ops.DeviceBufferMeta(
            to_device(buffer._extend_offset, dev), done_dev,
            to_device(buffer.last_index, dev), to_device(buffer._sizes, dev), to_device(buffer._ins, dev))
        if full:
            indices = torch.arange(n, dtype=torch.int64, device=dev)
            cols = up
        else:
            indices = ops.sample_all_indices(meta, capacity=n)
            cols = {k: ops.gather_rows(v, indices) for k, v in up.items()}
        if not buffer._save_obs_next:  # obs_next = obs[next(indices)]  (buffer_base.py:627-629)
            cols["obs_next"] = ops.gather_rows(up["obs"], ops.next_index(meta, indices))
        # segment ends that are not done flags: last written slot of every running episode
        unf, cnt = ops.unfinished_index_raw(meta)
        cols["_unfinished"] = ops.mark_members(indices, unf, table_size=buffer.maxsize, count=cnt)
        cols["done"] = torch.maximum(cols["terminated"], cols["truncated"])
        batch = Batch()
        for k, v in cols.items():
            batch.__dict__[k] = v
        batch.__dict__["info"] = Batch()
        batch.__dict__["policy"] = Batch()
        return batch, indices

    # ------------------------------------------------------------------ value pass + GAE
    def _add_returns_and_advantages(self, batch: Batch, buffer: ReplayBuffer | None, indices: Any) -> Batch:
        """batch.v_s / returns / adv as f32 device tensors (a2c.py:115-153)."""
        self._flat.ensure_adopted()
        n = batch.obs.shape[0]
        v_s = self._buf("v_s", n, torch.float32)
        v_next = self._buf("v_next", n, torch.float32)
        r, w = self._ranks()
        if self._layered is not None:
            self._layered.critic_values(batch.obs, v_s)
            self._layered.critic_values(batch.obs_next, v_next)
        elif self.rollout_partition == "shared" and w > 1 and n % w == 0:
            # shared rollout on several GPUs: every rank evaluates the critic on ITS 1 / world of the rows (contiguous env range),
            # one all-gather makes v_s / v_s_ complete everywhere; the 17 us scan below runs redundantly (replicas identical)
            import torch.distributed as dist
            lo, hi = r * (n // w), (r + 1) * (n // w)
            pair = self._buf("v_pair_local", (2, n // w), torch.float32)
            ops.critic_forward(self._flat.flat, self._desc, batch.obs[lo:hi], batch.obs_next[lo:hi], out=pair[0], out2=pair[1])
            full = self._buf("v_pair_full", (w, 2, n // w), torch.float32)
            dist.all_gather_into_tensor(full, pair)
            v_s.view(w, n // w).copy_(full[:, 0])
            v_next.view(w, n // w).copy_(full[:, 1])
        else:
            amap = self._next_alias_map(batch, build=buffer is not None)
            if amap is not None:
                ops.critic_forward_dedup(self._flat.flat, self._desc, batch.obs, batch.obs_next, amap, out=v_s, out2=v_next)
            else:
                ops.critic_forward(self._flat.flat, self._desc, batch.obs, batch.obs_next, out=v_s, out2=v_next)
        rms = self._rms_device() if self.return_scaling else None
        adv = self._buf("adv", n, torch.float32)
        ret = self._buf("returns", n, torch.float32)
        moments = None
        # per-rank rollout shards: the ranks' batch moments are merged in rank order; a shared rollout needs no exchange
        # (every rank scans the same transitions)
        if rms is not None and w > 1 and self.rollout_partition == "per_rank":
            moments = self._buf("rms_moments", 3, torch.float64)
        ops.gae(v_s, v_next, batch.rew, batch.terminated, batch.truncated, batch.get("_unfinished"),
                gamma=self.gamma, gae_lambda=self.gae_lambda, rms_state=rms, rms_eps=self._eps,
                out=(adv, ret), workspace=self._gae_workspace(n), batch_moments_out=moments)
        if moments is not None:
            self._merge_rms_across_ranks(rms, moments)
        batch.__dict__["v_s"], batch.__dict__["returns"], batch.__dict__["adv"] = v_s, ret, adv
        return batch

    def _next_alias_map(self, batch: Batch, build: bool = False) -> ops.NextAliasMap | None:
        """The map of the rows of ``batch.obs_next`` that repeat the next row of ``batch.obs``, so that the value pass
        evaluates the critic once per distinct observation.  Built from the data once per update (``build``: the
        preprocess call); the recompute calls get it back as long as the batch still holds the very tensors it was
        built from, and None (= evaluate both inputs in full) otherwise."""
        obs, obs_next = batch.obs, batch.obs_next
        if build:
            n = obs.shape[0]
            amap = ops.NextAliasMap(self._buf("next_alias", n, torch.uint8), self._buf("next_extra", n, torch.int32),
                                    self._buf("next_extra_count", 1, torch.int32))
            need = int(load_library().ts_next_alias_workspace_bytes(n))
            ops.next_alias_map(obs, obs_next, out=amap, workspace=self._buf("next_alias_ws", max(need, 4), torch.uint8))
            self._next_alias = (weakref.ref(obs), weakref.ref(obs_next), amap)
        if self._next_alias is None:
            return None
        ref_obs, ref_next, amap = self._next_alias
        return amap if ref_obs() is obs and ref_next() is obs_next else None

    def _gae_workspace(self, n: int) -> torch.Tensor:
        from ..._cabi import load_library
        need = int(load_library().ts_gae_workspace_bytes(n))
        return self._buf("gae_ws", max(need, 64), torch.uint8)

    # RunningMeanStd lives on the device for the duration of an update() call
    def _rms_device(self) -> torch.Tensor:
        t = self._scratch.get("rms")
        if t is None:
            t = self._scratch["rms"] = self.ret_rms.device_state(self.device)
        return t

    def _rms_begin(self) -> None:
        if self.return_scaling:
            self._scratch["rms"] = self.ret_rms.device_state(self.device)

    def _rms_end(self) -> None:
        if self.return_scaling and "rms" in self._scratch:
            self.ret_rms.load_device_state(self._scratch.pop("rms"))

    # ------------------------------------------------------------------ multi-GPU hooks
    def _merge_rms_across_ranks(self, rms: torch.Tensor, moments: torch.Tensor) -> None:
        from ...parallel import allgather_moments
        from ..._cabi import call, ptr, stream_ptr
        allm = allgather_moments(moments)
        call("ts_rms_merge", ptr(rms), ptr(allm), allm.shape[0], stream_ptr(self.device))

    # ------------------------------------------------------------------ hyper-parameters
    def _hparams(self, **over: Any) -> PPOHParams:
        hp = PPOHParams()
        hp.eps_clip, hp.dual_clip, hp.vf_coef, hp.ent_coef = 0.0, 0.0, 0.5, 0.01
        hp.max_grad_norm = float(self.max_grad_norm) if self.max_grad_norm is not None else 0.0
        hp.adv_eps = self._eps
        for k, v in optimizer_hyperparams(self.optim._optim).items():   # the scheduler's lr of this update
            setattr(hp, k, v)
        hp.value_clip, hp.advantage_normalization = 0, 0
        for k, v in over.items():
            setattr(hp, k, v)
        return hp

    def _stats_from_device(self, stats: torch.Tensor) -> A2CTrainingStats:
        """ONE D2H for all per-minibatch losses (vs 4 ``.item()`` per step, ppo.py:213-216)."""
        s = stats.cpu().numpy().astype(np.float64)
        # per-minibatch (loss, clip/actor loss, vf loss, entropy, grad norm, rows) of the last update, in step order: what
        # the reference appends to its four lists per optimiser step (ppo.py:213-216)
        self.last_loss_table = s[:, :6].copy()
        return A2CTrainingStats(
            loss=SequenceSummaryStats.from_sequence(s[:, 0]),
            actor_loss=SequenceSummaryStats.from_sequence(s[:, 1]),
            vf_loss=SequenceSummaryStats.from_sequence(s[:, 2]),
            ent_loss=SequenceSummaryStats.from_sequence(s[:, 3]),
            gradient_steps=int(s.shape[0]),
        )

    def _alloc_stats(self, rows: int) -> torch.Tensor:
        return torch.zeros((rows, STATS_STRIDE), dtype=torch.float32, device=self.device)


def __getattr__(name: str) -> Any:
    """``A2C`` shares the fused update loop with PPO and lives next to it (ppo.py imports this module, so the
    reference's import path ``...modelfree.a2c.A2C`` is served lazily)."""
    if name == "A2C":
        from .ppo import A2C
        return A2C
    raise AttributeError(name)
