"""Policy / Algorithm base classes and the two static return estimators.

API contract: tianshou/algorithm/algorithm_base.py (Policy :133-373, Algorithm :435-825,
OnPolicyAlgorithm :828-865, OffPolicyAlgorithm :868-903).  ``compute_episodic_return`` and
``compute_nstep_return`` keep their signatures and numpy/torch in-out behaviour but run on the
device through the C ABI (csrc/gae.cu, csrc/nstep.cu, csrc/index.cu); there is no host
implementation.
"""
from __future__ import annotations

import logging
import time
from abc import ABC, abstractmethod
from collections.abc import Callable, Mapping
from dataclasses import dataclass, field
from typing import Any, Literal

import numpy as np
import torch
from torch import nn
from torch.optim.lr_scheduler import LRScheduler

from .. import ops
from .._cabi import to_device
from ..data import Batch, ReplayBuffer, SequenceSummaryStats, to_numpy, to_torch_as
from ..utils.torch_utils import policy_within_training_step, torch_train_mode
from .optim import OptimizerFactory

logger = logging.getLogger(__name__)


@dataclass(kw_only=True)
class TrainingStats:
    """Result of one ``update()`` (algorithm_base.py:63-101)."""

    _non_loss_fields = ("train_time", "smoothed_loss")
    train_time: float = 0.0
    smoothed_loss: dict = field(default_factory=dict)

    def _get_self_dict(self) -> dict[str, Any]:
        return self.__dict__

    def get_loss_stats_dict(self) -> dict[str, float]:
        out = {}
        for k, v in self._get_self_dict().items():
            if k.startswith("_") or k in self._non_loss_fields or v is None:
                continue
            out[k] = v.mean if isinstance(v, SequenceSummaryStats) else v
        return out


def _space_kind(space: Any) -> Literal["discrete", "continuous"]:
    """Duck-typed gymnasium space classification (gymnasium itself is not a dependency)."""
    name = type(space).__name__
    if name in ("Discrete", "MultiDiscrete", "MultiBinary") or hasattr(space, "n") or hasattr(space, "nvec"):
        return "discrete"
    if name == "Box" or (hasattr(space, "low") and hasattr(space, "high")):
        return "continuous"
    raise ValueError(f"Unsupported action space: {space}.")


class Policy(nn.Module, ABC):
    """obs -> action mapping (algorithm_base.py:133-373)."""

    def __init__(self, action_space: Any, observation_space: Any | None = None, action_scaling: bool = False,
                 action_bound_method: Literal["clip", "tanh"] | None = "clip") -> None:
        if action_bound_method is not None and action_bound_method not in ("clip", "tanh"):
            raise ValueError(f"Got invalid {action_bound_method=}. Valid values are: ('clip', 'tanh').")
        kind = _space_kind(action_space)
        if action_scaling and kind != "continuous":
            raise ValueError(f"action_scaling can only be True when action_space is Box but got: {action_space}")
        super().__init__()
        self.observation_space = observation_space
        self.action_space = action_space
        self._action_type = kind
        self.agent_id = 0
        self.action_scaling = action_scaling
        self.action_bound_method = action_bound_method
        self.is_within_training_step = False

    @property
    def action_type(self) -> Literal["discrete", "continuous"]:
        return self._action_type

    def map_action(self, act: Any) -> np.ndarray:
        """Bound then scale raw network output to the env's action range (:258-293)."""
        act = to_numpy(act)
        if not isinstance(act, np.ndarray):
            raise ValueError(f"act should have been be a numpy.ndarray, but got {type(act)}.")
        if self._action_type == "continuous":
            if self.action_bound_method == "clip":
                act = np.clip(act, -1.0, 1.0)
            elif self.action_bound_method == "tanh":
                act = np.tanh(act)
            if self.action_scaling:
                assert np.min(act) >= -1.0 and np.max(act) <= 1.0, (
                    f"action scaling only accepts raw action range = [-1, 1], but got: {act}")
                low, high = self.action_space.low, self.action_space.high
                act = low + (high - low) * (act + 1.0) / 2.0
        return act

    def map_action_inverse(self, act: Any) -> np.ndarray:
        act = to_numpy(act)
        if self._action_type == "continuous":
            if self.action_scaling:
                low, high = self.action_space.low, self.action_space.high
                scale = high - low
                eps = np.finfo(np.float32).eps.item()
                scale[scale < eps] += eps
                act = (act - low) * 2.0 / scale - 1.0
            if self.action_bound_method == "tanh":
                act = (np.log(1.0 + act) - np.log(1.0 - act)) / 2.0
        return act

    def compute_action(self, obs: Any, info: dict[str, Any] | None = None, state: Any = None) -> np.ndarray | int:
        obs = np.array(obs)[None, :]
        act = self.forward(Batch(obs=obs, info=info), state=state).act.squeeze()
        if isinstance(act, torch.Tensor):
            act = act.detach().cpu().numpy()
        act = self.map_action(act)
        if self._action_type == "discrete" and np.ndim(act) == 0:
            act = int(act)
        return act

    def add_exploration_noise(self, act: Any, batch: Any) -> Any:
        return act


class Algorithm(nn.Module, ABC):
    """How to update the networks from a batch (algorithm_base.py:435-825)."""

    _STATE_DICT_KEY_OPTIMIZERS = "_optimizers"

    def __init__(self, *, policy: Policy) -> None:
        super().__init__()
        self.policy = policy
        self.lr_schedulers: list[LRScheduler] = []
        self._optimizers: list[Algorithm.Optimizer] = []

    class Optimizer:
        """torch optimizer + optional global-norm clipping (algorithm_base.py:457-511).
        ``step(loss)`` is the generic eager path kept for API users; the device updates drive the
        same optimizer state through the ``FlatGroup`` that ``bind_optimizer`` sets as ``_flat``."""

        def __init__(self, optim: torch.optim.Optimizer, module: nn.Module, max_grad_norm: float | None = None):
            self._optim = optim
            self._module = module
            self._max_grad_norm = max_grad_norm
            self._flat: Any = None  # set by fused algorithms

        def step(self, loss: torch.Tensor, retain_graph: bool | None = None, create_graph: bool = False) -> None:
            self._optim.zero_grad()
            loss.backward(retain_graph=retain_graph, create_graph=create_graph)
            if self._max_grad_norm is not None:
                nn.utils.clip_grad_norm_(self._module.parameters(), max_norm=self._max_grad_norm)
            self._optim.step()
            if self._flat is not None:
                self._flat.import_state(self._optim)

        def state_dict(self) -> dict:
            if self._flat is not None:
                self._flat.export_state(self._optim)
            return self._optim.state_dict()

        def load_state_dict(self, state_dict: dict) -> None:
            self._optim.load_state_dict(state_dict)
            if self._flat is not None:
                self._flat.import_state(self._optim)

    def _create_optimizer(self, module: nn.Module, factory: OptimizerFactory,
                          max_grad_norm: float | None = None) -> "Algorithm.Optimizer":
        optimizer, lr_scheduler = factory.create_instances(module)
        if lr_scheduler is not None:
            self.lr_schedulers.append(lr_scheduler)
        optim = self.Optimizer(optimizer, module, max_grad_norm=max_grad_norm)
        self._optimizers.append(optim)
        return optim

    def state_dict(self, *args, destination=None, prefix="", keep_vars=False):  # type: ignore[override]
        d = super().state_dict(*args, destination=destination, prefix=prefix, keep_vars=keep_vars)
        key = prefix + self._STATE_DICT_KEY_OPTIMIZERS
        assert key not in d
        d[key] = [o.state_dict() for o in self._optimizers]
        return d

    def load_state_dict(self, state_dict: Mapping[str, Any], strict: bool = True, assign: bool = False):  # type: ignore[override]
        state_dict = dict(state_dict)
        opt_states = state_dict.pop(self._STATE_DICT_KEY_OPTIMIZERS)
        result = super().load_state_dict(state_dict, strict=strict, assign=assign)
        for optim, st in zip(self._optimizers, opt_states, strict=True):
            optim.load_state_dict(st)
        return result

    # ------------------------------------------------------------------ update skeleton
    def _preprocess_batch(self, batch: Batch, buffer: ReplayBuffer, indices: Any) -> Batch:
        return batch

    def _postprocess_batch(self, batch: Batch, buffer: ReplayBuffer, indices: Any) -> None:
        """PER priority update (algorithm_base.py:562-584)."""
        if hasattr(buffer, "update_weight"):
            if hasattr(batch, "weight"):
                buffer.update_weight(indices, batch.weight)
            else:
                logger.warning("batch has no attribute 'weight', but buffer has an update_weight method. "
                               "Prioritized replay is disabled for this batch.")

    def _sample(self, buffer: ReplayBuffer, sample_size: int | None) -> tuple[Batch, Any]:
        """Hook: how the update obtains its batch (fused algorithms return device tensors)."""
        return buffer.sample(sample_size)

    def _update(self, sample_size: int | None, buffer: ReplayBuffer | None,
                update_with_batch_fn: Callable[[Batch], TrainingStats]) -> TrainingStats:
        """sample -> preprocess -> update -> postprocess -> lr schedule (algorithm_base.py:586-631)."""
        if not self.policy.is_within_training_step:
            raise RuntimeError(
                f"update() was called outside of a training step as signalled by {self.policy.is_within_training_step=} "
                "If you want to update the policy without a Trainer, you will have to manage the above-mentioned "
                f"flag yourself. You can to this e.g., by using the contextmanager {policy_within_training_step.__name__}."
            )
        if buffer is None:
            return TrainingStats()
        start = time.time()
        batch, indices = self._sample(buffer, sample_size)
        batch = self._preprocess_batch(batch, buffer, indices)
        with torch_train_mode(self):
            stat = update_with_batch_fn(batch)
        self._postprocess_batch(batch, buffer, indices)
        for sched in self.lr_schedulers:
            sched.step()
        stat.train_time = time.time() - start
        return stat

    # ------------------------------------------------------------------ static estimators
    @staticmethod
    def value_mask(buffer: ReplayBuffer, indices: np.ndarray) -> np.ndarray:
        """True where obs_next of buffer[indices] is a real state (algorithm_base.py:633-651)."""
        return ~buffer.terminated[indices]

    @staticmethod
    def compute_episodic_return(
        batch: Batch,
        buffer: ReplayBuffer,
        indices: np.ndarray,
        v_s_: np.ndarray | torch.Tensor | None = None,
        v_s: np.ndarray | torch.Tensor | None = None,
        gamma: float = 0.99,
        gae_lambda: float = 0.95,
    ) -> tuple[np.ndarray, np.ndarray]:
        """GAE returns / advantages as float64 numpy arrays (algorithm_base.py:653-719).

        Runs ``ts_gae`` (segmented reverse scan) on the buffer's device.  Segment ends are
        ``terminated | truncated | (index in buffer.unfinished_index())``; the value mask zeroes
        ``v_s_`` after termination only.
        """
        dev = buffer.device
        rew = to_device(np.asarray(batch.rew, dtype=np.float64), dev)
        n = rew.numel()
        idx = to_device(np.asarray(indices, dtype=np.int64), dev)
        meta = buffer.device_meta()
        if v_s_ is None:
            assert np.isclose(gae_lambda, 1.0)
            v_next = torch.zeros(n, dtype=torch.float64, device=dev)
            term_mask = None
        else:
            v_next = to_device(to_numpy(v_s_.flatten()), dev)
            if v_next.dtype not in (torch.float32, torch.float64):
                v_next = v_next.to(torch.float64)
            term_mask = ops.gather_rows(_u8_view(buffer.device_array("terminated")), idx)
        if v_s is None:
            masked = v_next if term_mask is None else v_next * (term_mask == 0).to(v_next.dtype)
            v_cur = torch.roll(masked, 1)
        else:
            v_cur = to_device(to_numpy(v_s.flatten()), dev)
            if v_cur.dtype != v_next.dtype:  # mixed precision: do the scan on f64 values
                v_cur, v_next = v_cur.to(torch.float64), v_next.to(torch.float64)
        unf = ops.unfinished_index(meta)
        extra = ops.mark_members(idx, unf, table_size=buffer.maxsize)
        term = to_device(np.asarray(batch.terminated).astype(bool), dev)
        trunc = to_device(np.asarray(batch.truncated).astype(bool), dev)
        # `terminated` of the batch ends segments; the value mask uses buffer.terminated[indices]
        # (identical for batch == buffer[indices], kept separate for exactness)
        end = torch.maximum(term, trunc)
        adv, ret = ops.gae(v_cur, v_next, rew, term_mask, end, extra, gamma=gamma, gae_lambda=gae_lambda,
                           out_dtype=torch.float64, terminated_ends=False)
        return ret.cpu().numpy(), adv.cpu().numpy()

    @staticmethod
    def compute_nstep_return(
        batch: Batch,
        buffer: ReplayBuffer,
        indices: np.ndarray,
        target_q_fn: Callable[[ReplayBuffer, np.ndarray], torch.Tensor],
        gamma: float = 0.99,
        n_step: int = 1,
    ) -> Batch:
        """n-step TD target into ``batch.returns`` (algorithm_base.py:721-817).

        ``next`` chains, end flags, value mask and the windowed gather-reduce are CUDA kernels;
        ``target_q_fn`` is the user's torch callable evaluated at the indices n steps ahead.
        """
        if len(indices) != len(batch):
            raise ValueError(f"Batch size {len(batch)} and indices size {len(indices)} mismatch.")
        dev = buffer.device
        meta = buffer.device_meta()
        I = len(indices)
        stacked = ops.stack_next_indices(meta, np.asarray(indices, dtype=np.int64), n_step)
        last_idx = stacked[-1].cpu().numpy()
        with torch.no_grad():
            target_q_torch = target_q_fn(buffer, last_idx)
        tq = target_q_torch.reshape(I, -1).to(dev, torch.float32).contiguous().clone()
        # whole-buffer columns come from the device mirror / a version-keyed cache: no per-call upload of B-sized arrays
        term = _u8_view(buffer.device_array("terminated"))
        ops.value_mask_rows(tq, term, stacked[-1].contiguous())
        end_flag = ops.buffer_end_flags(meta)
        rew = buffer.device_array("rew")
        if rew.dtype != torch.float64:
            rew = rew.to(torch.float64)
        out = ops.nstep_return(rew, end_flag, tq, stacked, gamma, n_step, out_dtype=torch.float64)
        batch.returns = out.reshape(target_q_torch.reshape(I, -1).shape).to(
            dtype=target_q_torch.dtype, device=target_q_torch.device)
        if hasattr(batch, "weight"):
            batch.weight = to_torch_as(batch.weight, target_q_torch)
        return batch


def _u8_view(t: torch.Tensor) -> torch.Tensor:
    return t.view(torch.uint8) if t.dtype == torch.bool else t


class OnPolicyAlgorithm(Algorithm, ABC):
    """update(buffer, batch_size, repeat) over the whole buffer (algorithm_base.py:828-865)."""

    @abstractmethod
    def _update_with_batch(self, batch: Batch, batch_size: int | None, repeat: int) -> TrainingStats: ...

    def update(self, buffer: ReplayBuffer, batch_size: int | None, repeat: int) -> TrainingStats:
        return self._update(
            sample_size=0, buffer=buffer,
            update_with_batch_fn=lambda batch: self._update_with_batch(batch=batch, batch_size=batch_size,
                                                                        repeat=repeat))


class OffPolicyAlgorithm(Algorithm, ABC):
    """update(buffer, sample_size) (algorithm_base.py:868-903)."""

    @abstractmethod
    def _update_with_batch(self, batch: Batch) -> TrainingStats: ...

    def update(self, buffer: ReplayBuffer, sample_size: int | None) -> TrainingStats:
        return self._update(sample_size=sample_size, buffer=buffer,
                            update_with_batch_fn=lambda batch: self._update_with_batch(batch))


class OfflineAlgorithm(Algorithm, ABC):
    """Learns from a fixed buffer: ``process_buffer`` once, then update(buffer, sample_size) (algorithm_base.py:906-951)."""

    def process_buffer(self, buffer: ReplayBuffer) -> ReplayBuffer:
        """Prepare the buffer for offline learning, e.g. add keys to it (algorithm_base.py:913-915)."""
        return buffer

    @abstractmethod
    def _update_with_batch(self, batch: Batch) -> TrainingStats: ...

    def update(self, buffer: ReplayBuffer, sample_size: int | None) -> TrainingStats:
        return self._update(sample_size=sample_size, buffer=buffer,
                            update_with_batch_fn=lambda batch: self._update_with_batch(batch))
