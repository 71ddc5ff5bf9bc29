"""Replay buffers: numpy storage on the host (so the reference ``Collector`` can ``add`` to them
unchanged), index arithmetic on the device.

Contract mirrored from the reference:
  ReplayBuffer            tianshou/data/buffer/buffer_base.py:25-670
  ReplayBufferManager     tianshou/data/buffer/manager.py:13-310  (+ numba kernels :311-363)
  VectorReplayBuffer      tianshou/data/buffer/vecbuf.py:14-37

Design differences (GPU-first, same observable behaviour):
  * ONE implementation for E >= 1 sub-buffers: all per-sub-buffer bookkeeping (size, insertion
    index, episode return/length/start) lives in numpy arrays of length E, so ``add`` for
    thousands of envs is a handful of vectorised numpy ops instead of a Python loop over child
    objects (reference: manager.py:157-174, ~8 us per transition).
  * ``next`` / ``prev`` / ``unfinished_index`` / ``sample_indices(0)`` run as CUDA kernels
    (csrc/index.cu) on a lazily refreshed device mirror of (edges, done, last_index, lengths);
    results are bit-identical int64.  There is no host implementation of these four.
  * numeric storage is allocated in pinned host memory when CUDA is present, so the per-update
    bulk H2D of the rollout runs at PCIe speed without a staging copy.
"""
from __future__ import annotations

from typing import Any, ClassVar, cast

import numpy as np
import torch

from ... import ops
from ..._cabi import to_device
from ..batch import Batch, IndexType, _coerce, alloc_by_keys_diff, create_value


class MalformedBufferError(RuntimeError):
    pass


def _pin_numeric_leaves(b: Batch, keep: list) -> None:
    """Re-home numeric ndarray leaves of ``b`` in pinned host memory (same values, same dtype)."""
    for k, v in list(b.items()):
        if isinstance(v, Batch):
            _pin_numeric_leaves(v, keep)
        elif isinstance(v, np.ndarray) and v.dtype != object and v.size > 0:
            try:
                t = torch.empty(v.shape, dtype=torch.from_numpy(v[:0]).dtype, pin_memory=True)
            except (RuntimeError, TypeError):
                continue
            arr = t.numpy()
            arr[...] = v
            if v.dtype == np.bool_:
                arr = arr.view(np.bool_)
            keep.append(t)
            b.__dict__[k] = arr


class _SubBufferView:
    """Read-only view of sub-buffer ``e`` (what the reference exposes as ``manager.buffers[e]``)."""

    def __init__(self, parent: "ReplayBuffer", e: int) -> None:
        self._p, self._e = parent, e

    @property
    def maxsize(self) -> int:
        return int(self._p._cap[self._e])

    @property
    def _size(self) -> int:
        return int(self._p._sizes[self._e])

    @property
    def _insertion_idx(self) -> int:
        return int(self._p._ins[self._e])

    @property
    def last_index(self) -> np.ndarray:
        return np.array([self._p.last_index[self._e] - self._p._offset[self._e]])

    @property
    def _meta(self) -> Batch:
        lo = int(self._p._offset[self._e])
        return self._p._meta[lo : lo + self.maxsize]

    def __len__(self) -> int:
        return self._size

    def unfinished_index(self) -> np.ndarray:
        p, e = self._p, self._e
        if p._sizes[e] == 0:
            return np.array([], int)
        last = int(p.last_index[e])
        return np.array([] if p.done[last] else [last - int(p._offset[e])], int)

    def sample_indices(self, batch_size: int | None) -> np.ndarray:
        return self._p._child_sample_indices(self._e, batch_size)


class ReplayBuffer:
    """Circular transition store (see module docstring)."""

    _reserved_keys = ("obs", "act", "rew", "terminated", "truncated", "done", "obs_next", "info", "policy")
    _input_keys = ("obs", "act", "rew", "terminated", "truncated", "obs_next", "info", "policy")
    _required_keys_for_add: ClassVar[set[str]] = {"obs", "act", "rew", "terminated", "truncated", "done"}

    def __init__(
        self,
        size: int,
        stack_num: int = 1,
        ignore_obs_next: bool = False,
        save_only_last_obs: bool = False,
        sample_avail: bool = False,
        random_seed: int = 42,
        device: torch.device | str | None = None,
        device_mirror: bool = False,
        **kwargs: Any,
    ) -> None:
        self.__dict__["_device_mirror_arg"] = bool(device_mirror)
        self.options: dict[str, Any] = {
            "stack_num": stack_num,
            "ignore_obs_next": ignore_obs_next,
            "save_only_last_obs": save_only_last_obs,
            "sample_avail": sample_avail,
        }
        self._init_layout(np.array([int(size)]), random_seed, device)
        assert stack_num > 0, "stack_num should be greater than 0"
        self.stack_num = stack_num
        self._save_obs_next = not ignore_obs_next
        self._save_only_last_obs = save_only_last_obs
        self._sample_avail = sample_avail

    # ------------------------------------------------------------------ layout / state
    def _init_layout(self, caps: np.ndarray, random_seed: int, device: Any) -> None:
        d = self.__dict__
        caps = np.asarray(caps, dtype=np.int64)
        d["_cap"] = caps
        d["_offset"] = np.concatenate([[0], np.cumsum(caps)[:-1]]).astype(np.int64)
        d["_extend_offset"] = np.concatenate([[0], np.cumsum(caps)]).astype(np.int64)
        d["maxsize"] = int(caps.sum())
        d["buffer_num"] = len(caps)
        d["_indices"] = np.arange(d["maxsize"])
        d["_meta"] = Batch()
        d["_random_seed"] = random_seed
        d["_random_state"] = np.random.RandomState(random_seed)
        d["_child_rngs"] = {}
        d["_device_arg"] = device
        d["_pinned"] = []
        d["_mirror"] = None
        d["_mirror_version"] = -1
        d["_version"] = 0
        d["_dmirror"] = None            # asynchronous device copy of the transition arrays (mirror.py)
        d.setdefault("_device_mirror_arg", False)
        self._reset_state(keep_statistics=False)

    def _reset_state(self, keep_statistics: bool) -> None:
        d = self.__dict__
        E = len(self._cap)
        d["last_index"] = self._offset.copy()
        d["_sizes"] = np.zeros(E, dtype=np.int64)
        d["_ins"] = np.zeros(E, dtype=np.int64)
        d["_ep_start"] = np.zeros(E, dtype=np.int64)
        if not keep_statistics or "_ep_return" not in d:
            d["_ep_return"] = np.zeros(E, dtype=np.float64)
            d["_ep_len"] = np.zeros(E, dtype=np.int64)
        d["_version"] = d.get("_version", 0) + 1

    # properties the reference exposes on the plain buffer
    @property
    def _size(self) -> int:
        return int(self._sizes.sum())

    @property
    def _lengths(self) -> np.ndarray:
        return self._sizes

    @property
    def _insertion_idx(self) -> int:
        return int(self._ins[0])

    @property
    def subbuffer_edges(self) -> np.ndarray:
        return self._extend_offset

    @property
    def buffers(self) -> list[_SubBufferView]:
        return [_SubBufferView(self, e) for e in range(self.buffer_num)]

    def __len__(self) -> int:
        return int(self._sizes.sum())

    def __repr__(self) -> str:
        inner = self._meta.__repr__()[len(self._meta.__class__.__name__):]
        return self.__class__.__name__ + inner

    def __getattr__(self, key: str) -> Any:
        try:
            return self.__dict__["_meta"][key]
        except KeyError as e:
            raise AttributeError(key) from e

    def __setattr__(self, key: str, value: Any) -> None:
        assert key not in self._reserved_keys, f"key '{key}' is reserved and cannot be assigned"
        super().__setattr__(key, value)

    def __getstate__(self) -> dict[str, Any]:
        state = dict(self.__dict__)
        state["_pinned"] = []
        state["_mirror"] = None
        state["_mirror_version"] = -1
        state["_dmirror"] = None
        return state

    def __setstate__(self, state: dict[str, Any]) -> None:
        self.__dict__.update(state)

    # ------------------------------------------------------------------ device mirror
    @property
    def device(self) -> torch.device:
        if self._device_arg is not None:
            return torch.device(self._device_arg)
        from ..._cabi import require_cuda
        require_cuda()
        return torch.device("cuda", torch.cuda.current_device())

    def device_meta(self) -> ops.DeviceBufferMeta:
        """(edges, done, last_index, lengths) on the device, refreshed when the buffer changed."""
        if self._mirror is None or self._mirror_version != self._version:
            cols = self.device_columns()
            if cols is not None and "done" in cols:
                # the B-sized `done` column is already on the device (mirror, kept current by add()): only the E-sized
                # bookkeeping arrays travel -- an off-policy loop (collect a step, update, ...) refreshes this every update
                dev = self.device
                self.__dict__["_mirror"] = ops.DeviceBufferMeta(
                    to_device(np.asarray(self._extend_offset, dtype=np.int64), dev), cols["done"].view(torch.uint8),
                    to_device(np.asarray(self.last_index, dtype=np.int64), dev), to_device(np.asarray(self._sizes, dtype=np.int64), dev),
                    to_device(np.asarray(self._ins, dtype=np.int64), dev))
            else:
                done = self._meta.get("done")
                if done is None or (isinstance(done, Batch)):
                    done = np.zeros(self.maxsize, dtype=bool)
                self.__dict__["_mirror"] = ops.DeviceBufferMeta.from_host(
                    self._extend_offset, done, self.last_index, self._sizes, self.device, ins=self._ins)
            self.__dict__["_mirror_version"] = self._version
        return self._mirror

    def _touch(self) -> None:
        self.__dict__["_version"] += 1

    # asynchronous device mirror of the transition arrays (opt-in: ``device_mirror=True``)
    def enable_device_mirror(self) -> None:
        """Keep a device copy of obs / act / rew / flags / obs_next up to date from ``add()`` on (mirror.py)."""
        self.__dict__["_device_mirror_arg"] = True

    def _mirror_add(self, idx: np.ndarray, batch: Batch) -> None:
        if not self._device_mirror_arg:
            return
        if self._dmirror is None:
            from .mirror import DeviceMirror
            self.__dict__["_dmirror"] = DeviceMirror(self)
        self._dmirror.push(np.asarray(idx, dtype=np.int64).reshape(-1), batch)

    def device_columns(self) -> "dict[str, torch.Tensor] | None":
        """Device-resident transition arrays if the mirror is enabled and reflects the host buffer, else None."""
        return self._dmirror.columns() if self._dmirror is not None else None

    def device_array(self, key: str) -> "torch.Tensor":
        """The whole column ``key`` on the device WITHOUT a per-call upload: the mirror's copy when the buffer keeps
        one, else an upload cached until the buffer next changes (``add`` / ``reset`` / ``set_batch`` ... bump the
        version).  Used by the n-step / GAE entry points, which index whole-buffer ``rew`` / ``terminated`` arrays
        (algorithm_base.py:711,798-800) with a few hundred sampled indices."""
        cols = self.device_columns()
        if cols is not None and key in cols:
            return cols[key]
        cache = self.__dict__.setdefault("_dev_cache", {})
        ent = cache.get(key)
        if ent is None or ent[0] != self._version:
            ent = cache[key] = (self._version, to_device(np.asarray(self._meta[key]), self.device))
        return ent[1]

    def sync_device_mirror(self) -> None:
        """Re-upload everything (after edits that bypass ``add()``, e.g. in-place numpy writes)."""
        if self._device_mirror_arg and len(self._meta.get_keys()) > 0:
            if self._dmirror is None:
                from .mirror import DeviceMirror
                self.__dict__["_dmirror"] = DeviceMirror(self)
            self._dmirror.resync()

    # ------------------------------------------------------------------ index API (CUDA)
    def unfinished_index(self) -> np.ndarray:
        """Last-written slot of every sub-buffer whose episode is still running
        (buffer_base.py:314-317, manager.py:85-91) -- ``ts_unfinished_index``."""
        if len(self) == 0:
            return np.array([], int)
        return ops.unfinished_index(self.device_meta()).cpu().numpy()

    def prev(self, index: int | np.ndarray) -> np.ndarray:
        """Predecessor clamped at episode starts (buffer_base.py:319-326, manager.py:311-336)."""
        return self._step(index, ops.prev_index)

    def next(self, index: int | np.ndarray) -> np.ndarray:
        """Successor clamped at episode ends / last written slot (buffer_base.py:328-334,
        manager.py:339-363)."""
        return self._step(index, ops.next_index)

    def _step(self, index: Any, fn: Any) -> Any:
        scalar = not isinstance(index, (list, np.ndarray))
        arr = np.asarray([index] if scalar else index, dtype=np.int64)
        out = fn(self.device_meta(), arr.reshape(-1)).cpu().numpy().reshape(arr.shape)
        return out[0] if scalar else out

    def _all_indices(self) -> np.ndarray:
        """sample_indices(0): every valid slot, sub-buffer-major, chronological
        (buffer_base.py:519-525, manager.py:217-234)."""
        if len(self) == 0:
            return np.array([], int)
        return ops.sample_all_indices(self.device_meta(), capacity=len(self)).cpu().numpy()

    # ------------------------------------------------------------------ add
    def _allocate(self, batch: Batch, stack: bool) -> None:
        if len(self._meta.get_keys()) == 0:
            self.__dict__["_meta"] = create_value(batch, self.maxsize, stack)
        else:
            alloc_by_keys_diff(self._meta, batch, self.maxsize, stack)
        if torch.cuda.is_available():
            _pin_numeric_leaves(self._meta, self._pinned)

    def _advance(self, ids: np.ndarray, rew: np.ndarray, done: np.ndarray
                 ) -> tuple[np.ndarray, np.ndarray, np.ndarray, np.ndarray]:
        """Vectorised ``_update_state_pre_add`` (buffer_base.py:360-418) for sub-buffers ``ids``
        (each at most once).  Returns absolute (insertion idx, ep_return, ep_len, ep_start idx)."""
        ids = np.asarray(ids, dtype=np.int64)
        # duplicate check without a sort: strictly increasing ids (the Collector's ready_env_ids / arange) are unique
        unique = len(ids) <= 1 or bool(np.all(ids[1:] > ids[:-1]))
        if not unique:
            seen = np.zeros(len(self._cap), dtype=bool)
            seen[ids] = True
            unique = int(seen.sum()) == len(ids)
        if not unique:  # same sub-buffer twice: order matters, go one by one
            parts = [self._advance(ids[k:k + 1], rew[k:k + 1], done[k:k + 1]) for k in range(len(ids))]
            return tuple(np.concatenate(p) for p in zip(*parts, strict=True))  # type: ignore[return-value]
        off, cap = self._offset[ids], self._cap[ids]
        ins = self._ins[ids]
        self.last_index[ids] = ins + off
        self._sizes[ids] = np.minimum(self._sizes[ids] + 1, cap)
        new_ins = (ins + 1) % cap
        self._ins[ids] = new_ins
        self._ep_return[ids] += rew
        self._ep_len[ids] += 1
        bad = self._ep_start[ids] > self._sizes[ids]
        if bad.any():
            k = int(np.flatnonzero(bad)[0])
            raise MalformedBufferError(
                f"Encountered a starting index {self._ep_start[ids][k]} that is outside the currently "
                f"available samples len={self._sizes[ids][k]}. The buffer is malformed."
            )
        done = done.astype(bool)
        ep_ret = np.where(done, self._ep_return[ids], 0.0)
        ep_len = np.where(done, self._ep_len[ids], 0)
        ep_start = self._ep_start[ids] + off
        fin = ids[done]
        self._ep_return[fin] = 0.0
        self._ep_len[fin] = 0
        self._ep_start[fin] = new_ins[done]
        self._touch()
        return ins + off, ep_ret, ep_len, ep_start

    def add(self, batch: Batch, buffer_ids: np.ndarray | list[int] | None = None
            ) -> tuple[np.ndarray, np.ndarray, np.ndarray, np.ndarray]:
        """Add one transition (buffer_base.py:420-501).  Returns (index, ep_rew, ep_len, ep_start)."""
        new = Batch()
        for k in batch.get_keys():
            new.__dict__[k] = _coerce(batch[k])
        batch = new
        batch.__dict__["done"] = np.logical_or(batch.terminated, batch.truncated)
        if not self._required_keys_for_add.issubset(batch.get_keys()):
            raise ValueError(f"Input batch must have the following keys: {self._required_keys_for_add}")
        stacked = False
        if buffer_ids is not None:
            if len(buffer_ids) != 1 and buffer_ids[0] != 0:
                raise ValueError(
                    "If `buffer_ids` is not None, it must be a single element with value 0 for the "
                    f"non-vectorized `ReplayBuffer`. Got {buffer_ids=}."
                )
            if len(batch) != 1:
                raise ValueError(
                    f"If `buffer_ids` is not None, the batch must have the shape (1, len(data)) but got {len(batch)=}."
                )
            stacked = True
        if self._save_only_last_obs:
            batch.obs = batch.obs[:, -1] if stacked else batch.obs[-1]
        if not self._save_obs_next:
            batch.pop("obs_next", None)
        elif self._save_only_last_obs:
            batch.obs_next = batch.obs_next[:, -1] if stacked else batch.obs_next[-1]
        rew, done = (batch.rew[0], batch.done[0]) if stacked else (batch.rew, batch.done)
        idx, ep_ret, ep_len, ep_start = self._advance(
            np.array([0]), np.asarray(rew, dtype=np.float64).reshape(1), np.asarray(done).reshape(1))
        try:
            self._meta[idx] = batch
        except ValueError:
            batch.rew = batch.rew.astype(float)
            batch.done = batch.done.astype(bool)
            batch.terminated = batch.terminated.astype(bool)
            batch.truncated = batch.truncated.astype(bool)
            self._allocate(batch, stack=not stacked)
            self._meta[idx] = batch
        self._mirror_add(idx, batch)
        return idx, ep_ret, ep_len, ep_start

    def update(self, buffer: "ReplayBuffer") -> np.ndarray:
        """Append all of ``buffer``'s transitions, oldest first (buffer_base.py:336-358)."""
        if len(buffer) == 0 or self.maxsize == 0:
            return np.array([], int)
        stack_num, buffer.stack_num = buffer.stack_num, 1
        src = buffer.sample_indices(0)
        buffer.stack_num = stack_num
        if len(src) == 0:
            return np.array([], int)
        n, cap = len(src), int(self._cap[0])
        dst = (self._ins[0] + np.arange(n)) % cap
        self.last_index[0] = dst[-1]
        self._ins[0] = (dst[-1] + 1) % cap
        self._sizes[0] = min(self._sizes[0] + n, cap)
        if len(self._meta.get_keys()) == 0:
            self.__dict__["_meta"] = create_value(buffer._meta, self.maxsize, stack=False)
        self._meta[dst] = buffer._meta[src]
        self._touch()
        return dst

    def reset(self, keep_statistics: bool = False) -> None:
        self._reset_state(keep_statistics)
        if self._dmirror is not None:
            self._dmirror.on_reset()

    def set_batch(self, batch: Batch) -> None:
        assert len(batch) == self.maxsize and set(batch.get_keys()).issubset(self._reserved_keys), (
            "Input batch doesn't meet ReplayBuffer's data form requirement.")
        self.__dict__["_meta"] = batch
        self._touch()

    @classmethod
    def from_data(cls, obs: Any, act: Any, rew: Any, terminated: Any, truncated: Any, done: Any,
                  obs_next: Any) -> "ReplayBuffer":
        size = len(obs)
        assert all(len(d) == size for d in [obs, act, rew, terminated, truncated, done, obs_next]), (
            "Lengths of all hdf5 datasets need to be equal.")
        buf = cls(size)
        if size == 0:
            return buf
        buf.set_batch(Batch(obs=obs, act=act, rew=rew, terminated=terminated, truncated=truncated,
                            done=done, obs_next=obs_next))
        buf._sizes[0] = size
        buf._touch()
        return buf

    # ------------------------------------------------------------------ sampling
    def _child_rng(self, e: int) -> np.random.RandomState:
        raise NotImplementedError

    def _child_sample_indices(self, e: int, batch_size: int | None) -> np.ndarray:
        raise NotImplementedError

    def sample_indices(self, batch_size: int | None) -> np.ndarray:
        """buffer_base.py:503-545.  Random draws stay on the host RandomState (identical stream);
        the all-indices case and the ``prev`` chains run on the device."""
        if batch_size is None:
            batch_size = len(self)
        if self.stack_num == 1 or not self._sample_avail:
            if batch_size > 0:
                return self._random_state.choice(self._size, batch_size)
            if batch_size == 0:
                return self._all_indices()
            return np.array([], int)
        if batch_size < 0:
            return np.array([], int)
        all_indices = prev_indices = self._all_indices()
        for _ in range(self.stack_num - 2):
            prev_indices = self.prev(prev_indices)
        all_indices = all_indices[prev_indices != self.prev(prev_indices)]
        if batch_size > 0:
            return self._random_state.choice(all_indices, batch_size)
        return all_indices

    def sample(self, batch_size: int | None) -> tuple[Batch, np.ndarray]:
        indices = self.sample_indices(batch_size)
        return self[indices], indices

    def get(self, index: int | list[int] | np.ndarray, key: str, default_value: Any = None,
            stack_num: int | None = None) -> Batch | np.ndarray:
        """Value of ``key`` at ``index`` with frame stacking through ``prev`` (buffer_base.py:557-603)."""
        if key not in self._meta.get_keys() and default_value is not None:
            return default_value
        val = self._meta[key]
        if stack_num is None:
            stack_num = self.stack_num
        try:
            if stack_num == 1:
                return val[index]
            frames: list[Any] = []
            indices = np.array(index) if isinstance(index, list) else index
            for _ in range(stack_num):
                frames = [val[indices], *frames]
                indices = self.prev(indices)
            indices = cast(np.ndarray, indices)
            if isinstance(val, Batch):
                return Batch.stack(frames, axis=np.ndim(indices))
            return np.stack(frames, axis=np.ndim(indices))
        except IndexError as e:
            if not (isinstance(val, Batch) and len(val.keys()) == 0):
                raise e
            return Batch()

    def __getitem__(self, index: IndexType) -> Batch:
        """A copy of the transitions at ``index`` (buffer_base.py:605-649)."""
        if isinstance(index, slice):
            indices = self.sample_indices(0) if index == slice(None) else self._indices[: len(self)][index]
        else:
            indices = index
        obs = self.get(indices, "obs")
        if self._save_obs_next:
            obs_next = self.get(indices, "obs_next", Batch())
        else:
            obs_next = self.get(self.next(indices), "obs", Batch())
        out = {
            "obs": obs,
            "act": self.act[indices],
            "rew": self.rew[indices],
            "terminated": self.terminated[indices],
            "truncated": self.truncated[indices],
            "done": self.done[indices],
            "obs_next": obs_next,
            "info": self.get(indices, "info", Batch()),
            "policy": self.get(indices, "policy", Batch()),
        }
        for key in set(self._meta.get_keys()) - set(self._input_keys):
            out[key] = self._meta[key][indices]
        return Batch(out)

    def get_buffer_indices(self, start: int, stop: int) -> np.ndarray:
        """Indices of [start, stop) inside ONE sub-buffer, wrapping at its edge
        (buffer_base.py:160-200)."""
        edges = self.subbuffer_edges
        lo_e = np.searchsorted(edges, start, side="right") - 1
        hi_e = np.searchsorted(edges, stop - 1, side="right") - 1
        if lo_e != hi_e:
            raise ValueError(
                "Start and stop indices must be within the same subbuffer. "
                f"Got {start=} in subbuffer edge {lo_e} and {stop=} in subbuffer edge {hi_e}."
            )
        if stop >= start:
            return np.arange(start, stop, dtype=int)
        upper = int(edges[int(np.searchsorted(edges, start, side="left"))])
        lower = int(edges[int(np.searchsorted(edges, start, side="left")) - 1])
        if lower >= stop:
            raise ValueError(f"The edge before the crossed edge should be smaller than the stop, but got {lower=}, {stop=}.")
        return np.concatenate((np.arange(start, upper, dtype=int), np.arange(lower, stop, dtype=int)))

    def set_array_at_key(self, seq: np.ndarray, key: str, index: IndexType | None = None,
                         default_value: float | None = None) -> None:
        self._meta.set_array_at_key(seq, key, index, default_value)
        self._touch()

    def hasnull(self) -> bool:
        """Any NaN / None among the valid transitions (the trainer asks after every collect, trainer.py:953).  The answer does
        not depend on the order of the rows, so the stored arrays are scanned in place -- no ``buffer[:]`` copy of the whole
        rollout in ``sample_indices(0)`` order (buffer_base.py:605-649) and no device work."""
        n = len(self)
        if n == 0:
            return False
        if n == self.maxsize:
            return self._meta.hasnull()
        valid = np.concatenate([np.arange(o, o + k) for o, k in zip(self._offset, self._sizes, strict=True) if k > 0])
        return self._meta[valid].hasnull()

    def isnull(self) -> Batch:
        return self[:].isnull()

    def dropnull(self) -> None:
        self.__dict__["_meta"] = self._meta.dropnull()
        n = len(self._meta)
        self._sizes[0] = n
        self._ins[0] = n
        self._touch()


class ReplayBufferManager(ReplayBuffer):
    """E sub-buffers laid out contiguously; transitions of env ``e`` go to sub-buffer ``e``
    (manager.py:13-310)."""

    def __init__(self, buffer_list: list[ReplayBuffer]) -> None:
        first = buffer_list[0]
        kwargs = dict(first.options)
        for b in buffer_list:
            assert len(b._meta.get_keys()) == 0
            assert type(b) is type(first)
            assert b.options == first.options
            if b.buffer_num != 1:
                raise ValueError(
                    f"{self.__class__.__name__} only supports buffers with a single index (non-vector buffers)."
                )
        caps = np.array([b.maxsize for b in buffer_list], dtype=np.int64)
        self._setup(caps, first._random_seed, first._device_arg, kwargs)

    def _setup(self, caps: np.ndarray, seed: int, device: Any, kwargs: dict[str, Any]) -> None:
        opts = {k: kwargs[k] for k in ("stack_num", "ignore_obs_next", "save_only_last_obs", "sample_avail")}
        self.__dict__["options"] = dict(kwargs)
        self._init_layout(caps, seed, device)
        self.__dict__.update(
            stack_num=opts["stack_num"],
            _save_obs_next=not opts["ignore_obs_next"],
            _save_only_last_obs=opts["save_only_last_obs"],
            _sample_avail=opts["sample_avail"],
        )
        assert self.stack_num > 0, "stack_num should be greater than 0"

    @property
    def _size(self) -> int:  # the reference's manager keeps its own `_size` at 0; len() is what counts
        return int(self._sizes.sum())

    def update(self, buffer: ReplayBuffer) -> np.ndarray:
        raise NotImplementedError

    def add(self, batch: Batch, buffer_ids: np.ndarray | list[int] | None = None
            ) -> tuple[np.ndarray, np.ndarray, np.ndarray, np.ndarray]:
        """Add one transition per listed sub-buffer (manager.py:131-198)."""
        new = Batch()
        for k in set(self._reserved_keys).intersection(batch.get_keys()):
            new.__dict__[k] = _coerce(batch[k])         # (entries of a foreign Batch implementation are adopted)
        batch = new
        batch.__dict__["done"] = np.logical_or(batch.terminated, batch.truncated)
        assert {"obs", "act", "rew", "terminated", "truncated", "done"}.issubset(batch.get_keys())
        if self._save_only_last_obs:
            batch.obs = batch.obs[:, -1]
        if not self._save_obs_next:
            batch.pop("obs_next", None)
        elif self._save_only_last_obs:
            batch.obs_next = batch.obs_next[:, -1]
        if buffer_ids is None:
            buffer_ids = np.arange(self.buffer_num)
        ids = np.asarray(buffer_ids, dtype=np.int64)
        idx, ep_ret, ep_len, ep_start = self._advance(
            ids, np.asarray(batch.rew, dtype=np.float64)[: len(ids)], np.asarray(batch.done)[: len(ids)])
        # lock-step rollouts write an arithmetic progression of slots (env e at e * cap + t): a strided slice
        # assignment instead of a fancy-indexed one (one strided memcpy per key instead of E small ones)
        where: Any = idx
        if len(idx) > 1:
            step = int(idx[1] - idx[0])
            if step > 0 and bool(np.all(idx[1:] - idx[:-1] == step)):
                where = slice(int(idx[0]), int(idx[-1]) + 1, step)
        try:
            self._meta[where] = batch
        except ValueError:
            batch.rew = batch.rew.astype(float)
            batch.done = batch.done.astype(bool)
            batch.terminated = batch.terminated.astype(bool)
            batch.truncated = batch.truncated.astype(bool)
            self._allocate(batch, stack=False)
            self._meta[where] = batch
        self._mirror_add(idx, batch)
        return idx, ep_ret, ep_len, ep_start

    def _child_rng(self, e: int) -> np.random.RandomState:
        rng = self.__dict__["_child_rngs"].get(e)
        if rng is None:  # every child of the reference owns RandomState(seed) (buffer_base.py:98)
            rng = self.__dict__["_child_rngs"][e] = np.random.RandomState(self._random_seed)
        return rng

    def _child_sample_indices(self, e: int, batch_size: int | None) -> np.ndarray:
        size, ins = int(self._sizes[e]), int(self._ins[e])
        if batch_size is None:
            batch_size = size
        if self.stack_num == 1 or not self._sample_avail:
            if batch_size > 0:
                return self._child_rng(e).choice(size, batch_size)
            if batch_size == 0:
                return np.concatenate([np.arange(ins, size), np.arange(ins)])
            return np.array([], int)
        raise NotImplementedError("per-child sample_avail is handled by the manager")

    def sample_indices(self, batch_size: int | None) -> np.ndarray:
        """manager.py:200-234 -- host RNG draws in the reference's order (manager RandomState
        picks sub-buffers, each sub-buffer's own RandomState picks slots)."""
        if batch_size is not None and batch_size < 0:
            return np.array([], int)
        if self._sample_avail and self.stack_num > 1:
            all_indices = prev_indices = self._all_indices()
            for _ in range(self.stack_num - 2):
                prev_indices = self.prev(prev_indices)
            all_indices = all_indices[prev_indices != self.prev(prev_indices)]
            if batch_size == 0:
                return all_indices
            if batch_size is None:
                batch_size = len(all_indices)
            return self._random_state.choice(all_indices, batch_size)
        if batch_size == 0 or batch_size is None:
            return self._all_indices()
        which = self._random_state.choice(self.buffer_num, batch_size, p=self._sizes / self._sizes.sum())
        counts = np.bincount(which, minlength=self.buffer_num)
        parts = [self._child_rng(e).choice(int(self._sizes[e]), int(counts[e])) + self._offset[e]
                 for e in np.flatnonzero(counts)]
        return np.concatenate(parts) if parts else np.array([], int)


class VectorReplayBuffer(ReplayBufferManager):
    """``buffer_num`` equal sub-buffers of ``ceil(total_size / buffer_num)`` slots (vecbuf.py:14-37)."""

    def __init__(self, total_size: int, buffer_num: int, **kwargs: Any) -> None:
        assert buffer_num > 0
        size = int(np.ceil(total_size / buffer_num))
        probe = ReplayBuffer(size, **kwargs)
        self.__dict__["_device_mirror_arg"] = probe._device_mirror_arg
        self._setup(np.full(buffer_num, size, dtype=np.int64), probe._random_seed, probe._device_arg,
                    probe.options)
