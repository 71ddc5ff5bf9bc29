"""The minibatch orders of one on-policy update: where each pass's rows come from, and when the device may read them.

Every pass of ``update(buffer, batch_size, repeat)`` walks the minibatches in one row permutation -- the order that
``Batch.split(shuffle=True)`` draws with ``np.random.permutation(N)`` (reference batch.py:1209).  Three sources:

* numpy (default): the reference's draws on numpy's global stream, bit-identical, made by the background host job
  ``NumpyGlobalPermutationJob`` into pinned rows; a feed (``ts_host_perm_feed_*``) copies each row to the device on a copy
  stream, and the compute stream waits for row r (``ready(r)``, or ``ts_ppo_update`` given ``feed``) -- never the host;
* device (``minibatch_shuffle="device"``): a keyed bijection generated on the GPU (``ts_make_permutation``), one epoch per
  pass; same distribution, different stream;
* rank 0: ONE rollout shared by several GPUs (NCCL): rank 0 runs the numpy job and broadcasts each row before its pass, and
  numpy's advanced state when the update completes; the other ranks run no host job.
"""
from __future__ import annotations

import ctypes as C
from typing import Any

import numpy as np
import torch
import torch.distributed as dist

from .. import ops
from .._cabi import call, ptr, stream_ptr
from ..data.batch import NumpyGlobalPermutationJob


class MinibatchOrder:
    """The ``repeat`` orders of one update over ``n`` rows.  ``rows``: int32 device tensor [repeat, n]; ``feed``: the row
    feed for ``ts_ppo_update`` (or None); ``ready(r)`` before the device reads ``rows[r]``; ``close`` exactly once."""

    def __init__(self, algo: Any, repeat: int, n: int) -> None:
        self.shape = (repeat, n)
        self.feed: Any = None
        self._device = algo.device
        self._host_job: NumpyGlobalPermutationJob | None = None
        self._from_rank0 = False
        if algo.minibatch_shuffle == "device":
            self.rows = ops.make_permutation(algo._shuffle_seed, algo._shuffle_epoch, repeat, n, self._device)
            algo._shuffle_epoch += repeat
            return
        rank, world = algo._ranks()
        self._from_rank0 = algo.rollout_partition == "shared" and world > 1 and dist.get_backend() == "nccl"
        self.rows = algo._buf("perms_dev", (repeat, n), torch.int32)
        if self._from_rank0 and rank != 0:
            return
        host = algo._scratch.get("host_perms")
        if host is None or host.shape[0] < repeat or host.shape[1] != n:
            host = algo._scratch["host_perms"] = torch.empty((repeat, n), dtype=torch.int32, pin_memory=True)
        self._host_job = NumpyGlobalPermutationJob(host, repeat)
        if self._host_job.handle is None:     # no background job (foreign bit generator): the rows are complete already
            self.rows.copy_(host[:repeat], non_blocking=True)
        else:
            feed = C.c_void_p()
            try:
                call("ts_host_perm_feed_start", self._host_job.handle, C.c_void_p(host.data_ptr()), ptr(self.rows), n, repeat,
                     C.byref(feed))
            except BaseException:
                self.close(False)
                raise
            self.feed = feed

    def ready(self, r: int) -> None:
        """The current stream waits until ``rows[r]`` is on the device (the host does not wait)."""
        if self.feed is not None:
            call("ts_host_perm_feed_wait_row", self.feed, r, stream_ptr(self._device))
        if self._from_rank0:
            dist.broadcast(self.rows[r], 0)

    def close(self, completed: bool) -> None:
        """Finish the feed once its consumers have run (the feed's host functions use the job), then the job (numpy's
        advanced state written back), then -- only if the update completed: the other ranks may never reach the collective
        while an exception unwinds -- rank 0's numpy state to every rank."""
        if self.feed is not None:
            torch.cuda.current_stream(self._device).synchronize()
            call("ts_host_perm_feed_finish", self.feed)
            self.feed = None
        if self._host_job is not None:
            self._host_job.__exit__(None, None, None)
            self._host_job = None
        if self._from_rank0 and completed:
            broadcast_numpy_state(self._device)


def shared_slice(perm_r: torch.Tensor, bounds: list[tuple[int, int]], rank: int, wsize: int
                 ) -> tuple[torch.Tensor, list[tuple[int, int]]]:
    """This rank's contiguous 1 / wsize slice of every minibatch of ``perm_r`` as a local permutation + bounds."""
    n_mb = len(bounds)
    size = bounds[0][1] - bounds[0][0]
    regular = all(lo == m * size and hi == lo + size for m, (lo, hi) in enumerate(bounds))
    if not regular or size % wsize != 0:
        raise ValueError(f"rollout_partition='shared' needs len(buffer) % batch_size == 0 and batch_size % world_size == 0 "
                         f"(got {bounds[-1][1]} transitions, minibatch {size}, {wsize} ranks)")
    local = size // wsize
    sl = perm_r[: n_mb * size].view(n_mb, wsize, local)[:, rank, :].contiguous().view(-1)
    return sl, [(m * local, (m + 1) * local) for m in range(n_mb)]


def pack_numpy_state(st: tuple) -> np.ndarray:
    """numpy's legacy MT19937 state tuple as 627 float64 (every field is exactly representable: 32-bit words, small ints)."""
    out = np.empty(627, dtype=np.float64)
    out[:624] = np.asarray(st[1], dtype=np.float64)
    out[624], out[625], out[626] = float(st[2]), float(st[3]), float(st[4])
    return out


def unpack_numpy_state(kind: str, h: np.ndarray) -> tuple:
    return (kind, h[:624].astype(np.uint32), int(h[624]), int(h[625]), float(h[626]))


def broadcast_numpy_state(device: torch.device) -> None:
    """numpy's global legacy state of rank 0 -> every rank (they all consumed the same draws: rank 0 made them)."""
    st = np.random.get_state()
    t = torch.zeros(627, dtype=torch.float64, device=device)
    if dist.get_rank() == 0:
        t.copy_(torch.from_numpy(pack_numpy_state(st)))
    dist.broadcast(t, 0)
    if dist.get_rank() != 0:
        np.random.set_state(unpack_numpy_state(st[0], t.cpu().numpy()))
