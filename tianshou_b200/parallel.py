"""Multi-GPU plumbing for the data-parallel policy update (one process per GPU, NCCL).

The reference has no distributed path (only single-process ``nn.DataParallel``,
tianshou/utils/net/common.py:473-515).  Here every rank holds a full replica of the 11k
parameters + Adam state and its own shard of the rollout; per optimiser step exactly ONE
all-reduce carries the flat gradient and the loss sums (n_params + 4 floats).  All functions work
on whatever backend the process group uses, so the host-side logic is testable with ``gloo`` on
CPU tensors (tests/test_parallel.py).
"""
from __future__ import annotations

import torch
import torch.distributed as dist


def world() -> tuple[int, int]:
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


def shard_bounds(lo: int, hi: int, rank: int, world_size: int) -> tuple[int, int]:
    """Contiguous slice of minibatch positions [lo, hi) owned by ``rank`` (sizes differ by <= 1)."""
    n = hi - lo
    base, rem = divmod(n, world_size)
    start = lo + rank * base + min(rank, rem)
    return start, start + base + (1 if rank < rem else 0)


def allreduce_sum_(flat: torch.Tensor) -> torch.Tensor:
    """In-place SUM all-reduce of the flat gradient(+loss sums) buffer."""
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(flat, op=dist.ReduceOp.SUM)
    return flat


def allgather_moments(moments: torch.Tensor) -> torch.Tensor:
    """[world, 3] tensor of every rank's (count, mean, M2), identical on all ranks, rank order."""
    _, w = world()
    if w == 1:
        return moments.reshape(1, 3)
    out = torch.empty((w, 3), dtype=moments.dtype, device=moments.device)
    dist.all_gather_into_tensor(out, moments.reshape(1, 3).contiguous())
    return out


def broadcast_params_(flat: torch.Tensor, src: int = 0) -> torch.Tensor:
    """Make replicas bit-identical at start-up."""
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        dist.broadcast(flat, src=src)
    return flat


class PeerExchange:
    """Exchange buffers of the in-kernel gradient all-reduce (``ts_ppo_epoch_multi``).

    Every rank allocates one IPC-shareable buffer (``ts_peer_alloc``), the handles (``TS_PEER_HANDLE_BYTES``
    each) travel through ``all_gather`` and every rank maps its peers' buffers (``ts_peer_open``).  After that the
    data path is kernel-only: 8-byte (value, sequence) packets over NVLink.  ``create`` is collective
    (every rank must call it) and returns None on EVERY rank when any rank cannot allocate or map
    (no P2P between the devices, IPC blocked); the caller then keeps the NCCL path.
    """

    def __init__(self) -> None:
        self.rank, self.world = world()
        self._own = None
        self._opened: list = []
        self.ptrs = None

    @staticmethod
    def _all_ok(ok: bool, device: torch.device) -> bool:
        flag = torch.tensor([1 if ok else 0], dtype=torch.int32, device=device)
        dist.all_reduce(flag, op=dist.ReduceOp.MIN)
        return int(flag.item()) == 1

    @classmethod
    def create(cls, desc, device: torch.device) -> "PeerExchange | None":
        import ctypes as C

        from ._cabi import TS_PEER_HANDLE_BYTES, call, load_library
        ex = cls()
        handle = (C.c_uint8 * TS_PEER_HANDLE_BYTES)()
        ok = True
        try:   # phase 1 (local): allocate + export
            nbytes = int(load_library().ts_ppo_peer_buffer_bytes(C.byref(desc), ex.world))
            if nbytes <= 0:
                raise RuntimeError(f"no peer exchange for world size {ex.world}")
            own = C.c_void_p()
            call("ts_peer_alloc", nbytes, C.byref(own), handle)
            ex._own = own
        except Exception:  # noqa: BLE001 - any failure means "use NCCL"
            ok = False
        if not cls._all_ok(ok, device):
            ex.close()
            return None
        mine = torch.tensor(list(handle), dtype=torch.uint8, device=device)
        allh = torch.empty((ex.world, TS_PEER_HANDLE_BYTES), dtype=torch.uint8, device=device)
        dist.all_gather_into_tensor(allh, mine.reshape(1, TS_PEER_HANDLE_BYTES))
        allh = allh.cpu()
        ex.ptrs = (C.c_void_p * ex.world)()
        try:   # phase 2 (local): map the peers
            for r in range(ex.world):
                if r == ex.rank:
                    ex.ptrs[r] = ex._own.value
                else:
                    h = (C.c_uint8 * TS_PEER_HANDLE_BYTES)(*allh[r].tolist())
                    p = C.c_void_p()
                    call("ts_peer_open", h, C.byref(p))
                    ex._opened.append(p)
                    ex.ptrs[r] = p.value
        except Exception:  # noqa: BLE001
            ok = False
        if not cls._all_ok(ok, device):   # also the barrier: nobody launches before every mapping exists
            ex.close()
            return None
        return ex

    def close(self) -> None:
        from ._cabi import call
        for p in self._opened:
            call("ts_peer_close", p)
        self._opened = []
        if self._own is not None:
            call("ts_peer_free", self._own)
            self._own = None
