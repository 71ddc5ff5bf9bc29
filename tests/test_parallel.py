"""Host-side logic of the multi-GPU path on CPU: world_size-2 gloo process group.
(The kernels themselves need a GPU; what is covered here is the sharding arithmetic, the
single-collective-per-step contract and the cross-rank RunningMeanStd merge order.)"""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tianshou_b200.parallel import allgather_moments, allreduce_sum_, broadcast_params_, shard_bounds, world


def test_shard_bounds_cover_range_exactly():
    for lo, hi in [(0, 16384), (5, 5), (3, 10), (100, 16485)]:
        for w in (1, 2, 3, 4, 8):
            parts = [shard_bounds(lo, hi, r, w) for r in range(w)]
            assert parts[0][0] == lo and parts[-1][1] == hi
            for a, b in zip(parts[:-1], parts[1:], strict=True):
                assert a[1] == b[0]
            sizes = [b - a for a, b in parts]
            assert max(sizes) - min(sizes) <= 1


def _free_port() -> int:
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank: int, world_size: int, port: int, out_dir: str) -> None:
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world_size))
    dist.init_process_group("gloo", rank=rank, world_size=world_size)
    try:
        assert world() == (rank, world_size)
        # (1) replicas start identical
        flat = torch.full((11085,), float(rank + 1))
        broadcast_params_(flat)
        assert torch.all(flat == 1.0)
        # (2) ONE all-reduce carries gradient + loss sums: emulate each rank's partial sums
        n_params, extra = 11085, 4
        rng = np.random.default_rng(rank)
        local = torch.from_numpy(rng.standard_normal(n_params + extra).astype(np.float32))
        local[-1] = 8192.0                                   # this rank's row count
        total = allreduce_sum_(local.clone())
        ref = sum(torch.from_numpy(np.random.default_rng(r).standard_normal(n_params + extra).astype(np.float32))
                  for r in range(world_size))
        ref[-1] = 8192.0 * world_size
        assert torch.allclose(total, ref, atol=1e-6)
        # (3) RunningMeanStd moments: all-gather in rank order, identical on every rank
        data = np.random.default_rng(100 + rank).standard_normal(1000 + 10 * rank) * (rank + 1)
        mom = torch.tensor([len(data), data.mean(), ((data - data.mean()) ** 2).sum()], dtype=torch.float64)
        allm = allgather_moments(mom)
        assert allm.shape == (world_size, 3)
        n, mean, M2 = 0.0, 0.0, 0.0
        for k in range(world_size):                           # same Chan merge as ts_rms_merge (csrc/gae.cu)
            n2, m2, M2b = allm[k].tolist()
            tot = n + n2
            d = m2 - mean
            mean, M2, n = (m2, M2b, n2) if n == 0 else (mean + d * (n2 / tot), M2 + M2b + d * d * (n * n2 / tot), tot)
        alld = np.concatenate([np.random.default_rng(100 + r).standard_normal(1000 + 10 * r) * (r + 1)
                               for r in range(world_size)])
        assert abs(mean - alld.mean()) < 1e-12 and abs(M2 / n - alld.var()) < 1e-10
        torch.save(allm, os.path.join(out_dir, f"m{rank}.pt"))
    finally:
        dist.destroy_process_group()


def test_two_rank_gloo(tmp_path):
    port = _free_port()
    mp.spawn(_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    a, b = torch.load(tmp_path / "m0.pt"), torch.load(tmp_path / "m1.pt")
    assert torch.equal(a, b)


def test_single_process_defaults():
    assert world() == (0, 1)
    t = torch.ones(4)
    assert allreduce_sum_(t) is t
    assert allgather_moments(torch.tensor([1.0, 2.0, 3.0], dtype=torch.float64)).shape == (1, 3)
