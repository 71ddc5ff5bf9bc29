"""The host-side helpers of algorithm/minibatch_order.py: the shared-rollout slicing of a minibatch order and the transport
format of numpy's generator state between ranks."""
import numpy as np
import pytest
import torch


def test_shared_slice_partitions_every_minibatch():
    """rollout_partition='shared' (SURVEY 8(e)): with the SAME permutation on every rank, rank r takes the r-th contiguous
    1 / world slice of every minibatch -- the ranks' local minibatches tile the global one in order, nothing else."""
    from tianshou_b200.algorithm.minibatch_order import shared_slice
    from tianshou_b200.data.batch import minibatch_bounds
    N, B = 4096, 512
    perm = torch.randperm(N, generator=torch.Generator().manual_seed(0)).to(torch.int32)
    bounds = minibatch_bounds(N, B, merge_last=True)
    for w in (2, 4, 8):
        parts = [shared_slice(perm, bounds, r, w) for r in range(w)]
        local = B // w
        for r, (sl, lb) in enumerate(parts):
            assert sl.numel() == N // w and lb == [(m * local, (m + 1) * local) for m in range(len(bounds))]
        for m, (lo, hi) in enumerate(bounds):
            glued = torch.cat([parts[r][0][m * local:(m + 1) * local] for r in range(w)])
            assert torch.equal(glued, perm[lo:hi])
    with pytest.raises(ValueError):       # a merged tail / a minibatch that does not divide: refused, not silently re-balanced
        shared_slice(perm[:4000], minibatch_bounds(4000, 512, merge_last=True), 0, 2)
    with pytest.raises(ValueError):
        shared_slice(perm, minibatch_bounds(N, 512, merge_last=True), 0, 3)


def test_numpy_state_pack_roundtrip():
    """Shared rollout on several GPUs: rank 0's generator state travels to the other ranks as 627 float64 (broadcast_numpy_state)."""
    from tianshou_b200.algorithm.minibatch_order import pack_numpy_state, unpack_numpy_state
    np.random.seed(123)
    np.random.standard_normal(3)                  # has_gauss = 1, a cached gaussian
    np.random.permutation(1000)
    st = np.random.get_state()
    a = np.random.rand(5)
    np.random.seed(0)
    np.random.set_state(unpack_numpy_state(st[0], pack_numpy_state(st)))
    assert np.array_equal(np.random.rand(5), a)
    np.random.set_state(st)
    g1 = np.random.standard_normal(1)
    np.random.set_state(unpack_numpy_state(st[0], pack_numpy_state(st)))
    assert np.array_equal(np.random.standard_normal(1), g1)       # the cached gaussian survived
