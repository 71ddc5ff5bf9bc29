"""CPU-side tests: Batch semantics, buffer bookkeeping + host RNG streams, C-ABI surface.
(No kernel is executed here -- there is no CPU implementation of the device path.)"""
import ctypes
import os
import pickle
import re

import numpy as np
import pytest
import torch

from tianshou_b200.data import Batch, ReplayBuffer, VectorReplayBuffer
from tianshou_b200.data.batch import minibatch_bounds
from ts_testutil import load_golden, set_buffer_state, synth_rollout


# ------------------------------------------------------------------------------------- Batch
def test_batch_basic_indexing_and_assignment():
    b = Batch(a=np.arange(6).reshape(3, 2), b=Batch(c=np.zeros(3), d=torch.ones(3, 2)), e=None)
    assert len(b) == 3 and Batch(a=np.zeros((3, 2)), c=np.zeros(3)).shape == [3]
    s = b[[0, 2]]
    assert s.a.tolist() == [[0, 1], [4, 5]] and s.b.d.shape == (2, 2) and s.e is None
    b[1] = Batch(a=np.array([7, 7]), b=Batch(c=np.float64(5), d=torch.zeros(2)))
    assert b.a[1].tolist() == [7, 7] and b.b.c[1] == 5
    with pytest.raises(ValueError):
        b[0] = Batch(zzz=1)
    with pytest.raises(IndexError):
        Batch()[0]
    assert "a" in b and b.get("nope", 3) == 3
    b2 = pickle.loads(pickle.dumps(b))
    assert b2 == b


def test_batch_cat_stack_split():
    x = Batch(a=np.ones((3, 2)), b=Batch(c=np.arange(3)))
    y = Batch(a=np.zeros((2, 2)), b=Batch(c=np.arange(2)), only=np.array([5.0, 6.0]))
    z = Batch.cat([x, y])
    assert z.a.shape == (5, 2) and z.b.c.tolist() == [0, 1, 2, 0, 1]
    assert z.only.tolist() == [0, 0, 0, 5, 6]           # partial keys are zero padded
    s = Batch.stack([Batch(a=1.0, b=np.array([1, 2])), Batch(a=2.0, b=np.array([3, 4]))])
    assert s.a.tolist() == [1, 2] and s.b.shape == (2, 2)
    lst = Batch([{"a": 1, "b": {"c": 2.0}}, {"a": 3, "b": {"c": 4.0}}])
    assert lst.a.tolist() == [1, 3] and lst.b.c.tolist() == [2.0, 4.0]
    np.random.seed(0)
    parts = list(Batch(v=np.arange(10)).split(4, shuffle=True, merge_last=True))
    np.random.seed(0)
    perm = np.random.permutation(10)
    assert [len(p) for p in parts] == [4, 6]
    assert np.array_equal(np.concatenate([p.v for p in parts]), perm)
    assert [len(p) for p in Batch(v=np.arange(10)).split(4, shuffle=False)] == [4, 4, 2]
    assert [len(p) for p in Batch(v=np.arange(10)).split(-1)] == [10]


@pytest.mark.parametrize("n,size", [(10, 4), (8, 4), (5, 10), (1, 1), (524288, 16384), (100, 33), (12, 5)])
def test_minibatch_bounds_match_reference_rule(n, size):
    """Same chunking as Batch.split (tianshou/data/batch.py:1199-1215)."""
    got = minibatch_bounds(n, size, merge_last=True)
    merge = n % size > 0
    exp = []
    for idx in range(0, n, size):
        if merge and idx + size + size >= n:
            exp.append((idx, n)); break
        exp.append((idx, min(idx + size, n)))
    assert got == exp and got[0][0] == 0 and got[-1][1] == n


def test_batch_to_torch_numpy_and_null():
    b = Batch(a=np.array([1.0, np.nan]), b=Batch(c=np.array([1, 2])))
    assert b.hasnull()
    assert not Batch(a=np.array([1.0, 2.0])).hasnull()
    t = b.to_torch()
    assert isinstance(t.a, torch.Tensor) and isinstance(t.b.c, torch.Tensor)
    assert isinstance(t.to_numpy().a, np.ndarray)
    assert len(b.dropnull()) == 1


# ------------------------------------------------------------------------------- buffers (host)
def test_vector_buffer_add_matches_reference_bookkeeping():
    """Vectorised add == the reference's per-child state machine (golden: states after scripted adds)."""
    g = load_golden("index_ref.npz")
    rng = np.random.default_rng(77)
    from oracle.gen_golden_replay import replay_index_cases   # deterministic replay of the generator script
    for c, (buf, exp) in enumerate(replay_index_cases(rng, VectorReplayBuffer, Batch)):
        p = f"idx{c}_"
        assert np.array_equal(buf.last_index, g[p + "last_index"]), c
        assert np.array_equal(buf._sizes, g[p + "lengths"]), c
        assert np.array_equal(np.asarray(buf.done, dtype=bool), g[p + "done"]), c
        # host RNG streams: manager RandomState(42) + one RandomState(42) per sub-buffer
        assert np.array_equal(buf.sample_indices(37), g[p + "sample37"]), c
        assert np.array_equal(buf.sample_indices(5), g[p + "sample5"]), c


def test_buffer_episode_statistics_and_reset():
    buf = VectorReplayBuffer(12, 3)
    for t in range(5):
        done = np.array([t == 2, False, t == 4])
        idx, ep_ret, ep_len, ep_start = buf.add(
            Batch(obs=np.zeros((3, 2)), act=np.zeros(3), rew=np.array([1.0, 2.0, 3.0]), terminated=done,
                  truncated=np.zeros(3, bool), obs_next=np.zeros((3, 2))))
        if t == 2:
            assert ep_ret.tolist() == [3.0, 0.0, 0.0] and ep_len.tolist() == [3, 0, 0] and ep_start.tolist() == [0, 4, 8]
        if t == 4:
            assert ep_ret.tolist() == [0.0, 0.0, 15.0] and ep_len.tolist() == [0, 0, 5]
            assert idx.tolist() == [0, 4, 8]          # capacity 4 per env: wrapped
    assert len(buf) == 12 and buf.rew.dtype == np.float64 and buf.done.dtype == np.bool_
    buf.reset(keep_statistics=True)
    assert len(buf) == 0 and buf._ep_len.tolist() == [2, 5, 0]
    buf.reset()
    assert buf._ep_len.tolist() == [0, 0, 0]
    with pytest.raises(AssertionError):
        buf.rew = 1


def test_single_buffer_add_and_sample_stream():
    buf = ReplayBuffer(5)
    for i in range(7):
        idx, ep_ret, ep_len, ep_start = buf.add(Batch(obs=i, act=i, rew=float(i), terminated=i == 3, truncated=False))
    assert len(buf) == 5 and buf.last_index.tolist() == [1] and buf._insertion_idx == 2
    assert buf.rew.tolist() == [5.0, 6.0, 2.0, 3.0, 4.0]
    ref = np.random.RandomState(42).choice(5, 4)
    assert np.array_equal(buf.sample_indices(4), ref)
    assert buf.sample_indices(-1).tolist() == []
    with pytest.raises(ValueError):
        buf.add(Batch(obs=1, act=1, rew=1.0, terminated=False, truncated=False), buffer_ids=[1, 2])


def test_device_path_fails_loudly_without_gpu():
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from tianshou_b200._cabi import ExtensionMissingError
    buf = ReplayBuffer(5)
    buf.add(Batch(obs=1, act=1, rew=1.0, terminated=False, truncated=False))
    with pytest.raises(ExtensionMissingError):
        buf.next(np.array([0]))
    with pytest.raises(ExtensionMissingError):
        buf.sample_indices(0)


# ------------------------------------------------------------------------------------ C ABI
def test_cabi_library_exports_every_parsed_declaration():
    from tianshou_b200 import _cabi
    lib = ctypes.CDLL(_cabi.LIB_PATH)
    names = sorted(_cabi.ABI.functions)
    assert len(names) >= 30
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/ts_b200.h but not exported"
    # diagnostics (phase timeline, wgmma self-test) live in a separate build and are NOT in the product library
    diag = sorted(_cabi.ABI.diag_functions)
    assert len(diag) == 2 and not set(diag) & set(names)
    for n in diag:
        assert not hasattr(lib, n), f"diagnostic entry {n} exported by the product library"
    lib2 = _cabi.load_library()
    assert all(getattr(lib2, n).argtypes is not None for n in names)     # every declaration is bound
    assert lib2.ts_version() == 1
    assert lib2.ts_gae_workspace_bytes(2048 * 3 + 1) > 0


def test_cabi_struct_layouts_match_header():
    from tianshou_b200._cabi import ActorCriticDesc, PPOHParams
    assert ctypes.sizeof(ActorCriticDesc) == 4 * 4 + 14 * 8
    assert ctypes.sizeof(PPOHParams) == 11 * 8 + 3 * 4 + 4      # trailing pad to 8
    assert ActorCriticDesc.a_w1.offset == 16 and ActorCriticDesc.n_params.offset == 120
    assert PPOHParams.optimizer.offset == 100


def test_cabi_prototypes_follow_the_type_rules():
    """One declaration per type rule of the header-derived binding, written out by hand."""
    from tianshou_b200._cabi import ABI, ActorCriticDesc, PPOHParams
    C = ctypes
    P, I, I32, I64, D, F = C.c_void_p, C.c_int, C.c_int32, C.c_int64, C.c_double, C.c_float
    fn = ABI.functions
    assert fn["ts_gae"] == (I, [P, P, I, P, P, P, P, I, I64, D, D, P, D, P, P, P, I, P, P])
    assert fn["ts_cql_rows"] == (I, [P, P, P, I64, I32, P, P, F, P, F, F, P, F, F, P, P, P, P, P])
    assert fn["ts_make_permutation"] == (I, [C.c_uint64, I32, I32, I64, P, P])
    desc, hp = C.POINTER(ActorCriticDesc), C.POINTER(PPOHParams)
    assert fn["ts_ppo_update"] == (I, [P, P, P, P, P, P, desc, hp, P, P, P, P, P, P, P, P, P, P, P, P, I64, P, I32, P, I32,
                                       I32, D, D, P, D, P, P, P, P, P, P])
    assert fn["ts_peer_open"] == (I, [P, C.POINTER(P)])
    assert fn["ts_ppo_epoch_multi"] == (I, [P, P, P, P, P, P, desc, hp, P, P, P, P, P, P, P, I64, I64, I64, I32, P, P, P,
                                            I32, I32, C.POINTER(P), P])
    assert fn["ts_gae_workspace_bytes"] == (C.c_size_t, [I64])
    assert fn["ts_last_error"] == (C.c_char_p, [])
    assert fn["ts_reset_launch_count"] == (None, [])


def test_cabi_header_parser_refuses_what_it_cannot_bind():
    from tianshou_b200._cabi import HeaderError, parse_header
    ok = parse_header("int ts_ok(int64_t n, const float* x, ts_stream_t s); /* ts_not_a_call( */\n")
    assert ok.functions == {"ts_ok": (ctypes.c_int, [ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p])}
    with pytest.raises(HeaderError, match="half h"):
        parse_header("int ts_ok(void);\nint ts_half(half h, ts_stream_t s);\n")
    with pytest.raises(HeaderError, match="ts_callback"):
        parse_header("int ts_ok(void);\nint ts_callback(void (*fn)(int), ts_stream_t s);\n")


# Exported functions that the suite reaches only through a Python wrapper, and the test that does: (file, test name).
ABI_REACHED_THROUGH = {
    "ts_npg_fvp_rows": ("test_npg_gpu.py", "test_fvp_vs_fp64_double_backward"),            # NPG._fvp
    "ts_segtree_setitem": ("test_buffer_kernels_gpu.py", "test_segtree_setitem_batches_with_duplicates"),
    "ts_segtree_reduce": ("test_buffer_kernels_gpu.py", "test_segtree_reduce_ranges"),
    "ts_segtree_prefix_sum_idx": ("test_buffer_kernels_gpu.py", "test_segtree_prefix_queries_ties_and_edges"),
    "ts_segtree_sample": ("test_kernels_gpu.py", "test_segtree_vs_reference_outputs"),    # SegmentTree.sample_device
    "ts_gather_rows": ("test_buffer_kernels_gpu.py", "test_gather_scatter_rows_alignment"),
    "ts_mark_members": ("test_buffer_kernels_gpu.py", "test_mark_members_edges"),
    "ts_narrow_i64_i32": ("test_buffer_kernels_gpu.py", "test_narrow_i64_i32_near_int32_limits"),
    "ts_next_index": ("test_buffer_kernels_gpu.py", "test_index_kernels_unequal_subbuffers"),
    "ts_prev_index": ("test_buffer_kernels_gpu.py", "test_index_kernels_unequal_subbuffers"),
    "ts_unfinished_index": ("test_buffer_kernels_gpu.py", "test_index_kernels_unequal_subbuffers"),
    "ts_stack_next_indices": ("test_buffer_kernels_gpu.py", "test_index_kernels_unequal_subbuffers"),
    "ts_nstep_return": ("test_buffer_kernels_gpu.py", "test_nstep_end_flag_at_every_window_position"),
    "ts_value_mask_rows": ("test_buffer_kernels_gpu.py", "test_value_mask_rows_special_values"),
    "ts_host_mt19937_permutation": ("test_host.py", "test_host_permutation_is_numpy_global_permutation_bit_for_bit"),
    "ts_host_perm_job_start": ("test_host.py", "test_permutation_job_matches_numpy_stream"),
    "ts_host_perm_job_wait": ("test_host.py", "test_permutation_job_matches_numpy_stream"),
    "ts_host_perm_job_finish": ("test_host.py", "test_permutation_job_matches_numpy_stream"),
    "ts_host_perm_feed_start": ("test_minibatch_order_gpu.py", "test_rows_and_numpy_state_per_source"),
    "ts_host_perm_feed_wait_row": ("test_minibatch_order_gpu.py", "test_rows_and_numpy_state_per_source"),
    "ts_host_perm_feed_finish": ("test_minibatch_order_gpu.py", "test_rows_and_numpy_state_per_source"),
}
# Exported functions that compute nothing a reference could check, with the reason.
ABI_PLUMBING = {
    "ts_launch_count": "a counter of kernel launches, read by _cabi.launch_count for the launch-budget tests",
    "ts_next_alias_workspace_bytes": "a workspace size for the caller's allocation",
    "ts_ppo_partial_rows": "the row count of the PPO gradient-partials workspace",
    "ts_ppo_weight_image_bytes": "a workspace size for the caller's allocation",
    "ts_ppo_peer_buffer_bytes": "the size of the peer-exchange buffer of multi-GPU PPO",
    "ts_peer_alloc": "IPC buffer lifecycle of multi-GPU PPO, driven by parallel.py in the two-rank tests",
    "ts_peer_close": "IPC buffer lifecycle of multi-GPU PPO, driven by parallel.py in the two-rank tests",
    "ts_peer_free": "IPC buffer lifecycle of multi-GPU PPO, driven by parallel.py in the two-rank tests",
}


def test_every_exported_function_is_tested():
    """Every function of the C ABI is named in some test, reached by a named test through a wrapper, or is plumbing that
    computes nothing checkable.  A new export without a test fails here; so does a stale entry in either table."""
    from tianshou_b200._cabi import ABI
    here = os.path.dirname(os.path.abspath(__file__))
    sources = {f: open(os.path.join(here, f)).read() for f in sorted(os.listdir(here)) if f.endswith(".py")}
    text = "\n".join(sources.values())
    exported = set(ABI.functions)
    assert set(ABI_REACHED_THROUGH) <= exported and set(ABI_PLUMBING) <= exported
    assert not set(ABI_REACHED_THROUGH) & set(ABI_PLUMBING)
    for name, (f, test) in ABI_REACHED_THROUGH.items():
        assert re.search(rf"^def {test}\(", sources.get(f, ""), flags=re.M), f"{name}: {f}::{test} does not exist"
    tables = set(ABI_REACHED_THROUGH) | set(ABI_PLUMBING)
    untested = sorted(n for n in exported - tables if not re.search(rf"\b{n}\b", text))
    assert not untested, f"exported but called by no test: {untested}"


def test_host_permutation_is_numpy_global_permutation_bit_for_bit():
    """The product path's minibatch order == np.random.permutation on the global stream (batch.py:1209),
    including the RNG state it leaves behind."""
    import torch

    from tianshou_b200.data.batch import numpy_global_permutation_
    for seed, n in [(0, 1), (1, 2), (2, 7), (3, 1000), (4, 65537), (5, 524288)]:
        np.random.seed(seed)
        ref = np.random.permutation(n)
        ref_next = np.random.rand(3)
        np.random.seed(seed)
        out = numpy_global_permutation_(torch.empty(n, dtype=torch.int32))
        assert np.array_equal(out.numpy(), ref), (seed, n)
        assert np.array_equal(np.random.rand(3), ref_next)     # the global stream continues identically


def test_permutation_job_matches_numpy_stream():
    """The background job behind PPO's default minibatch order: rows == consecutive np.random.permutation draws,
    generator state afterwards == numpy's (product path, host only)."""
    import torch

    from tianshou_b200.data.batch import NumpyGlobalPermutationJob
    for seed, n, rep in [(0, 1, 3), (1, 2, 2), (2, 3, 4), (3, 1000, 5), (4, 65537, 3), (5, 200_000, 6)]:
        np.random.seed(seed)
        ref = np.stack([np.random.permutation(n) for _ in range(rep)])
        ref_next = np.random.rand(3)
        np.random.seed(seed)
        rows = torch.empty((rep, n), dtype=torch.int32)
        with NumpyGlobalPermutationJob(rows, rep) as job:
            for r in reversed(range(rep)):            # any wait order
                job.wait(r)
        assert np.array_equal(rows.numpy(), ref), (seed, n)
        assert np.array_equal(np.random.rand(3), ref_next)


@pytest.mark.parametrize("isa", ["scalar", "avx2", "avx512"])
def test_numpy_permutation_job_every_instruction_set(isa, monkeypatch):
    """The walker's vector paths (csrc/hostperm_simd.cpp: groups of draws decided by two compares, accepted ones compacted)
    against np.random.permutation: rows AND the generator state afterwards, from generator positions that start mid-block,
    over sizes that cross several mask ranges, for repeat > the number of partner-list slots (slot reuse)."""
    import torch

    from tianshou_b200.data.batch import NumpyGlobalPermutationJob
    monkeypatch.setenv("TS_B200_PERM_ISA", isa)          # capped by what this CPU has (hostperm_simd.cpp detect_isa)
    for seed, burn, n, rep in [(10, 0, 31, 2), (11, 5, 33, 3), (12, 623, 64, 2), (13, 700, 4097, 9), (14, 1, 524288, 3),
                               (15, 17, 99_991, 8)]:
        np.random.seed(seed)
        np.random.randint(0, 2**31 - 1, size=burn)            # move the stream position off a block boundary
        st = np.random.get_state()
        ref = np.stack([np.random.permutation(n) for _ in range(rep)])
        ref_next = np.random.rand(3)
        np.random.set_state(st)
        rows = torch.empty((rep, n), dtype=torch.int32)
        with NumpyGlobalPermutationJob(rows, rep, n_workers=3) as job:
            for r in range(rep):
                job.wait(r)
        assert np.array_equal(rows.numpy(), ref), (isa, seed, n)
        assert np.array_equal(np.random.rand(3), ref_next), (isa, seed, n)


def test_numpy_permutation_job_many_jobs_and_fork():
    """The job's threads are parked between jobs (csrc/hostperm.cu Crew) and its scratch storage is cached: many jobs in a row,
    two jobs alive at the same time (the second gets fresh threads / storage), and a job in a forked child (the parked threads
    do not exist there: the crew is rebuilt) all reproduce numpy's stream."""
    import torch

    from tianshou_b200.data.batch import NumpyGlobalPermutationJob

    def check(seed, n, rep):
        np.random.seed(seed)
        ref = np.stack([np.random.permutation(n) for _ in range(rep)])
        np.random.seed(seed)
        rows = torch.empty((rep, n), dtype=torch.int32)
        with NumpyGlobalPermutationJob(rows, rep) as job:
            job.wait(rep - 1)
        return np.array_equal(rows.numpy(), ref)

    for k in range(25):
        assert check(k, 3000 + 17 * k, 1 + k % 7), k
    # two jobs interleaved: different generator states, each written to its own rows
    np.random.seed(1)
    s1 = np.random.get_state()
    ref1 = np.stack([np.random.permutation(5000) for _ in range(3)])
    np.random.seed(2)
    ref2 = np.stack([np.random.permutation(7000) for _ in range(4)])
    r1, r2 = torch.empty((3, 5000), dtype=torch.int32), torch.empty((4, 7000), dtype=torch.int32)
    np.random.set_state(s1)
    j1 = NumpyGlobalPermutationJob(r1, 3)
    np.random.seed(2)
    j2 = NumpyGlobalPermutationJob(r2, 4)
    j2.wait(3); j1.wait(2)
    j2.__exit__(None, None, None)
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")            # job 1 finds the global stream moved by job 2: reported, not an error
        j1.__exit__(None, None, None)
    assert np.array_equal(r1.numpy(), ref1) and np.array_equal(r2.numpy(), ref2)
    pid = os.fork()
    if pid == 0:                                   # child: no parked threads survived the fork
        ok = False
        try:
            ok = check(77, 4096, 3)
        finally:
            os._exit(0 if ok else 1)
    _, status = os.waitpid(pid, 0)
    assert os.WIFEXITED(status) and os.WEXITSTATUS(status) == 0


def test_numpy_permutation_job_numa_confinement(tmp_path):
    """The crew is confined to the CPUs of the caller's NUMA node (csrc/hostperm.cu caller_node_cpus).  Fake two-node topology
    through TS_B200_SYSFS_NODE_DIR: the job reports the confinement and still reproduces numpy's stream."""
    import subprocess
    import sys
    cpus = sorted(os.sched_getaffinity(0))
    if len(cpus) < 4:
        pytest.skip("needs >= 4 CPUs")
    half = len(cpus) // 2
    for k, part in enumerate((cpus[:half], cpus[half:])):
        d = tmp_path / f"node{k}"
        d.mkdir()
        (d / "cpulist").write_text(",".join(str(c) for c in part) + "\n")
    code = (
        "import numpy as np, torch\n"
        "from tianshou_b200.data.batch import NumpyGlobalPermutationJob\n"
        "np.random.seed(3); ref = np.stack([np.random.permutation(70001) for _ in range(4)])\n"
        "np.random.seed(3); rows = torch.empty((4, 70001), dtype=torch.int32)\n"
        "with NumpyGlobalPermutationJob(rows, 4) as job:\n"
        "    job.wait(3)\n"
        "assert np.array_equal(rows.numpy(), ref)\n"
        "print('rows ok')\n")
    env = dict(os.environ, TS_B200_SYSFS_NODE_DIR=str(tmp_path), TS_B200_PERM_PIN_MIN_CPUS="2", TS_B200_PERM_TRACE="1",
               PYTHONPATH=os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
    env.pop("TS_B200_PERM_PIN", None)
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "rows ok" in r.stdout, r.stderr[-2000:]
    m = re.search(r"numa_pinned=(\d) \((\d+) cpus\)", r.stderr)
    assert m and m.group(1) == "1" and int(m.group(2)) in (half, len(cpus) - half), r.stderr[-500:]
    env["TS_B200_PERM_PIN"] = "0"
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "numa_pinned=0" in r.stderr


def test_vector_buffer_add_slice_path_equals_fancy_path():
    """Lock-step adds (ids = arange) take the strided-slice write; any other id order takes the fancy-indexed write.
    Same buffer contents, same returned (index, ep_return, ep_len, ep_start) rows (manager.py:131-198)."""
    from tianshou_b200.data import Batch, VectorReplayBuffer
    rng = np.random.default_rng(1)
    E, cap = 12, 5
    a, b = VectorReplayBuffer(E * cap, E), VectorReplayBuffer(E * cap, E)
    for _ in range(13):                                 # wraps every sub-buffer twice
        s = Batch(obs=rng.standard_normal((E, 3)).astype(np.float32), act=rng.integers(0, 2, E), rew=rng.standard_normal(E),
                  terminated=rng.random(E) < 0.2, truncated=np.zeros(E, bool),
                  obs_next=rng.standard_normal((E, 3)).astype(np.float32), info=Batch())
        ra = a.add(s, buffer_ids=np.arange(E))
        perm = rng.permutation(E)
        sb = Batch(obs=s.obs[perm], act=s.act[perm], rew=s.rew[perm], terminated=s.terminated[perm],
                   truncated=s.truncated[perm], obs_next=s.obs_next[perm], info=Batch())
        rb = b.add(sb, buffer_ids=perm)
        for x, y in zip(ra, rb, strict=True):
            assert np.array_equal(np.asarray(x)[perm], np.asarray(y))
    for k in ("obs", "act", "rew", "terminated", "truncated", "done", "obs_next"):
        assert np.array_equal(np.asarray(a._meta[k]), np.asarray(b._meta[k])), k
    assert np.array_equal(a.last_index, b.last_index) and len(a) == len(b)
