"""Plumbing shared by the off-policy and offline test modules: the device handles, stand-ins for the action spaces, readers of
the golden files, ptxas's register report, hooks that capture what an update sampled and computed, and the machinery that
runs an update at one batch size after another."""
import contextlib
import copy
import math
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from oracle import oracle_discrete_sac as ods
from ts_testutil import Box, record_parity  # noqa: F401  (Box(dim, m) is this family's continuous action space)

DEV = "cuda:0"
EPS = float(np.finfo(np.float32).eps)
GEMM_BK = 64            # net_gemm's K chunk: a GEMM can split K only from two chunks on
B_SMALL, B_LARGE = 17, 200          # one K chunk / four K chunks; CQL and BCQ repeat them to 170 / 2000 rows


def stream():
    from tianshou_b200._cabi import stream_ptr
    return stream_ptr(torch.device(DEV))


def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ------------------------------------------------------------------------------------------------------------ action spaces
class Discrete:
    def __init__(self, n):
        self.n = n
        self.shape = ()


class MultiDiscrete:
    def __init__(self, nvec):
        self.nvec = np.asarray(nvec)
        self.shape = self.nvec.shape


# ------------------------------------------------------------------------------------------------------------ goldens
def golden_cfg(g):
    """A golden's ``cfg_*`` entries without the prefix."""
    return {k[4:]: g[k] for k in g.files if k.startswith("cfg_")}


def load_params(mod, g, prefix):
    """The golden's ``<prefix><i>`` arrays into the module's parameters, in ``parameters()`` order."""
    with torch.no_grad():
        for i, p in enumerate(mod.parameters()):
            p.copy_(torch.as_tensor(g[f"{prefix}{i}"]).reshape(p.shape))


def check_params(tag, mod, g, prefix, lr, view=None):
    """The module's parameters against the golden's ``<prefix><i>``: Adam normalises a step to ~lr per element, so the absolute
    term is stated in units of one step.  ``view`` maps a parameter to what the golden stores (default: all of it)."""
    view = view or (lambda t: t.detach().cpu().numpy())
    for i, p in enumerate(mod.parameters()):
        record_parity(f"{tag}/{prefix}{i}", view(p), g[f"{prefix}{i}"], rtol=1e-3, atol=0.1 * lr)


def oracle_buffer(g):
    """The arrays ``oracle_td3.nstep_targets`` reads, for the single buffer of a golden."""
    d = {k: g["buf_" + k] for k in ("obs", "act", "rew", "done", "terminated", "obs_next")}
    size, n = len(g["buf_obs"]), int(g["buf_len"])
    last = (int(g["buf_insertion_idx"]) - 1) % n
    d.update(offset=np.array([0, size]), last_index=g["buf_last_index"], lengths=np.array([n]),
             unfinished=[last] if not d["done"][last] else [])
    return d


def vector_buffer_from_golden(g, mirror=False):
    """The vector buffer of a discrete golden's rollout (``roll<i>_*``); prioritised when the golden sets ``cfg_per``, and for
    the CNN goldens a four-frame stack of which only the last frame is stored."""
    from tianshou_b200.data import Batch, PrioritizedVectorReplayBuffer, VectorReplayBuffer
    E, cap = int(g["cfg_E"]), int(g["cfg_cap"])
    cnn = str(g["cfg_kind"]) == "cnn"
    kw = dict(stack_num=4, ignore_obs_next=True, save_only_last_obs=True) if cnn else {}
    if "cfg_per" in g.files and bool(g["cfg_per"]):
        buf = PrioritizedVectorReplayBuffer(E * cap, E, alpha=float(g["cfg_alpha"]), beta=float(g["cfg_beta"]), device=DEV,
                                            device_mirror=mirror, **kw)
    else:
        buf = VectorReplayBuffer(E * cap, E, device=DEV, device_mirror=mirror, **kw)
    for i in range(int(g["cfg_steps"])):
        s = {k: g[f"roll{i}_{k}"] for k in ("obs", "act", "rew", "terminated", "truncated")}
        if cnn:
            s["obs"] = np.repeat(s["obs"][:, None], 4, axis=1)        # only the last frame is stored
            s["obs_next"] = s["obs"]
        else:
            s["obs_next"] = g[f"roll{i}_obs_next"]
        buf.add(Batch(**s), buffer_ids=np.arange(E))
    return buf


def check_final_state(tag, g, algo, lagged=None):
    """Final parameters / Adam moments / lagged parameters of a discrete Q-learning algorithm within the bars DESIGN.md
    section 4 uses for DQN and the discrete offline algorithms: Adam normalises a step to ~lr per element, so the absolute term
    is stated in units of one step.  Without ``lagged`` the lagged parameters are ``algo.model_old``'s, and there must be as
    many of them as online ones exactly when the golden updates a target network."""
    view = ods.golden_view if bool(g["cfg_compact"]) else (lambda t: t.detach().cpu().numpy())
    lr = float(g["cfg_lr"])
    grp = algo._group
    for i, p in enumerate(grp.params):
        record_parity(f"{tag}/pf_{i}", view(p), g[f"pf_{i}"], rtol=1e-3, atol=0.1 * lr)
        m, v = g[f"m_{i}"], g[f"v_{i}"]
        record_parity(f"{tag}/m_{i}", view(grp.view(grp.exp_avg, p).view(p.shape)), m, rtol=2e-3, atol=2e-3 * float(np.abs(m).max()) + 1e-12)
        record_parity(f"{tag}/v_{i}", view(grp.view(grp.exp_avg_sq, p).view(p.shape)), v, rtol=4e-3, atol=4e-3 * float(np.abs(v).max()) + 1e-20)
    assert grp.sync_step_from_device() == int(g["adam_step"]) and algo._iter == int(g["iter"])
    if lagged is None:
        lagged = list(algo.model_old.parameters()) if algo.model_old is not None else []
        assert len(lagged) == (len(grp.params) if int(g["cfg_freq"]) > 0 else 0)
    for i, p in enumerate(lagged):
        record_parity(f"{tag}/old_{i}", view(p), g[f"old_{i}"], rtol=1e-3, atol=0.1 * lr)


# ------------------------------------------------------------------------------------------------------------ register report
def ptxas_log(cu_file, out_dir):
    """What nvcc prints compiling one source under tianshou_b200/csrc with the build's flags (ptxas -v for sm_90a).  Skips when
    there is no nvcc."""
    from tianshou_b200.csrc import build as B
    if shutil.which(B.NVCC) is None and not os.path.exists(B.NVCC):
        pytest.skip("nvcc not available")
    src = os.path.join(B.HERE, cu_file)
    r = subprocess.run([B.NVCC, *B.FLAGS, "-c", src, "-o", os.path.join(str(out_dir), os.path.basename(src) + ".o")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    return r.stdout + r.stderr


def parse_ptxas(log):
    """{entry: (stack frame, spill stores, spill loads)} in bytes, from ptxas's report."""
    return {m.group(1): (int(m.group(2)), int(m.group(3)), int(m.group(4))) for m in re.finditer(
        r"Compiling entry function '(\S+)' for 'sm_90a'\n(?:.*\n)*?\s*(\d+) bytes stack frame, (\d+) bytes spill "
        r"stores, (\d+) bytes spill loads", log)}


def ptxas_report(cu_file, out_dir):
    return parse_ptxas(ptxas_log(cu_file, out_dir))


def assert_spill_free(report):
    """Every entry of the report without a stack frame or spills."""
    assert report and all(v == (0, 0, 0) for v in report.values()), report


# ------------------------------------------------------------------------------------------------------------ capture
@contextlib.contextmanager
def capture_batches(algo):
    """Inside the block, every update records into the yielded dict the sampled ``indices`` (numpy), the ``returns`` of the
    preprocessed batch and the ``prio`` the update hands back (device tensors, or None where the batch has none)."""
    cap = {}
    orig_pre, orig_post = algo._preprocess_batch, algo._postprocess_batch

    def pre(batch, buffer, indices):
        b = orig_pre(batch, buffer, indices)
        r = b.__dict__.get("returns")
        cap["indices"], cap["returns"] = np.asarray(indices).copy(), None if r is None else torch.as_tensor(r).detach().clone()
        return b

    def post(batch, buffer, indices):
        w = batch.__dict__.get("weight")
        cap["prio"] = None if w is None else torch.as_tensor(w).detach().clone()
        return orig_post(batch, buffer, indices)

    algo._preprocess_batch, algo._postprocess_batch = pre, post
    try:
        yield cap
    finally:
        algo._preprocess_batch, algo._postprocess_batch = orig_pre, orig_post


@contextlib.contextmanager
def capture_grads(group, step="adam_step"):
    """Inside the block, the group's flat gradient ``grad[:n]`` is appended to the yielded list before each of its optimiser
    steps (``step`` names the method: FQF's fraction group takes ``optimizer_step``)."""
    grads = []
    real = getattr(type(group), step)

    def hooked(optimizer, mgn):
        grads.append(group.grad[: group.n].clone())
        real(group, optimizer, mgn)

    setattr(group, step, hooked)
    try:
        yield grads
    finally:
        delattr(group, step)


# ------------------------------------------------------------------------------------------------------------ batch edges
def grid_caps():
    """How many items (threads, or rows for the warp- and block-per-row kernels) one launch covers before its grid is capped and
    it strides; every item past a cap is reached only by the kernel's grid-stride loop."""
    s = sm_count()
    return {"net_ops_1d": s * 16 * 256,      # net_ops.cu TS_LAUNCH_1D: 16 blocks of 256 threads per SM, an item per thread
            "offpolicy_1d": s * 4 * 256,     # grid_for of td3.cu / cql.cu / bcq.cu: 4 blocks of 256 threads per SM
            "warp_per_row": s * 16 * 8,      # row_grid of row_sums.cuh / discrete_sac.cu: 16 blocks of 8 warps per SM
            "block_per_row": s * 8,          # ts_qrdqn_rows / ts_iqn_rows: 8 blocks per SM, a block per row
            "iqn_1d": s * 8 * 256}           # ew_grid of iqn.cu: 8 blocks of 256 threads per SM


def gemm_splits_k(K, M=64, N=64):
    """Whether ``ts_net_gemm`` splits K for a one-tile output (every weight gradient of the small networks below)."""
    from tianshou_b200._cabi import load_library
    return int(load_library().ts_net_gemm_workspace_floats(M, N, K)) > 0


def _flat_groups(algo):
    from tianshou_b200.algorithm.flat_params import FlatGroup
    out = []
    for v in vars(algo).values():
        for x in (v if isinstance(v, (list, tuple)) else (v,)):
            if isinstance(x, FlatGroup):
                out.append(x)
    return out


def _fused_stacks(algo):
    """Every FusedStack the algorithm reaches through its own (non-module) attributes: the networks' scratch owners."""
    from tianshou_b200.algorithm.netgraph import FusedStack
    found, seen = [], set()

    def walk(x, depth):
        if id(x) in seen or depth > 3 or isinstance(x, (torch.nn.Module, torch.Tensor)):
            return
        seen.add(id(x))
        if isinstance(x, FusedStack):
            found.append(x)
        elif isinstance(x, (list, tuple)):
            for y in x:
                walk(y, depth + 1)
        elif isinstance(x, dict):
            for y in x.values():
                walk(y, depth + 1)
        elif type(x).__module__.startswith("tianshou_b200.algorithm"):
            for y in vars(x).values():
                walk(y, depth + 1)

    for v in vars(algo).values():
        walk(v, 0)
    return found


def poison_scratch(algo):
    """NaN into every floating tensor of the algorithm's DeviceScratch and every FusedStack buffer (workspace included)."""
    n = 0
    for t in list(algo._scratch.values()) + [t for s in _fused_stacks(algo) for t in s._bufs.values()]:
        if isinstance(t, torch.Tensor) and t.is_floating_point() and t.is_cuda:
            t.fill_(float("nan"))
            n += 1
    return n


def rng_state(buf):
    return copy.deepcopy((buf.__dict__["_random_state"], buf.__dict__.get("_child_rngs")))


def set_rng_state(buf, state):
    rs, child = copy.deepcopy(state)
    buf.__dict__["_random_state"] = rs
    if child is not None:
        buf.__dict__["_child_rngs"] = child


def seeded_update(algo, buf, B, seed):
    """One update with every random source seeded: what ``capture_batches`` recorded, and the scalar statistics it returned."""
    from tianshou_b200.utils import policy_within_training_step
    np.random.seed(seed)
    torch.manual_seed(seed)
    with capture_batches(algo) as cap, policy_within_training_step(algo.policy):
        stats = algo.update(buffer=buf, sample_size=B)
    torch.cuda.synchronize()
    scalars = {k: v for k, v in vars(stats).items() if k != "train_time" and (v is None or isinstance(v, (int, float)))}
    return cap, scalars


def carry_outside_state_dict(a, b):
    """What the reference keeps outside ``state_dict()`` and whoever restores a run carries over by hand: the plain update
    counters, CQL's Lagrange multiplier with its Adam, AutoAlpha's Adam."""
    for attr in ("_iter", "_cnt", "_last"):
        if hasattr(a, attr):
            setattr(b, attr, copy.copy(getattr(a, attr)))
    if getattr(a, "with_lagrange", False):
        with torch.no_grad():
            b.cql_log_alpha.copy_(a.cql_log_alpha)
        b.cql_alpha_optim.load_state_dict(copy.deepcopy(a.cql_alpha_optim.state_dict()))
    alpha_optim = getattr(getattr(a, "alpha", None), "_optim", None)
    if alpha_optim is not None:
        b.alpha._optim.load_state_dict(copy.deepcopy(alpha_optim.state_dict()))


def optimiser_state(algo):
    """Every flat group's parameters, Adam moments and step, four tensors per group."""
    out = []
    for g in _flat_groups(algo):
        out += [g.flat.clone(), g.exp_avg.clone(), g.exp_avg_sq.clone(), torch.tensor([g.sync_step_from_device()])]
    return out


def check_second_batch_size(build, buf, B1, B2, carry=carry_outside_state_dict, name=""):
    """A ``B1`` update, every scratch tensor filled with NaN, then a ``B2`` update: the indices, statistics, priorities written
    back and every flat group's state must equal, bit for bit, the ``B2`` update of a fresh instance loaded from the same
    ``state_dict()`` with the same random state.  Returns the first instance's capture and state."""
    a = build()
    seeded_update(a, buf, B1, seed=1)
    b = build()
    b.load_state_dict(copy.deepcopy(a.state_dict()))
    carry(a, b)
    rng = rng_state(buf)
    assert poison_scratch(a) > 0
    cap_a, stats_a = seeded_update(a, buf, B2, seed=2)
    set_rng_state(buf, rng)
    cap_b, stats_b = seeded_update(b, buf, B2, seed=2)
    assert np.array_equal(cap_a["indices"], cap_b["indices"]) and len(cap_a["indices"]) == B2
    assert stats_a == stats_b, f"{name}: losses differ after a batch of {B1}: {stats_a} vs {stats_b}"
    assert all(v is None or math.isfinite(v) for v in stats_a.values())
    if cap_a["prio"] is not None:
        assert cap_a["prio"].numel() == B2 and torch.equal(cap_a["prio"], cap_b["prio"])
    sa, sb = optimiser_state(a), optimiser_state(b)
    for i, (x, y) in enumerate(zip(sa, sb, strict=True)):
        assert torch.equal(x, y), f"{name}: state tensor {i} (group {i // 4}, {('flat', 'exp_avg', 'exp_avg_sq', 'step')[i % 4]}) differs"
    return cap_a, sa
