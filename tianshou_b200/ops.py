"""Device-level operators: thin torch-tensor wrappers over the C ABI (``include/ts_b200.h``).

Inputs are CUDA tensors (or numpy arrays, which are uploaded); outputs are CUDA tensors.  All
work is enqueued on torch's current stream; nothing here synchronises with the host.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np
import torch

from . import _cabi
from ._cabi import TS_F32, TS_F64, ActorCriticDesc, PPOHParams, call, ptr, stream_ptr, to_device


def _dev(device: torch.device | str | None) -> torch.device:
    _cabi.require_cuda()
    if device is None:
        return torch.device("cuda", torch.cuda.current_device())
    d = torch.device(device)
    if d.type != "cuda":
        raise _cabi.ExtensionMissingError(f"tianshou_b200 kernels need a CUDA device, got {d}")
    return d


def _dt(t: torch.dtype) -> int:
    if t == torch.float32:
        return TS_F32
    if t == torch.float64:
        return TS_F64
    raise TypeError(f"unsupported dtype {t}")


def _u8(x: np.ndarray | torch.Tensor | None, device: torch.device) -> torch.Tensor | None:
    if x is None:
        return None
    if isinstance(x, np.ndarray) and x.dtype != np.bool_ and x.dtype != np.uint8:
        x = x.astype(bool)
    if isinstance(x, torch.Tensor) and x.dtype not in (torch.bool, torch.uint8):
        x = x != 0
    return to_device(x, device)


# ------------------------------------------------------------------------------------- GAE
def gae(
    v_s: torch.Tensor | np.ndarray,
    v_s_next: torch.Tensor | np.ndarray,
    rew: torch.Tensor | np.ndarray,
    terminated: torch.Tensor | np.ndarray | None,
    truncated: torch.Tensor | np.ndarray | None,
    extra_end: torch.Tensor | np.ndarray | None = None,
    *,
    gamma: float,
    gae_lambda: float,
    rms_state: torch.Tensor | None = None,
    rms_eps: float = 1e-8,
    out_dtype: torch.dtype = torch.float32,
    terminated_ends: bool = True,
    device: torch.device | str | None = None,
    workspace: torch.Tensor | None = None,
    out: tuple[torch.Tensor, torch.Tensor] | None = None,
    batch_moments_out: torch.Tensor | None = None,
) -> tuple[torch.Tensor, torch.Tensor]:
    """(advantages, returns) -- see ``ts_gae`` in include/ts_b200.h.
    Reference: algorithm_base.py:704-719,1085-1140; a2c.py:131-152."""
    dev = v_s.device if isinstance(v_s, torch.Tensor) and v_s.is_cuda else _dev(device)
    v_s = to_device(v_s, dev)
    v_s_next = to_device(v_s_next, dev, dtype=v_s.dtype)
    rew = to_device(rew, dev, dtype=torch.float64)
    n = v_s.numel()
    assert v_s_next.numel() == n and rew.numel() == n
    term, trunc, extra = _u8(terminated, dev), _u8(truncated, dev), _u8(extra_end, dev)
    if out is None:
        adv = torch.empty(n, dtype=out_dtype, device=dev)
        ret = torch.empty(n, dtype=out_dtype, device=dev)
    else:
        adv, ret = out
    lib = _cabi.load_library()
    need = int(lib.ts_gae_workspace_bytes(n))
    if workspace is None or workspace.numel() < need:
        workspace = torch.empty(max(need, 64), dtype=torch.uint8, device=dev)
    call("ts_gae", ptr(v_s), ptr(v_s_next), _dt(v_s.dtype), ptr(rew), ptr(term), ptr(trunc), ptr(extra),
         int(terminated_ends), n, float(gamma), float(gae_lambda), ptr(rms_state), float(rms_eps),
         ptr(batch_moments_out), ptr(adv), ptr(ret), _dt(adv.dtype), ptr(workspace), stream_ptr(dev))
    return adv, ret


# ------------------------------------------------------------------------------- buffer indices
@dataclass
class DeviceBufferMeta:
    """Device copy of the bookkeeping arrays the index kernels read (manager.py:30-49)."""

    offset: torch.Tensor      # int64[E+1]
    done: torch.Tensor        # uint8[B]
    last_index: torch.Tensor  # int64[E]
    lengths: torch.Tensor     # int64[E]
    ins: torch.Tensor | None = None   # int64[E] per-sub-buffer insertion index (None: derived from last_index)

    @property
    def E(self) -> int:
        return self.last_index.numel()

    @property
    def device(self) -> torch.device:
        return self.done.device

    @staticmethod
    def from_host(offset: np.ndarray, done: np.ndarray, last_index: np.ndarray, lengths: np.ndarray,
                  device: torch.device | str | None = None, ins: np.ndarray | None = None) -> "DeviceBufferMeta":
        dev = _dev(device)
        return DeviceBufferMeta(
            to_device(np.asarray(offset, dtype=np.int64), dev),
            to_device(np.asarray(done, dtype=bool), dev),
            to_device(np.asarray(last_index, dtype=np.int64), dev),
            to_device(np.asarray(lengths, dtype=np.int64), dev),
            None if ins is None else to_device(np.asarray(ins, dtype=np.int64), dev),
        )

    def _args(self) -> tuple:
        return (ptr(self.offset), self.E, ptr(self.done), ptr(self.last_index), ptr(self.lengths))


def _idx(index: np.ndarray | torch.Tensor, dev: torch.device) -> torch.Tensor:
    if isinstance(index, np.ndarray):
        index = np.asarray(index, dtype=np.int64)
    return to_device(index, dev, dtype=torch.int64)


def next_index(meta: DeviceBufferMeta, index: np.ndarray | torch.Tensor) -> torch.Tensor:
    idx = _idx(index, meta.device)
    out = torch.empty_like(idx)
    o, E, d, l, n = meta._args()
    call("ts_next_index", ptr(idx), idx.numel(), o, E, d, l, n, ptr(out), stream_ptr(meta.device))
    return out


def prev_index(meta: DeviceBufferMeta, index: np.ndarray | torch.Tensor) -> torch.Tensor:
    idx = _idx(index, meta.device)
    out = torch.empty_like(idx)
    o, E, d, l, n = meta._args()
    call("ts_prev_index", ptr(idx), idx.numel(), o, E, d, l, n, ptr(out), stream_ptr(meta.device))
    return out


def stack_next_indices(meta: DeviceBufferMeta, index: np.ndarray | torch.Tensor, n_step: int) -> torch.Tensor:
    idx = _idx(index, meta.device).reshape(-1)
    out = torch.empty((n_step, idx.numel()), dtype=torch.int64, device=meta.device)
    o, E, d, l, n = meta._args()
    call("ts_stack_next_indices", ptr(idx), idx.numel(), int(n_step), o, E, d, l, n, ptr(out),
         stream_ptr(meta.device))
    return out


def unfinished_index_raw(meta: DeviceBufferMeta) -> tuple[torch.Tensor, torch.Tensor]:
    """(slots[E], count[1]) on the device, no host sync (manager.py:85-91)."""
    out = torch.empty(meta.E, dtype=torch.int64, device=meta.device)
    cnt = torch.zeros(1, dtype=torch.int64, device=meta.device)
    o, E, d, l, n = meta._args()
    call("ts_unfinished_index", o, E, d, l, n, ptr(meta.ins), ptr(out), ptr(cnt), stream_ptr(meta.device))
    return out, cnt


def unfinished_index(meta: DeviceBufferMeta) -> torch.Tensor:
    """Ordered unfinished slots (device int64[count]); one D2H of the count."""
    out, cnt = unfinished_index_raw(meta)
    return out[: int(cnt.item())]


def sample_all_indices(meta: DeviceBufferMeta, capacity: int | None = None) -> torch.Tensor:
    cap = int(meta.done.numel() if capacity is None else capacity)
    out = torch.empty(cap, dtype=torch.int64, device=meta.device)
    seg = torch.empty(meta.E + 1, dtype=torch.int64, device=meta.device)
    tot = torch.zeros(1, dtype=torch.int64, device=meta.device)
    call("ts_sample_all_indices", ptr(meta.offset), meta.E, ptr(meta.last_index), ptr(meta.lengths), ptr(meta.ins),
         ptr(seg), ptr(out), cap, ptr(tot), stream_ptr(meta.device))
    return out[: int(tot.item())]


def buffer_end_flags(meta: DeviceBufferMeta) -> torch.Tensor:
    out = torch.empty_like(meta.done)
    call("ts_buffer_end_flags", ptr(meta.done), ptr(meta.offset), ptr(meta.last_index), ptr(meta.lengths),
         meta.E, ptr(out), stream_ptr(meta.device))
    return out


def mark_members(idx: torch.Tensor, members: torch.Tensor, table_size: int,
                 table: torch.Tensor | None = None, count: torch.Tensor | None = None) -> torch.Tensor:
    """np.isin(idx, members[:count]) as uint8 (algorithm_base.py:715); ``count`` is an optional
    device int64[1] so that no host sync is needed for a variable-length member list."""
    dev = idx.device
    if table is None:
        table = torch.zeros(table_size, dtype=torch.uint8, device=dev)
    out = torch.empty(idx.numel(), dtype=torch.uint8, device=dev)
    call("ts_mark_members", ptr(idx), idx.numel(), ptr(members) if members.numel() else None, ptr(count),
         members.numel(), ptr(table), table.numel(), ptr(out), stream_ptr(dev))
    return out


def gather_rows(src: torch.Tensor, idx: torch.Tensor, out: torch.Tensor | None = None) -> torch.Tensor:
    """src[idx] along dim 0 for a dense tensor (buffer_base.py:605-649)."""
    assert src.is_contiguous()
    n = idx.numel()
    row_bytes = (src[0].numel() if src.dim() > 1 else 1) * src.element_size()
    if out is None:
        out = torch.empty((n, *src.shape[1:]), dtype=src.dtype, device=src.device)
    call("ts_gather_rows", ptr(src), row_bytes, ptr(idx), n, ptr(out), stream_ptr(src.device))
    return out


def buffer_rows(buffer, key: str, indices: np.ndarray | torch.Tensor, device: torch.device,
                cols: dict[str, torch.Tensor] | None = None) -> torch.Tensor:
    """buffer[key][indices] as a dense fp32 [I, width] device tensor: gathered from the device mirror ``cols`` (default: the
    buffer's own, when it keeps one) with no host traffic, else a host gather of the sampled rows + one upload."""
    if cols is None and hasattr(buffer, "device_columns"):
        cols = buffer.device_columns()
    if cols is not None and key in cols:
        idx = indices if isinstance(indices, torch.Tensor) else to_device(np.asarray(indices, dtype=np.int64), device)
        src = cols[key]
        return gather_rows(src.reshape(src.shape[0], -1), idx).to(torch.float32)
    arr = np.asarray(buffer._meta[key])[np.asarray(indices)]
    return to_device(np.ascontiguousarray(arr.reshape(len(arr), -1)), device, dtype=torch.float32)


def value_mask_rows(target_q: torch.Tensor, terminated: torch.Tensor, idx: torch.Tensor) -> None:
    I = idx.numel()
    A = target_q.numel() // max(I, 1)
    call("ts_value_mask_rows", ptr(target_q), ptr(terminated), ptr(idx), I, A, stream_ptr(target_q.device))


def nstep_return(rew: torch.Tensor, end_flag: torch.Tensor, target_q: torch.Tensor, stacked_idx: torch.Tensor,
                 gamma: float, n_step: int, out_dtype: torch.dtype = torch.float32) -> torch.Tensor:
    I = stacked_idx.shape[1]
    A = target_q.numel() // max(I, 1)
    out = torch.empty((I, A), dtype=out_dtype, device=rew.device)
    call("ts_nstep_return", ptr(rew), ptr(end_flag), ptr(target_q), ptr(stacked_idx), I, A, int(n_step),
         float(gamma), ptr(out), _dt(out_dtype), stream_ptr(rew.device))
    return out


# ------------------------------------------------------------------------------------ sum tree
def segtree_setitem(tree: torch.Tensor, bound: int, index: torch.Tensor, value: torch.Tensor) -> None:
    call("ts_segtree_setitem", ptr(tree), bound, ptr(index), ptr(value), _dt(value.dtype), index.numel(),
         stream_ptr(tree.device))


def segtree_reduce(tree: torch.Tensor, bound: int, start: int, end: int) -> torch.Tensor:
    out = torch.empty(1, dtype=torch.float64, device=tree.device)
    call("ts_segtree_reduce", ptr(tree), bound, int(start), int(end), ptr(out), stream_ptr(tree.device))
    return out


def segtree_prefix_sum_idx(tree: torch.Tensor, bound: int, value: torch.Tensor) -> torch.Tensor:
    out = torch.empty(value.numel(), dtype=torch.int64, device=tree.device)
    call("ts_segtree_prefix_sum_idx", ptr(tree), bound, ptr(value), value.numel(), ptr(out),
         stream_ptr(tree.device))
    return out


def segtree_sample(tree: torch.Tensor, bound: int, u: torch.Tensor) -> torch.Tensor:
    out = torch.empty(u.numel(), dtype=torch.int64, device=tree.device)
    call("ts_segtree_sample", ptr(tree), bound, ptr(u), u.numel(), ptr(out), stream_ptr(tree.device))
    return out


# ----------------------------------------------------------------------------------- MLP / PPO
def critic_forward(params: torch.Tensor, desc: ActorCriticDesc, obs: torch.Tensor,
                   obs2: torch.Tensor | None = None,
                   out: torch.Tensor | None = None, out2: torch.Tensor | None = None):
    n = obs.shape[0]
    if out is None:
        out = torch.empty(n, dtype=torch.float32, device=obs.device)
    if obs2 is not None and out2 is None:
        out2 = torch.empty(n, dtype=torch.float32, device=obs.device)
    call("ts_critic_forward", ptr(params), C.byref(desc), ptr(obs), ptr(out), ptr(obs2), ptr(out2), n,
         stream_ptr(obs.device))
    return (out, out2) if obs2 is not None else out


@dataclass
class NextAliasMap:
    """Which rows of ``obs_next`` repeat the following row of ``obs`` (``ts_next_alias_map``): ``alias`` uint8[n],
    ``extra`` int32[n] of which the first ``count[0]`` entries list the rows with ``alias == 0`` in ascending order."""

    alias: torch.Tensor
    extra: torch.Tensor
    count: torch.Tensor       # int32[1] on the device: reading it is a host sync, the kernels never need one


def next_alias_map(obs: torch.Tensor, obs_next: torch.Tensor, out: NextAliasMap | None = None,
                   workspace: torch.Tensor | None = None) -> NextAliasMap:
    n, dev = obs.shape[0], obs.device
    assert obs.dtype == torch.float32 and obs_next.dtype == torch.float32 and obs.shape == obs_next.shape
    if out is None:
        out = NextAliasMap(torch.empty(n, dtype=torch.uint8, device=dev), torch.empty(n, dtype=torch.int32, device=dev),
                           torch.empty(1, dtype=torch.int32, device=dev))
    need = int(_cabi.load_library().ts_next_alias_workspace_bytes(n))
    if workspace is None or workspace.numel() < need:
        workspace = torch.empty(max(need, 4), dtype=torch.uint8, device=dev)
    call("ts_next_alias_map", ptr(obs), ptr(obs_next), n, obs[0].numel() if n else 1, ptr(out.alias), ptr(out.extra),
         ptr(out.count), ptr(workspace), stream_ptr(dev))
    return out


def critic_forward_dedup(params: torch.Tensor, desc: ActorCriticDesc, obs: torch.Tensor, obs_next: torch.Tensor,
                         amap: NextAliasMap, out: torch.Tensor | None = None, out2: torch.Tensor | None = None):
    """``critic_forward(params, desc, obs, obs_next)`` with one evaluation per distinct row; ``amap`` must be
    ``next_alias_map(obs, obs_next)`` of these very tensors.  Same bits as ``critic_forward``."""
    n = obs.shape[0]
    if out is None:
        out = torch.empty(n, dtype=torch.float32, device=obs.device)
    if out2 is None:
        out2 = torch.empty(n, dtype=torch.float32, device=obs.device)
    call("ts_critic_forward_dedup", ptr(params), C.byref(desc), ptr(obs), ptr(obs_next), ptr(amap.alias), ptr(amap.extra),
         ptr(amap.count), ptr(out), ptr(out2), n, stream_ptr(obs.device))
    return out, out2


def actor_logp(params: torch.Tensor, desc: ActorCriticDesc, obs: torch.Tensor, act: torch.Tensor,
               want_mu: bool = False, out: torch.Tensor | None = None):
    n = obs.shape[0]
    if out is None:
        out = torch.empty(n, dtype=torch.float32, device=obs.device)
    mu = torch.empty((n, desc.act_dim), dtype=torch.float32, device=obs.device) if want_mu else None
    call("ts_actor_logp", ptr(params), C.byref(desc), ptr(obs), ptr(act), n, ptr(out), ptr(mu),
         stream_ptr(obs.device))
    return (out, mu) if want_mu else out


def make_permutation(seed: int, first_epoch: int, n_epochs: int, n: int, device: torch.device) -> torch.Tensor:
    out = torch.empty((n_epochs, n), dtype=torch.int32, device=device)
    call("ts_make_permutation", C.c_uint64(seed & (2**64 - 1)), int(first_epoch), int(n_epochs), int(n),
         ptr(out), stream_ptr(device))
    return out


def narrow_i64_i32(src: torch.Tensor) -> torch.Tensor:
    out = torch.empty(src.shape, dtype=torch.int32, device=src.device)
    call("ts_narrow_i64_i32", ptr(src), src.numel(), ptr(out), stream_ptr(src.device))
    return out


# ------------------------------------------------------------------------------------------------ PSRL
def psrl_update(obs: torch.Tensor, act: torch.Tensor, obs_next: torch.Tensor, rew: torch.Tensor, done: torch.Tensor | None,
                perm: torch.Tensor, *, sq_f32: bool, add_done_loop: bool, state: tuple[torch.Tensor, ...],
                rew_std_prior: torch.Tensor, workspace: torch.Tensor | None, result: torch.Tensor) -> torch.Tensor:
    """``ts_psrl_update``: the posterior update over the rows in ``perm``'s order.  ``obs`` / ``act`` / ``obs_next`` are all int64
    or all float32; ``state`` is (trans_count, rew_mean, rew_std, rew_square_sum, rew_count) on one device, updated in place.
    Returns the workspace (grown when too small: a new one starts zeroed, as the kernels require)."""
    n = perm.numel()
    trans_count, rew_mean = state[0], state[1]
    n_s, n_a = rew_mean.shape
    dev = rew_mean.device
    idx_f32 = obs.dtype == torch.float32
    assert act.dtype == obs.dtype and obs_next.dtype == obs.dtype and (idx_f32 or obs.dtype == torch.int64)
    need = int(_cabi.load_library().ts_psrl_update_workspace_bytes(n, n_s, n_a))
    if workspace is None or workspace.numel() < need:
        workspace = torch.zeros(need, dtype=torch.uint8, device=dev)
    call("ts_psrl_update", ptr(obs), ptr(act), ptr(obs_next), int(idx_f32), ptr(rew), _dt(rew.dtype), int(sq_f32), ptr(done),
         int(add_done_loop), ptr(perm), n, n_s, n_a, ptr(trans_count), ptr(rew_mean), *(ptr(t) for t in state[2:]),
         ptr(rew_std_prior), ptr(workspace), workspace.numel(), ptr(result), stream_ptr(dev))
    return workspace


def psrl_observe(batch: tuple[torch.Tensor, ...], state: tuple[torch.Tensor, ...], rew_std_prior: torch.Tensor,
                 flag: torch.Tensor, result: torch.Tensor) -> None:
    """``ts_psrl_observe``: ``batch`` = dense (trans_count, rew_sum, rew_square_sum, rew_count) float64 device arrays."""
    n_s, n_a = state[1].shape
    call("ts_psrl_observe", *(ptr(t) for t in batch), n_s, n_a, *(ptr(t) for t in state), ptr(rew_std_prior), ptr(flag),
         ptr(result), stream_ptr(state[1].device))


def psrl_max_states() -> int:
    return int(_cabi.load_library().ts_psrl_max_states())


def psrl_value_iteration(trans_prob: torch.Tensor, rew: torch.Tensor, noise: torch.Tensor, gamma: float, eps: float,
                         max_iterations: int, value: torch.Tensor, scratch: torch.Tensor | None = None,
                         out: torch.Tensor | None = None) -> tuple[torch.Tensor, torch.Tensor]:
    """``ts_psrl_value_iteration``: ``value`` is updated in place when the sweeps converge.  Returns (scratch, out) with ``out``
    int64 [n_state + 3] = (policy, sweeps, converged, bits of the last max |V' - V|), still on the device."""
    n_s, n_a = rew.shape
    dev = rew.device
    need = int(_cabi.load_library().ts_psrl_value_iteration_scratch_bytes(n_s, n_a))
    if scratch is None or scratch.numel() < need:
        scratch = torch.empty(need, dtype=torch.uint8, device=dev)
    if out is None:
        out = torch.empty(n_s + 3, dtype=torch.int64, device=dev)
    call("ts_psrl_value_iteration", ptr(trans_prob), ptr(rew), ptr(noise), n_s, n_a, float(gamma), float(eps), int(max_iterations),
         ptr(value), ptr(scratch), ptr(out), stream_ptr(dev))
    return scratch, out


__all__ = [n for n in dir() if not n.startswith("_")]
