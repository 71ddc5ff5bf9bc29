"""``buffer[indices].obs`` / ``.obs_next`` as the layered networks' first layer reads it, without materialising the batch on
the host: dense fp32 rows, or uint8 frames plus the frame slots of every sample for the first convolution's fused
frame-stack + im2col gather.  Shared by the off-policy algorithms whose networks read observations (DQN, discrete SAC).

Reference: data/buffer/buffer_base.py:557-603 (frame stacking), :627-629 (obs_next = obs[next(index)] when it is not
stored), env/atari/atari_network.py:26-55 (the observation divided by a denominator before the network).
"""
from __future__ import annotations

from collections.abc import Callable

import numpy as np
import torch

from .. import ops
from .._cabi import call, ptr, stream_ptr
from ..data import ReplayBuffer
from .flat_params import UnsupportedModelError


class DeviceObsSource:
    """``buffer[indices].obs`` as the kernels read it: either dense fp32 rows ``x`` or (uint8 frames, frame slots per
    sample, scale) for the first convolution's fused frame-stack + im2col gather.  Sized like the batch it stands for.
    ``steps > 1``: ``x`` is a time-major sequence ``[steps * rows, D]`` (step t of sample b at row ``t * rows + b``)."""

    ndim = 1

    def __init__(self, rows: int, x: torch.Tensor | None = None, frames: tuple | None = None, steps: int = 1) -> None:
        self.rows, self.x, self.frames, self.steps = rows, x, frames, steps

    def __len__(self) -> int:
        return self.rows


def device_obs_source(buffer: ReplayBuffer, indices: np.ndarray | torch.Tensor, key: str, in_shape: tuple[int, ...],
                      in_scale: float, device: torch.device,
                      scratch: Callable[[str, tuple[int, ...], torch.dtype], torch.Tensor],
                      seq: bool = False) -> DeviceObsSource:
    """How a network with input shape ``in_shape`` and input denominator ``in_scale`` reads ``buffer[indices].<key>``.
    Convolutional input from a frame-stacking buffer: the S frame slots per sample (prev() chain) + the uint8 frame
    column of the device mirror (or a version-cached upload).  Flat observations: gathered fp32 rows; from a buffer with
    ``stack_num = S > 1`` the S rows of the prev() chain, oldest first (buffer_base.py:585-600), flattened to ``[n, S * D]`` as
    a flat network reads them, or with ``seq`` (a recurrent network over ``D = in_shape[0]`` features per step) as the
    time-major sequence ``[S * n, D]``.  A row width that is not the network's input is refused.  ``scratch(name, shape,
    dtype)`` returns a reusable device tensor for the frame slots."""
    idx = ops._idx(np.asarray(indices) if not isinstance(indices, torch.Tensor) else indices, device)
    if key == "obs_next":
        if buffer._save_obs_next:
            col = "obs_next"
        else:        # obs_next = obs[next(index)] (buffer_base.py:627-629)
            idx, col = ops.next_index(buffer.device_meta(), idx), "obs"
    else:
        col = "obs"
    n = idx.numel()
    if len(in_shape) == 3:
        C, H, W = in_shape
        frames = buffer.device_array(col)
        S = int(buffer.stack_num)
        if frames.dim() == 3 and S == C:                      # single frames [slot, H, W]: stack through prev()
            m = buffer.device_meta()
            sidx = scratch(f"sidx_{key}", (n, S), torch.int64)
            o, E, d, l, ln = m._args()
            call("ts_stack_prev_indices", ptr(idx), n, S, o, E, d, l, ln, ptr(sidx), stream_ptr(device))
            if frames.dtype != torch.uint8:
                raise UnsupportedModelError("frame-stacked image observations must be stored as uint8")
            return DeviceObsSource(n, frames=(frames, sidx, in_scale))
        if frames.dim() == 4 and frames.shape[1] == C and S == 1:   # stored stacks [slot, C, H, W]
            if frames.dtype != torch.uint8:
                raise UnsupportedModelError("image observations must be stored as uint8")
            sidx = (idx.view(n, 1) * C + torch.arange(C, device=device).view(1, C)).contiguous()
            return DeviceObsSource(n, frames=(frames.view(-1, H, W), sidx, in_scale))
        raise UnsupportedModelError(f"observation storage {tuple(frames.shape)} / stack_num {S} does not match the network input {in_shape}")
    src = buffer.device_array(col)
    if seq and (src.dim() != 2 or not src.is_floating_point()):
        raise UnsupportedModelError(f"a recurrent network reads flat float observation rows, the buffer holds {src.dtype} "
                                    f"rows of shape {tuple(src.shape[1:])}")
    src = src.reshape(src.shape[0], -1)
    S, D = int(buffer.stack_num), int(src.shape[1])
    width = D if seq else S * D
    if len(in_shape) != 1 or width != in_shape[0]:
        what = f"{D} features per step" if seq else f"rows of {S} x {D} = {width} features" if S > 1 else f"rows of {D} features"
        raise UnsupportedModelError(f"the buffer holds {what} (stack_num {S}), the network reads {in_shape}")
    if S > 1:            # the prev() chain of every sample, oldest first; time-major for a sequence
        m = buffer.device_meta()
        sidx = scratch(f"sidx_{key}", (n, S), torch.int64)
        o, E, d, l, ln = m._args()
        call("ts_stack_prev_indices", ptr(idx), n, S, o, E, d, l, ln, ptr(sidx), stream_ptr(device))
        if seq:
            sidx = scratch(f"sidx_t_{key}", (S, n), torch.int64).copy_(sidx.t())
        idx = sidx.reshape(-1)
    x = ops.gather_rows(src, idx).to(torch.float32)
    if in_scale != 1.0:
        x = (x.to(torch.float64) / in_scale).to(torch.float32)
    return DeviceObsSource(n, x=x.reshape(S * n, D) if seq else x.reshape(n, width).contiguous(), steps=S if seq else 1)
