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
    sample, scale) for the first convolution's fused frame-stack + im2col gather.  Sized like the batch it stands for."""

    ndim = 1

    def __init__(self, rows: int, x: torch.Tensor | None = None, frames: tuple | None = None) -> None:
        self.rows, self.x, self.frames = rows, x, frames

    def __len__(self) -> int:
        return self.rows


def device_obs_source(buffer: ReplayBuffer, indices: np.ndarray | torch.Tensor, key: str, in_shape: tuple[int, ...],
                      in_scale: float, device: torch.device,
                      scratch: Callable[[str, tuple[int, ...], torch.dtype], torch.Tensor]) -> DeviceObsSource:
    """How a network with input shape ``in_shape`` and input denominator ``in_scale`` reads ``buffer[indices].<key>``.
    Convolutional input from a frame-stacking buffer: the S frame slots per sample (prev() chain) + the uint8 frame
    column of the device mirror (or a version-cached upload).  Flat observations: gathered fp32 rows.  ``scratch(name,
    shape, dtype)`` returns a reusable device tensor for the frame slots."""
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
    x = ops.gather_rows(src.reshape(src.shape[0], -1), idx).to(torch.float32)
    if in_scale != 1.0:
        x = (x.to(torch.float64) / in_scale).to(torch.float32)
    return DeviceObsSource(n, x=x.contiguous())
