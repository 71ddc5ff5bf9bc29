"""Layered networks on the device for the off-policy update bodies (SURVEY 8(f) ranks 2-3).

A ``FusedStack`` is the kernel-side view of a torch module stack made of ``nn.Linear`` / ``nn.Conv2d`` /
``nn.ReLU`` / ``nn.Flatten`` (the reference's ``MLP`` / ``Net`` / ``ContinuousCritic`` / ``DQNet``,
utils/net/common.py:76-369, utils/net/continuous.py:96-238, env/atari/atari_network.py:60-122): every layer's
forward, input gradient and weight gradient is ONE ``ts_net_gemm`` launch (wgmma, fp32-faithful), convolutions
run as implicit GEMM over im2col rows.  A chain of ``EnsembleLinear`` layers (utils/net/common.py, REDQ's critic ensemble)
runs every member of a layer in one batched launch (``ts_net_gemm_batched``) on ``[E, rows, features]`` activations.  Parameters live in a ``FlatGroup`` (flat_params.py: one flat fp32 buffer per optimiser,
``nn.Parameter``s are views of it) so Adam and the Polyak update are single kernels and ``state_dict()`` keeps
working.  There is no autograd graph and no eager-PyTorch path: unsupported layers raise ``UnsupportedModelError``.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Any

import torch
from torch import nn

from .._cabi import ABI, call, load_library, ptr, stream_ptr
from .flat_params import FlatGroup, UnsupportedModelError

ACT_NONE, ACT_RELU, ACT_TANH = ABI.consts["TS_ACT_NONE"], ABI.consts["TS_ACT_RELU"], ABI.consts["TS_ACT_TANH"]


def polyak_update(target: FlatGroup, source: FlatGroup, tau: float) -> None:
    """``polyak_parameter_update`` (utils/lagged_network.py:8-18) on the flat buffers."""
    assert target.n == source.n
    call("ts_polyak_update", ptr(target.flat), ptr(source.flat), target.n, float(tau), stream_ptr(target.device))


@dataclass
class _Layer:
    kind: str                      # "linear" | "conv" | "flatten" | "ensemble"
    weight: nn.Parameter | None = None
    bias: nn.Parameter | None = None
    act: int = ACT_NONE
    in_dim: int = 0
    out_dim: int = 0
    # conv: input NHWC [B, H, W, C] -> output NHWC [B, Ho, Wo, Cout]
    C: int = 0
    H: int = 0
    W: int = 0
    k: int = 0
    s: int = 0
    Ho: int = 0
    Wo: int = 0
    # ensemble: members E; weight [E, in, out] (W_e[k * out + n]), bias [E, 1, out]
    E: int = 0


def layer_params(layers: list[_Layer]) -> list[nn.Parameter]:
    """Every weight and bias of ``layers``, in layer order: the flat order of a ``FlatGroup`` over the chain."""
    return [p for L in layers if L.weight is not None for p in (L.weight, L.bias)]


def _activation_code(m: nn.Module) -> int:
    if type(m) is nn.ReLU:
        return ACT_RELU
    if type(m) is nn.Tanh:
        return ACT_TANH
    raise UnsupportedModelError(f"fused layered networks support ReLU / Tanh activations only, got {m}")


def _flat_chain(mods: list[nn.Module]) -> list[nn.Module]:
    out: list[nn.Module] = []
    for m in mods:
        out += _flat_chain(list(m)) if isinstance(m, nn.Sequential) else [m]
    return out


def compile_sequential(mods: list[nn.Module], input_shape: tuple[int, ...], ensemble: bool = False) -> list[_Layer]:
    """Linear / Conv2d / ReLU / Flatten chain -> layer list.  ``input_shape`` = (features,) or (C, H, W).  Nested
    ``nn.Sequential`` containers are read as the flat chain they run.  With ``ensemble`` a chain of ``EnsembleLinear`` layers
    (with ReLU / Tanh between them) is an ensemble chain: every layer has the same member count and a bias, and no other layer
    kind joins it."""
    from ..utils.net.common import EnsembleLinear
    layers: list[_Layer] = []
    shape = tuple(int(x) for x in input_shape)
    for m in _flat_chain(mods):
        if ensemble and isinstance(m, EnsembleLinear):
            E, d_in, d_out = (int(x) for x in m.weight.shape)
            if len(shape) != 1 or shape[0] != d_in:
                raise UnsupportedModelError(f"EnsembleLinear({d_in}) after shape {shape}")
            if m.bias_weights is None:
                raise UnsupportedModelError("EnsembleLinear layers need a bias")
            layers.append(_Layer("ensemble", m.weight, m.bias_weights, ACT_NONE, d_in, d_out, E=E))
            shape = (d_out,)
        elif isinstance(m, nn.Linear):
            if len(shape) != 1 or shape[0] != m.in_features:
                raise UnsupportedModelError(f"Linear({m.in_features}) after shape {shape}")
            if m.bias is None:
                raise UnsupportedModelError("Linear layers need a bias")
            layers.append(_Layer("linear", m.weight, m.bias, ACT_NONE, m.in_features, m.out_features))
            shape = (m.out_features,)
        elif isinstance(m, nn.Conv2d):
            if len(shape) != 3:
                raise UnsupportedModelError(f"Conv2d after shape {shape}")
            k, s = m.kernel_size, m.stride
            if (k[0] != k[1] or s[0] != s[1] or m.padding not in ((0, 0), 0) or m.dilation != (1, 1) or m.groups != 1
                    or m.bias is None or m.in_channels != shape[0]):
                raise UnsupportedModelError(f"unsupported Conv2d configuration {m}")
            Cc, H, W = shape
            if H < k[0] or W < k[0]:
                raise UnsupportedModelError(f"{m} on a {H} x {W} input: the kernel is larger than the input")
            Ho, Wo = (H - k[0]) // s[0] + 1, (W - k[0]) // s[0] + 1
            layers.append(_Layer("conv", m.weight, m.bias, ACT_NONE, Cc * k[0] * k[0], m.out_channels, C=Cc, H=H, W=W, k=k[0],
                                 s=s[0], Ho=Ho, Wo=Wo))
            shape = (m.out_channels, Ho, Wo)
        elif isinstance(m, nn.Flatten):
            if len(shape) == 3:
                # the stack flattens a convolution's NHWC rows into torch's NCHW order; a network input has no such rows
                # (the frame source feeds the first convolution only, dense rows are NCHW already)
                if not layers:
                    raise UnsupportedModelError(f"Flatten of the {shape} network input: flatten the observation before the "
                                                "network, or start the network with a convolution")
                layers.append(_Layer("flatten", C=shape[0], H=shape[1], W=shape[2], in_dim=shape[0] * shape[1] * shape[2],
                                     out_dim=shape[0] * shape[1] * shape[2]))
                shape = (shape[0] * shape[1] * shape[2],)
        elif isinstance(m, (nn.ReLU, nn.Tanh, nn.Sigmoid, nn.GELU, nn.ELU, nn.LeakyReLU)):
            code = _activation_code(m)
            if not layers or layers[-1].kind == "flatten" or layers[-1].act != ACT_NONE:
                raise UnsupportedModelError("activation without a producing layer")
            layers[-1].act = code
        elif isinstance(m, nn.Identity):
            continue
        else:
            raise UnsupportedModelError(f"layer {m} is outside the fused layered-network family")
    ens = {L.E for L in layers if L.kind == "ensemble"}
    if ens and any(L.kind != "ensemble" for L in layers):
        raise UnsupportedModelError("a chain mixes EnsembleLinear with other layers: an ensemble chain is EnsembleLinear + "
                                    "ReLU / Tanh only")
    if len(ens) > 1:
        raise UnsupportedModelError(f"EnsembleLinear layers of different ensemble sizes {sorted(ens)} in one chain")
    # FusedStack.backward masks a convolution's or a flatten's input gradient with ReLU only: refuse a Tanh there now
    # rather than in the middle of the first update
    for prev, L in zip(layers, layers[1:]):
        if L.kind in ("conv", "flatten") and prev.act == ACT_TANH:
            raise UnsupportedModelError(f"tanh in front of a {'convolution' if L.kind == 'conv' else 'flatten'} is not supported")
    return layers


def _out_shape(layers: list[_Layer], shape: tuple[int, ...]) -> tuple[int, ...]:
    for L in layers:
        if L.kind == "linear":
            shape = (L.out_dim,)
        elif L.kind == "conv":
            shape = (L.out_dim, L.Ho, L.Wo)
        else:
            shape = (L.out_dim,)
    return shape


class FusedStack:
    """Forward / backward of a layer list on ``[rows, features]`` fp32 matrices (NHWC between conv layers)."""

    def __init__(self, layers: list[_Layer], group: FlatGroup, name: str = "net") -> None:
        self.layers = layers
        self.group = group
        self.name = name
        self.device = group.device
        self._bufs: dict[tuple, torch.Tensor] = {}
        self._ws_sizes: dict[tuple[int, int, int], int] = {}
        self._lib = load_library()

    # ------------------------------------------------------------------ scratch
    def _buf(self, key: tuple, n: int) -> torch.Tensor:
        t = self._bufs.get(key)
        if t is None or t.numel() < n:
            t = self._bufs[key] = torch.empty(max(n, 1), dtype=torch.float32, device=self.device)
        return t

    def _gemm(self, a, lda, a_mn, b, ldb, b_mn, c, ldc, M, N, K, bias=None, act=ACT_NONE, mask=None, ld_mask=0,
              mask_kind=ACT_RELU, accumulate=False) -> None:
        ws_n = self._ws_sizes.get((M, N, K))
        if ws_n is None:
            ws_n = self._ws_sizes[(M, N, K)] = int(self._lib.ts_net_gemm_workspace_floats(M, N, K))
        ws = self._buf(("ws",), ws_n) if ws_n > 0 else None
        call("ts_net_gemm", a, lda, a_mn, b, ldb, b_mn, c, ldc, M, N, K, bias, act, mask, ld_mask, int(mask_kind), int(accumulate),
             ptr(ws) if ws is not None else None, ws_n, stream_ptr(self.device))

    def _gemm_batched(self, E, a, lda, a_mn, sa, b, ldb, b_mn, sb, c, ldc, sc, M, N, K, bias=None, s_bias=0, act=ACT_NONE,
                      mask=None, ld_mask=0, s_mask=0, mask_kind=ACT_RELU, accumulate=False) -> None:
        key = (E, M, N, K)
        ws_n = self._ws_sizes.get(key)
        if ws_n is None:
            ws_n = self._ws_sizes[key] = int(self._lib.ts_net_gemm_batched_workspace_floats(E, M, N, K))
        ws = self._buf(("ws",), ws_n) if ws_n > 0 else None
        call("ts_net_gemm_batched", E, a, lda, a_mn, sa, b, ldb, b_mn, sb, c, ldc, sc, M, N, K, bias, s_bias, act, mask, ld_mask,
             s_mask, int(mask_kind), int(accumulate), ptr(ws) if ws is not None else None, ws_n, stream_ptr(self.device))

    def _w(self, L: _Layer, flat: torch.Tensor | None = None) -> int:
        g = self.group
        base = (flat if flat is not None else g.flat).data_ptr()
        return base + 4 * g.offset(L.weight)

    def _b(self, L: _Layer, flat: torch.Tensor | None = None) -> int:
        g = self.group
        base = (flat if flat is not None else g.flat).data_ptr()
        return base + 4 * g.offset(L.bias)

    # ------------------------------------------------------------------ forward
    def forward(self, x: torch.Tensor | None, rows: int, tag: str = "a", *, frames: tuple | None = None,
                params: torch.Tensor | None = None) -> list[torch.Tensor]:
        """Returns the activation list ``[x0, y1, ..., yL]`` (``y_i`` = post-activation output of layer i; for conv layers
        rows * Ho * Wo NHWC rows).  ``frames`` = (uint8 frames, stack_idx int64 [rows, C], denom) feeds the first conv layer
        straight from single-frame storage (frame-stack gather + im2col in one kernel).  ``params``: evaluate with another
        flat parameter buffer of the same layout (the lagged / target copy)."""
        self.group.ensure_adopted()
        st = stream_ptr(self.device)
        acts: list[torch.Tensor] = [x]
        cur = x
        for i, L in enumerate(self.layers):
            if L.kind == "linear":
                y = self._buf((tag, "y", i), rows * L.out_dim)[: rows * L.out_dim].view(rows, L.out_dim)
                self._gemm(ptr(cur), L.in_dim, 0, self._w(L, params), L.in_dim, 0, ptr(y), L.out_dim, rows, L.out_dim, L.in_dim,
                           bias=self._b(L, params), act=L.act)
            elif L.kind == "ensemble":      # [E, rows, out]; the first layer reads the shared [rows, in] input
                n_out = L.E * rows * L.out_dim
                y = self._buf((tag, "y", i), n_out)[:n_out].view(L.E, rows, L.out_dim)
                self._gemm_batched(L.E, ptr(cur), L.in_dim, 0, 0 if i == 0 else rows * L.in_dim, self._w(L, params), L.out_dim, 1,
                                   L.in_dim * L.out_dim, ptr(y), L.out_dim, rows * L.out_dim, rows, L.out_dim, L.in_dim,
                                   bias=self._b(L, params), s_bias=L.out_dim, act=L.act)
            elif L.kind == "conv":
                R = rows * L.Ho * L.Wo
                col = self._buf((tag, "col", i), R * L.in_dim)[: R * L.in_dim].view(R, L.in_dim)
                if i == 0 and frames is not None:
                    fr, sidx, denom = frames
                    call("ts_im2col_u8", ptr(fr), ptr(sidx), rows, L.C, L.H, L.W, L.k, L.s, float(denom), ptr(col), st)
                else:
                    call("ts_im2col_f32", ptr(cur), rows, L.C, L.H, L.W, L.k, L.s, ptr(col), st)
                y = self._buf((tag, "y", i), R * L.out_dim)[: R * L.out_dim].view(R, L.out_dim)
                self._gemm(ptr(col), L.in_dim, 0, self._w(L, params), L.in_dim, 0, ptr(y), L.out_dim, R, L.out_dim, L.in_dim,
                           bias=self._b(L, params), act=L.act)
            else:  # flatten NHWC -> NCHW order
                y = self._buf((tag, "y", i), rows * L.out_dim)[: rows * L.out_dim].view(rows, L.out_dim)
                call("ts_nhwc_to_nchw_flat", ptr(cur), rows, L.H * L.W, L.C, ptr(y), st)
            acts.append(y)
            cur = y
        return acts

    # ------------------------------------------------------------------ tangent (forward-mode) pass
    def jvp(self, acts: list[torch.Tensor], tangent: torch.Tensor, rows: int, tag: str = "a",
            x_dot: torch.Tensor | None = None) -> list[torch.Tensor]:
        """Tangents ``[y1', ..., yL']`` of the layer outputs of ``forward`` (its activation list ``acts``) along the parameter
        direction ``tangent`` (a flat buffer in the group's layout), plus the input tangent ``x_dot`` (None: the input is
        data).  Per Linear layer ``y' = act'(y) * (x W'^T + b' + x' W^T)``: two GEMM launches, the second accumulating (one when
        ``x_dot`` is None)."""
        out: list[torch.Tensor] = []
        cur = x_dot
        for i, L in enumerate(self.layers):
            if L.kind != "linear":
                raise UnsupportedModelError(f"tangent passes support Linear layers only, not {L.kind} layers")
            yd = self._buf((tag, "t", i), rows * L.out_dim)[: rows * L.out_dim].view(rows, L.out_dim)
            mask = ptr(acts[i + 1]) if L.act != ACT_NONE else None
            kind = L.act if L.act != ACT_NONE else ACT_RELU
            self._gemm(ptr(acts[i]), L.in_dim, 0, self._w(L, tangent), L.in_dim, 0, ptr(yd), L.out_dim, rows, L.out_dim, L.in_dim,
                       bias=self._b(L, tangent), mask=mask, ld_mask=L.out_dim, mask_kind=kind)
            if cur is not None:
                self._gemm(ptr(cur), L.in_dim, 0, self._w(L), L.in_dim, 0, ptr(yd), L.out_dim, rows, L.out_dim, L.in_dim,
                           mask=mask, ld_mask=L.out_dim, mask_kind=kind, accumulate=True)
            out.append(yd)
            cur = yd
        return out

    # ------------------------------------------------------------------ backward
    def backward(self, acts: list[torch.Tensor], dy: torch.Tensor, rows: int, tag: str = "a", *, param_grads: bool = True,
                 input_grad: bool = False, input_cols: tuple[int, int] | None = None, dy_preact: bool = False,
                 input_act: tuple[int, torch.Tensor] | None = None, dx_out: torch.Tensor | None = None,
                 dx_accumulate: bool = False) -> torch.Tensor | None:
        """Back-propagate ``dy`` = gradient w.r.t. the LAST layer's output (its activation must be none, or ``dy_preact``: the
        caller already folded the last activation's derivative in).  Weight / bias gradients are STORED into the group's
        gradient buffer (``zero_grad`` + ``backward`` of algorithm_base.py:497-498).  With ``input_grad`` returns d loss /
        d input (columns ``input_cols`` of the first Linear's input), multiplied by the derivative of the activation
        ``input_act = (kind, y)`` that produced this stack's input (a head on top of a trunk; ``y`` holds all of the first
        Linear's input columns, the same columns of it are read), written to / accumulated into ``dx_out`` when given."""
        g = self.group
        st = stream_ptr(self.device)
        n = len(self.layers)
        if self.layers[-1].act != ACT_NONE and not dy_preact:
            raise UnsupportedModelError("backward expects a linear output layer")
        dz = dy                                   # gradient w.r.t. the pre-activation of layer i (mask already applied)
        for i in range(n - 1, -1, -1):
            L = self.layers[i]
            x_in = acts[i]
            prev_act = self._producer_act(i) if i > 0 else (input_act[0] if input_act is not None else ACT_NONE)
            act_src = x_in if i > 0 else (input_act[1] if input_act is not None else None)
            need_dx = i > 0 or input_grad
            if L.kind == "linear":
                M_rows = rows
                if param_grads:
                    gw = g.grad.data_ptr() + 4 * g.offset(L.weight)
                    gb = g.grad.data_ptr() + 4 * g.offset(L.bias)
                    self._gemm(ptr(dz), L.out_dim, 1, ptr(x_in), L.in_dim, 1, gw, L.in_dim, L.out_dim, L.in_dim, M_rows)
                    call("ts_net_colsum", ptr(dz), L.out_dim, M_rows, L.out_dim, gb, 0, st)
                if need_dx:
                    lo, hi = (0, L.in_dim) if (i > 0 or input_cols is None) else input_cols
                    width = hi - lo
                    if i == 0 and dx_out is not None:
                        dx = dx_out
                    else:
                        dx = self._buf((tag, "dx", i), M_rows * width)[: M_rows * width].view(M_rows, width)
                    mask = ptr(act_src) + 4 * lo if prev_act != ACT_NONE else None
                    self._gemm(ptr(dz), L.out_dim, 0, self._w(L) + 4 * lo, L.in_dim, 1, ptr(dx), width, M_rows, width, L.out_dim,
                               mask=mask, ld_mask=L.in_dim, mask_kind=prev_act if prev_act != ACT_NONE else ACT_RELU,
                               accumulate=(i == 0 and dx_accumulate))
                    dz = dx
            elif L.kind == "ensemble":
                s_x = 0 if i == 0 else rows * L.in_dim          # the first layer's input is shared by every member
                s_z = rows * L.out_dim
                if param_grads:
                    gw = g.grad.data_ptr() + 4 * g.offset(L.weight)
                    gb = g.grad.data_ptr() + 4 * g.offset(L.bias)
                    self._gemm_batched(L.E, ptr(x_in), L.in_dim, 1, s_x, ptr(dz), L.out_dim, 1, s_z, gw, L.out_dim,
                                       L.in_dim * L.out_dim, L.in_dim, L.out_dim, rows)
                    call("ts_net_colsum_batched", L.E, ptr(dz), L.out_dim, s_z, rows, L.out_dim, gb, L.out_dim, 0, st)
                if need_dx:
                    lo, hi = (0, L.in_dim) if (i > 0 or input_cols is None) else input_cols
                    width = hi - lo
                    n_dx = L.E * rows * width
                    dx = self._buf((tag, "dx", i), n_dx)[:n_dx].view(L.E, rows, width)
                    mask = ptr(act_src) + 4 * lo if prev_act != ACT_NONE else None
                    self._gemm_batched(L.E, ptr(dz), L.out_dim, 0, s_z, self._w(L) + 4 * lo * L.out_dim, L.out_dim, 0,
                                       L.in_dim * L.out_dim, ptr(dx), width, rows * width, rows, width, L.out_dim, mask=mask,
                                       ld_mask=L.in_dim, s_mask=s_x, mask_kind=prev_act if prev_act != ACT_NONE else ACT_RELU)
                    if i == 0:      # d loss / d input of the shared input: the members' gradients summed in member order
                        out = dx_out if dx_out is not None else self._buf((tag, "dxsum"), rows * width)[: rows * width].view(rows, width)
                        call("ts_net_member_sum", ptr(dx), L.E, rows * width, rows * width, ptr(out), int(dx_accumulate), st)
                        dx = out
                    dz = dx
            elif L.kind == "conv":
                if prev_act == ACT_TANH:
                    raise UnsupportedModelError("tanh in front of a convolution is not supported")
                R = rows * L.Ho * L.Wo
                col = self._bufs[(tag, "col", i)][: R * L.in_dim].view(R, L.in_dim)
                if param_grads:
                    gw = g.grad.data_ptr() + 4 * g.offset(L.weight)
                    gb = g.grad.data_ptr() + 4 * g.offset(L.bias)
                    self._gemm(ptr(dz), L.out_dim, 1, ptr(col), L.in_dim, 1, gw, L.in_dim, L.out_dim, L.in_dim, R)
                    call("ts_net_colsum", ptr(dz), L.out_dim, R, L.out_dim, gb, 0, st)
                if i > 0:
                    dcol = self._buf((tag, "dcol", i), R * L.in_dim)[: R * L.in_dim].view(R, L.in_dim)
                    self._gemm(ptr(dz), L.out_dim, 0, self._w(L), L.in_dim, 1, ptr(dcol), L.in_dim, R, L.in_dim, L.out_dim)
                    dx = self._buf((tag, "dx", i), rows * L.H * L.W * L.C)[: rows * L.H * L.W * L.C]
                    call("ts_col2im_f32", ptr(dcol), rows, L.C, L.H, L.W, L.k, L.s, ptr(x_in) if prev_act == ACT_RELU else None,
                         ptr(dx), st)
                    dz = dx
                elif input_grad:
                    raise UnsupportedModelError("input gradients through the first convolution are not provided")
            else:  # flatten: NCHW-flat gradient back to NHWC rows (+ the producer's ReLU mask)
                if prev_act == ACT_TANH:
                    raise UnsupportedModelError("tanh in front of a flatten is not supported")
                dx = self._buf((tag, "dx", i), rows * L.out_dim)[: rows * L.out_dim]
                call("ts_nchw_flat_to_nhwc", ptr(dz), rows, L.H * L.W, L.C, ptr(x_in) if prev_act == ACT_RELU else None, ptr(dx), st)
                dz = dx
        return dz if input_grad else None

    def _producer_act(self, i: int) -> int:
        """Activation that produced the input of layer i (looking through a flatten)."""
        j = i - 1
        while j >= 0 and self.layers[j].kind == "flatten":
            j -= 1
        return self.layers[j].act if j >= 0 else ACT_NONE


def module_layers(mod: Any) -> list[nn.Module]:
    """Flat module list of the reference-shaped containers: MLP / Net (``.model`` chains) or a plain Sequential."""
    if isinstance(mod, nn.Sequential):
        return list(mod)
    inner = getattr(mod, "model", None)
    if inner is not None:
        return module_layers(inner)
    net = getattr(mod, "net", None)            # DQNet
    if isinstance(net, nn.Sequential):
        return list(net)
    raise UnsupportedModelError(f"cannot read a layer chain from {type(mod).__name__}")
