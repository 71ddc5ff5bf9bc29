"""The recurrent Q-network of DRQN on the device: ``Recurrent`` (utils/net/common.py) = ``fc1`` -> ``nn.LSTM`` (L layers) -> ``fc2``
on the last step, forward and backpropagation through time over a time-major sequence ``[S * rows, D]`` (step t of sample b at
row ``t * rows + b``, as ``device_obs_source(seq=True)`` gathers it from a frame-stacking buffer).

Every GEMM is one ``ts_net_gemm`` launch (fp32-faithful bf16x3): ``fc1`` over all ``S * rows`` rows; per layer the input
projection of every step in one launch, then per step the recurrent product accumulated into that step's block and the cell
(``ts_lstm_cell``, which adds ``b_hh``).  The backward runs the top layer first: ``fc2``'s input gradient enters at the last step
only, per step ``ts_lstm_cell_bwd`` and ``dh_{t-1} = dgates_t W_hh``; then ``dW_ih``, ``dX`` (the ``dh`` of the layer below) and
``dW_hh`` (over the ``(S - 1) * rows`` rows where ``h_{t-1}`` and ``dgates_t`` are contiguous blocks) in one launch each, and
``db_ih = db_hh = colsum(dgates)``.  Training starts every sequence from zero ``(h, c)``, as the reference's ``policy(batch)`` with
``state=None`` does.

Reference: utils/net/common.py:372-453 (Recurrent), torch.nn.LSTM (gate chunks i, f, g, o), test/discrete/test_drqn.py.
"""
from __future__ import annotations

from typing import Any

import torch
from torch import nn

from .._cabi import call, ptr, stream_ptr
from .flat_params import FlatGroup, UnsupportedModelError
from .netgraph import FusedStack


def check_recurrent(model: Any) -> tuple[nn.Linear, nn.LSTM, nn.Linear]:
    """(fc1, lstm, fc2) of a network shaped like the reference's ``Recurrent``; anything else raises ``UnsupportedModelError``."""
    from ..utils.net.common import Recurrent
    if not isinstance(model, Recurrent):
        raise UnsupportedModelError(f"expected a Recurrent network, got {type(model).__name__}")
    fc1, lstm, fc2 = model.fc1, model.nn, model.fc2
    if type(lstm) is not nn.LSTM:
        raise UnsupportedModelError(f"Recurrent.nn must be an nn.LSTM, got {type(lstm).__name__}")
    if not lstm.bias:
        raise UnsupportedModelError("an LSTM without biases (bias=False) is not supported")
    if lstm.proj_size > 0:
        raise UnsupportedModelError("an LSTM with projections (proj_size > 0) is not supported")
    if lstm.bidirectional:
        raise UnsupportedModelError("a bidirectional LSTM is not supported")
    if lstm.dropout > 0:
        raise UnsupportedModelError("an LSTM with dropout between layers is not supported")
    if not lstm.batch_first:
        raise UnsupportedModelError("the LSTM must be batch_first, as Recurrent builds it")
    for lin, name in ((fc1, "fc1"), (fc2, "fc2")):
        if type(lin) is not nn.Linear or lin.bias is None:
            raise UnsupportedModelError(f"Recurrent.{name} must be an nn.Linear with a bias")
    if not fc1.out_features == lstm.input_size == lstm.hidden_size == fc2.in_features:
        raise UnsupportedModelError(f"fc1 -> LSTM -> fc2 widths do not chain: {fc1.out_features} -> ({lstm.input_size}, "
                                    f"{lstm.hidden_size}) -> {fc2.in_features}")
    return fc1, lstm, fc2


class RecurrentStack(FusedStack):
    """Forward / backward of a ``Recurrent`` network with ``FusedStack``'s contract: ``forward(x, rows, tag, params=...)`` returns
    an activation list whose last entry is the ``[rows, actions]`` output, ``backward(acts, dq, rows, tag)`` stores every
    parameter's gradient into the group.  ``x`` is ``[S * rows, D]`` time-major; S follows from its length.  The flat group is
    ``model.parameters()`` in order (the LSTM's, then fc1's, then fc2's), so a lagged copy of the model is a prefix of it.
    Scratch lives in ``FusedStack._bufs``."""

    def __init__(self, model: Any, device: torch.device, name: str = "q") -> None:
        self.fc1, self.lstm, self.fc2 = check_recurrent(model)
        super().__init__([], FlatGroup(list(model.parameters()), device), name)
        self.D, self.H, self.A = self.fc1.in_features, self.lstm.hidden_size, self.fc2.out_features
        self.L = self.lstm.num_layers
        self.cells = [tuple(getattr(self.lstm, f"{k}_l{l}") for k in ("weight_ih", "weight_hh", "bias_ih", "bias_hh"))
                      for l in range(self.L)]

    def _p(self, p: nn.Parameter, flat: torch.Tensor | None = None) -> int:
        return (flat if flat is not None else self.group.flat).data_ptr() + 4 * self.group.offset(p)

    def _g(self, p: nn.Parameter) -> int:
        return self.group.grad.data_ptr() + 4 * self.group.offset(p)

    def _scratch(self, tag: str, what: str, n: int, l: int = 0) -> torch.Tensor:
        return self._buf((tag, what, l), n)[:n]

    # ------------------------------------------------------------------ forward
    def forward(self, x: torch.Tensor, rows: int, tag: str = "a", *, frames: tuple | None = None,
                params: torch.Tensor | None = None, noise: torch.Tensor | None = None) -> list[torch.Tensor]:
        """``[x, y0, (gates, c, h) of every layer ..., q]``: ``y0 = fc1(x)`` and each layer's gates / c / h are ``[S * rows, .]``
        time-major, ``q = fc2(h_top at the last step)`` is ``[rows, A]``.  ``params``: another flat buffer of the same layout."""
        if frames is not None or x is None:
            raise UnsupportedModelError("a Recurrent network reads flat observation rows")
        self.group.ensure_adopted()
        st = stream_ptr(self.device)
        D, H, A, H4 = self.D, self.H, self.A, 4 * self.H
        S = x.shape[0] // rows
        R = S * rows
        y0 = self._scratch(tag, "y0", R * H).view(R, H)
        self._gemm(ptr(x), D, 0, self._p(self.fc1.weight, params), D, 0, ptr(y0), H, R, H, D, bias=self._p(self.fc1.bias, params))
        acts: list[torch.Tensor] = [x, y0]
        cur = y0
        pre = self._scratch(tag, "pre", R * H4)
        for l, (w_ih, w_hh, b_ih, b_hh) in enumerate(self.cells):
            gates = self._scratch(tag, "gates", R * H4, l).view(R, H4)
            c = self._scratch(tag, "c", R * H, l).view(R, H)
            h = self._scratch(tag, "h", R * H, l).view(R, H)
            self._gemm(ptr(cur), H, 0, self._p(w_ih, params), H, 0, ptr(pre), H4, R, H4, H, bias=self._p(b_ih, params))
            for t in range(S):
                pt = ptr(pre) + 4 * t * rows * H4
                if t > 0:
                    self._gemm(ptr(h) + 4 * (t - 1) * rows * H, H, 0, self._p(w_hh, params), H, 0, pt, H4, rows, H4, H,
                               accumulate=True)
                call("ts_lstm_cell", pt, self._p(b_hh, params), ptr(c) + 4 * (t - 1) * rows * H if t > 0 else None, rows, H,
                     ptr(gates) + 4 * t * rows * H4, ptr(c) + 4 * t * rows * H, ptr(h) + 4 * t * rows * H, st)
            acts += [gates, c, h]
            cur = h
        q = self._scratch(tag, "q", rows * A).view(rows, A)
        self._gemm(ptr(cur) + 4 * (S - 1) * rows * H, H, 0, self._p(self.fc2.weight, params), H, 0, ptr(q), A, rows, A, H,
                   bias=self._p(self.fc2.bias, params))
        acts.append(q)
        return acts

    # ------------------------------------------------------------------ backward
    def backward(self, acts: list[torch.Tensor], dy: torch.Tensor, rows: int, tag: str = "a", **kw: Any) -> None:
        """Back-propagate ``dy`` = d loss / d q ``[rows, A]`` through time; every parameter's gradient is STORED into the group's
        gradient buffer (the online parameters only)."""
        if kw:
            raise UnsupportedModelError(f"RecurrentStack.backward takes no options, got {sorted(kw)}")
        st = stream_ptr(self.device)
        D, H, A, H4 = self.D, self.H, self.A, 4 * self.H
        x, y0 = acts[0], acts[1]
        S = x.shape[0] // rows
        R = S * rows
        top_h = acts[-2]
        self._gemm(ptr(dy), A, 1, ptr(top_h) + 4 * (S - 1) * rows * H, H, 1, self._g(self.fc2.weight), H, A, H, rows)
        call("ts_net_colsum", ptr(dy), A, rows, A, self._g(self.fc2.bias), 0, st)
        dh = self._scratch(tag, "dh", R * H).view(R, H)          # d loss / d h of the current layer, then its dX in place
        self._gemm(ptr(dy), A, 0, self._p(self.fc2.weight), H, 1, ptr(dh) + 4 * (S - 1) * rows * H, H, rows, H, A)
        dc = self._scratch(tag, "dc", rows * H)
        dg = self._scratch(tag, "dgates", R * H4).view(R, H4)
        for l in range(self.L - 1, -1, -1):
            w_ih, w_hh, b_ih, b_hh = self.cells[l]
            gates, c, h = acts[2 + 3 * l: 5 + 3 * l]
            x_l = y0 if l == 0 else acts[4 + 3 * (l - 1)]
            for t in range(S - 1, -1, -1):
                dht = ptr(dh) + 4 * t * rows * H
                if t < S - 1:        # dh_t (+)= dgates_{t+1} W_hh; the top layer has no gradient from above before the last step
                    self._gemm(ptr(dg) + 4 * (t + 1) * rows * H4, H4, 0, self._p(w_hh), H, 1, dht, H, rows, H, H4,
                               accumulate=l < self.L - 1)
                call("ts_lstm_cell_bwd", ptr(gates) + 4 * t * rows * H4, ptr(c) + 4 * t * rows * H,
                     ptr(c) + 4 * (t - 1) * rows * H if t > 0 else None, dht, ptr(dc) if t < S - 1 else None, rows, H,
                     ptr(dg) + 4 * t * rows * H4, ptr(dc) if t > 0 else None, st)
            self._gemm(ptr(dg), H4, 1, ptr(x_l), H, 1, self._g(w_ih), H, H4, H, R)
            if S > 1:
                self._gemm(ptr(dg) + 4 * rows * H4, H4, 1, ptr(h), H, 1, self._g(w_hh), H, H4, H, (S - 1) * rows)
            else:            # a length-1 sequence never reads W_hh
                self.group.view(self.group.grad, w_hh).zero_()
            call("ts_net_colsum", ptr(dg), H4, R, H4, self._g(b_ih), 0, st)
            call("ts_net_colsum", ptr(dg), H4, R, H4, self._g(b_hh), 0, st)
            self._gemm(ptr(dg), H4, 0, self._p(w_ih), H, 1, ptr(dh), H, R, H, H4)
        self._gemm(ptr(dh), H, 1, ptr(x), D, 1, self._g(self.fc1.weight), D, H, D, R)
        call("ts_net_colsum", ptr(dh), H, R, H, self._g(self.fc1.bias), 0, st)
