"""TEST INFRASTRUCTURE -- float64 restatement of DRQN's update: ``DQN.update`` (dqn.py:365-404, as ``oracle_offpolicy.dqn_update``
restates it) on the reference's ``Recurrent`` network (utils/net/common.py:372-453) with the LSTM written out step by step.

The sampled observations are the buffer's ``stack_num`` rows along the prev() chain, oldest first (buffer_base.py:585-600);
``obs_next`` is that stack at ``next(index)`` when the buffer does not store it, else the stack over the stored ``obs_next``
column (buffer_base.py:627-649).  Every sequence starts from zero ``(h, c)``.  ``order`` feeds the generator's two alternatives
that must move the loss: ``"newest_only"`` (the last row alone) and ``"newest_first"`` (the stack reversed).
"""
from __future__ import annotations

from collections.abc import Callable

import numpy as np
import torch
from torch import nn

from oracle.oracle_offpolicy import compute_nstep_targets, next_index, stacked_obs


class DrqnNet(nn.Module):
    """``Recurrent(layer_num=L, state_shape=D, action_shape=A, hidden_layer_size=H)`` in float64, parameters in the reference's
    ``parameters()`` order: per LSTM layer ``weight_ih [4H, H]``, ``weight_hh [4H, H]``, ``bias_ih``, ``bias_hh``; then
    ``fc1`` (weight, bias), ``fc2`` (weight, bias)."""

    def __init__(self, L: int, D: int, A: int, H: int) -> None:
        super().__init__()
        self.L, self.H = L, H
        shapes = []
        for _ in range(L):
            shapes += [(4 * H, H), (4 * H, H), (4 * H,), (4 * H,)]
        shapes += [(H, D), (H,), (A, H), (A,)]
        self.ps = nn.ParameterList([nn.Parameter(torch.zeros(s, dtype=torch.float64)) for s in shapes])

    def forward(self, obs: torch.Tensor) -> torch.Tensor:
        """obs ``[n, S, D]`` -> Q ``[n, A]``: fc1 on every step, the LSTM layers from zero state, fc2 on the last step's h."""
        p = list(self.ps)
        w1, b1, w2, b2 = p[4 * self.L:]
        x = obs.to(torch.float64) @ w1.T + b1
        n, S, _ = x.shape
        for l in range(self.L):
            w_ih, w_hh, b_ih, b_hh = p[4 * l: 4 * l + 4]
            h = torch.zeros(n, self.H, dtype=torch.float64)
            c = torch.zeros(n, self.H, dtype=torch.float64)
            outs = []
            for t in range(S):
                z = x[:, t] @ w_ih.T + b_ih + h @ w_hh.T + b_hh
                i, f, g, o = z.chunk(4, dim=1)
                i, f, g, o = torch.sigmoid(i), torch.sigmoid(f), torch.tanh(g), torch.sigmoid(o)
                c = f * c + i * g
                h = o * torch.tanh(c)
                outs.append(h)
            x = torch.stack(outs, dim=1)
        return x[:, -1] @ w2.T + b2


def load_from(net: DrqnNet, params: list[torch.Tensor]) -> None:
    with torch.no_grad():
        for p, v in zip(net.ps, params, strict=True):
            p.copy_(torch.as_tensor(np.asarray(v.detach().cpu() if isinstance(v, torch.Tensor) else v), dtype=torch.float64).reshape(p.shape))


def seq_reader(buf: dict, stack: int, order: str = "ref") -> Callable[[np.ndarray, str], torch.Tensor]:
    """``reader(idx, col)``: the stacked rows of column ``col`` at ``idx`` as ``[n, S, D]`` float64, in the reference's order
    (``order="ref"``) or one of the alternatives."""
    def read(idx: np.ndarray, col: str) -> torch.Tensor:
        x = stacked_obs(buf[col], idx, buf, stack)
        if order == "newest_first":
            x = x[:, ::-1]
        elif order == "newest_only":
            x = x[:, -1:]
        return torch.as_tensor(np.ascontiguousarray(x), dtype=torch.float64)
    return read


def drqn_update(net: DrqnNet, net_old: DrqnNet | None, opt: torch.optim.Optimizer, buf: dict, indices: np.ndarray,
                is_weight: np.ndarray | None, gamma: float, n_step: int, is_double: bool, huber: float | None, stack: int,
                obs_next_stored: bool, sync_target: bool = False, order: str = "ref") -> dict:
    """One ``DQN.update`` with a ``Recurrent`` model on ``indices``.  ``sync_target``: the lagged copy is refreshed on this
    iteration, after the n-step targets were formed with the old copy (dqn.py:386, algorithm_base.py:619-623)."""
    read = seq_reader(buf, stack, order)

    def target_q(terminal: np.ndarray) -> torch.Tensor:
        if obs_next_stored:
            x = read(terminal, "obs_next")
        else:
            x = read(next_index(terminal, buf["offset"], buf["done"], buf["last_index"], buf["lengths"]), "obs")
        q_online = net(x)
        q_tgt = net_old(x) if net_old is not None else q_online
        if is_double:
            return q_tgt[np.arange(len(terminal)), q_online.argmax(dim=1)]
        return q_tgt.max(dim=1)[0]

    returns = torch.from_numpy(compute_nstep_targets(buf, indices, target_q, gamma, n_step)).flatten().to(torch.float64)
    if sync_target and net_old is not None:
        net_old.load_state_dict(net.state_dict())
    q = net(read(indices, "obs"))
    q = q[np.arange(len(indices)), buf["act"][indices]]
    td = returns - q
    if huber is not None:
        loss = torch.nn.functional.huber_loss(q.reshape(-1, 1), returns.reshape(-1, 1), delta=huber, reduction="mean")
    else:
        w = torch.as_tensor(is_weight, dtype=torch.float64) if is_weight is not None else 1.0
        loss = (td.pow(2) * w).mean()
    opt.zero_grad(); loss.backward(); opt.step()
    return dict(returns=returns.numpy(), td=td.detach().numpy(), loss=float(loss.detach()))
