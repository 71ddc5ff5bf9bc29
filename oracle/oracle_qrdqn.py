"""TEST INFRASTRUCTURE -- float64 numpy restatement of QR-DQN's and discrete CQL's target selection, loss rows, losses, loss
gradient and priorities, and their update on plain torch networks.

Only ``tests/`` and ``tools/`` may import this module; ``tianshou_b200`` never does.  It restates
tianshou/algorithm/modelfree/qrdqn.py and imitation/discrete_cql.py without the framework around it (no Batch / Policy /
Collector):

  target : qrdqn.py:94-106 (the lagged quantiles at the online arg-max of the quantile means, :18-20), algorithm_base.py:721-817
  loss   : qrdqn.py:108-131 (quantile-Huber loss, the priority), discrete_cql.py:80-113 (+ min_q_weight * the log-sum-exp penalty
           over the quantile means), the gradient written out by hand
  lagged : dqn.py:277-286 (full copy when ``_iter % freq == 0``, BEFORE the step, after the targets were formed)

``quantile_net`` is the plain layer chain of ``Net(num_atoms=N)`` / ``QRDQNet`` in the reference's parameter order, returning
``[B, A, N]``; with ``reference_loss`` (the reference's loss expression in torch) it makes ``qrdqn_update_torch``, the eager
baseline of tools/qrdqn_timing.py.

PINNING: tests/test_oracle_qrdqn.py replays tests/golden/{qrdqn,dcql}_ref_*.npz (outputs of the imported reference,
oracle/gen_golden_qrdqn.py) through ``qrdqn_update``, and checks ``qr_rows`` against float64 autograd of the reference's
broadcast expression.
"""
from __future__ import annotations

import copy
import warnings
from collections.abc import Callable

import numpy as np
import torch
from torch import nn

from oracle.oracle_offpolicy import compute_nstep_targets, mlp, nature_cnn
from oracle.oracle_discrete_bcq import obs_next_of


def tau_hat(N: int) -> np.ndarray:
    """The quantile midpoints as the reference forms them: fp32 ``(linspace(0, 1, N + 1)[:-1] + [1:]) / 2`` (qrdqn.py:86-91)."""
    tau = torch.linspace(0, 1, N + 1)
    return ((tau[:-1] + tau[1:]) / 2).numpy()


# ------------------------------------------------------------------------------------------------ rows, float64
def qr_select(q: np.ndarray) -> np.ndarray:
    """The policy's action on ``[B, A, N]`` quantiles: the first arg-max of the quantile means (qrdqn.py:18-20)."""
    return np.asarray(q, np.float64).mean(2).argmax(1)


def qr_target(q_online: np.ndarray, q_next: np.ndarray) -> np.ndarray:
    """``q_next[b, a*, :]`` with a* the online arg-max   (qrdqn.py:94-106)."""
    a = qr_select(q_online)
    return np.asarray(q_next)[np.arange(len(a)), a, :]


def qr_rows(q: np.ndarray, act: np.ndarray, returns: np.ndarray, tau: np.ndarray, weight: np.ndarray | None,
            min_q_weight: float = 0.0) -> dict:
    """(loss, qr_loss, cql_loss), d loss / d q ``[B, A, N]`` and the priorities ``[B]`` (qrdqn.py:108-131, discrete_cql.py:80-113).

    With c_i = q[b, act, i], u_ij = returns[b, j] - c_i, h = smooth_l1(u) and w_ij = |tau_i - 1[u_ij <= 0]| (detached):
    qr_b = (1/N) sum_ij h_ij w_ij, prio_b = (1/N) sum_ij h_ij, qr_loss = mean_b(weight_b qr_b), cql_loss = mean_b(logsumexp_a m_a
    - m_act) over the quantile means m."""
    q, ret, tau = np.asarray(q, np.float64), np.asarray(returns, np.float64), np.asarray(tau, np.float64).reshape(-1)
    B, A, N = q.shape
    rows = np.arange(B)
    w = np.ones(B) if weight is None else np.asarray(weight, np.float64).reshape(-1)
    c = q[rows, act, :]                                 # [B, N] over i
    u = ret[:, None, :] - c[:, :, None]                 # [B, i, j]
    au = np.abs(u)
    h = np.where(au < 1.0, 0.5 * u * u, au - 0.5)
    wt = np.abs(tau[None, :, None] - (u <= 0.0))
    qr_b = (h * wt).sum(-1).mean(1)
    prio = h.sum(-1).mean(1)
    qr_loss = (w * qr_b).mean()
    dq = np.zeros_like(q)
    dq[rows, act, :] = -(w[:, None] / (B * N)) * (wt * np.clip(u, -1.0, 1.0)).sum(-1)
    cql_loss = 0.0
    if min_q_weight != 0.0:
        m = q.mean(2)
        mx = m.max(1, keepdims=True)
        lse = mx[:, 0] + np.log(np.exp(m - mx).sum(1))
        cql_loss = (lse - m[rows, act]).mean()
        p = np.exp(m - lse[:, None])
        p[rows, act] -= 1.0
        dq += (min_q_weight / (B * N)) * p[:, :, None]
    return dict(losses=np.array([qr_loss + min_q_weight * cql_loss, qr_loss, cql_loss]), dq=dq, prio=prio)


def reference_loss(q: torch.Tensor, act: np.ndarray | torch.Tensor, returns: torch.Tensor, tau: torch.Tensor,
                   weight: torch.Tensor | float, min_q_weight: float) -> tuple[torch.Tensor, ...]:
    """(loss, qr_loss, cql_loss, prio): qrdqn.py:114-128 and discrete_cql.py:86-106 in torch, the ``[B, N, 1] x [B, 1, N]``
    broadcast written as the reference writes it (any dtype, any device)."""
    F = torch.nn.functional
    act = torch.as_tensor(act, device=q.device)
    curr_dist = q[torch.arange(len(act), device=q.device), act, :].unsqueeze(2)
    target_dist = returns.unsqueeze(1)
    with warnings.catch_warnings():
        warnings.filterwarnings("ignore", message="Using a target size")      # the broadcast is intended
        dist_diff = F.smooth_l1_loss(target_dist, curr_dist, reduction="none")
    huber_loss = (dist_diff * (tau.view(1, -1, 1) - (target_dist - curr_dist).detach().le(0.0).to(q.dtype)).abs()).sum(-1).mean(1)
    qr_loss = (huber_loss * weight).mean()
    prio = dist_diff.detach().abs().sum(-1).mean(1)
    m = q.mean(2)
    min_q_loss = m.logsumexp(1).mean() - m.gather(1, act.unsqueeze(1)).mean()
    return qr_loss + min_q_loss * min_q_weight, qr_loss, min_q_loss, prio


# ------------------------------------------------------------------------------------------------ networks
class QuantileView(nn.Module):
    """A layer chain whose last Linear has A * N outputs, viewed as ``[B, A, N]``."""

    def __init__(self, chain: nn.Sequential, A: int, N: int):
        super().__init__()
        self.chain, self.A, self.N = chain, A, N

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return self.chain(x).view(-1, self.A, self.N)


def quantile_net(kind: str, A: int, N: int, obs: int = 0, hidden: tuple[int, ...] = (), H: int = 0, W: int = 0) -> QuantileView:
    """``Net(state_shape=obs, action_shape=A, hidden_sizes=hidden, num_atoms=N)`` or ``QRDQNet(c=4, h=H, w=W, action_shape=A,
    num_quantiles=N)`` (common.py:298-369, atari_network.py:211-235)."""
    chain = nature_cnn(4, H, W, A * N) if kind == "cnn" else mlp([obs, *hidden, A * N], False)
    return QuantileView(chain, A, N)


def net_from_cfg(g) -> QuantileView:
    if str(g["cfg_kind"]) == "cnn":
        return quantile_net("cnn", int(g["cfg_A"]), int(g["cfg_N"]), H=int(g["cfg_H"]), W=int(g["cfg_W"]))
    return quantile_net("mlp", int(g["cfg_A"]), int(g["cfg_N"]), obs=int(g["cfg_obs"]), hidden=tuple(int(x) for x in g["cfg_hidden"]))


# ------------------------------------------------------------------------------------------------ update
class QrState:
    """The network, its lagged copy (None: ``target_update_freq == 0``), Adam and the iteration counter."""

    def __init__(self, net: QuantileView, lr: float, freq: int):
        self.net = net
        self.old = copy.deepcopy(net) if freq > 0 else None
        self.opt = torch.optim.Adam(net.parameters(), lr=lr)
        self.freq = freq
        self.iter = 0


def qrdqn_update(s: QrState, obs_of: Callable[[np.ndarray], torch.Tensor], buf: dict, indices: np.ndarray, is_weight: np.ndarray | None,
                 gamma: float, n_step: int, min_q_weight: float = 0.0) -> dict:
    """One ``QRDQN.update`` (``min_q_weight == 0``) or ``DiscreteCQL.update`` on the sampled ``indices``: the forwards in torch
    fp32, the rows in float64 numpy, their gradient pushed back through the network with autograd."""
    dev = next(s.net.parameters()).device
    N = s.net.N

    def target_q(terminal: np.ndarray) -> torch.Tensor:
        x = obs_next_of(obs_of, buf, terminal, dev)
        q = s.net(x)
        q_next = s.old(x) if s.old is not None else q
        return torch.from_numpy(qr_target(q.cpu().numpy(), q_next.cpu().numpy()))

    returns = compute_nstep_targets(buf, indices, target_q, gamma, n_step).reshape(-1, N)
    if s.old is not None and s.iter % s.freq == 0:
        s.old.load_state_dict(s.net.state_dict())
    s.iter += 1
    q = s.net(obs_of(indices))
    act = np.asarray(buf["act"])[indices].astype(np.int64).reshape(-1)
    r = qr_rows(q.detach().cpu().numpy(), act, returns, tau_hat(N), is_weight, min_q_weight)
    s.opt.zero_grad()
    q.backward(torch.as_tensor(r["dq"], dtype=torch.float32, device=dev))
    s.opt.step()
    return dict(returns=returns, losses=r["losses"], prio=r["prio"])


def qrdqn_update_torch(s: QrState, obs_of: Callable[[np.ndarray], torch.Tensor], buf: dict, indices: np.ndarray, gamma: float,
                       n_step: int, min_q_weight: float = 0.0) -> float:
    """The same update as the reference runs it in eager PyTorch: the target on the network's device, the n-step return on the
    host (algorithm_base.py:721-817), the loss by ``reference_loss`` and autograd, torch's Adam.  Returns the loss."""
    dev = next(s.net.parameters()).device
    N = s.net.N
    tau = torch.as_tensor(tau_hat(N), device=dev)

    def target_q(terminal: np.ndarray) -> torch.Tensor:
        x = obs_next_of(obs_of, buf, terminal, dev)
        q = s.net(x)
        q_next = s.old(x) if s.old is not None else q
        return q_next[torch.arange(len(terminal), device=dev), q.mean(2).argmax(1), :].cpu()

    returns = torch.as_tensor(compute_nstep_targets(buf, indices, target_q, gamma, n_step).reshape(-1, N), device=dev)
    if s.old is not None and s.iter % s.freq == 0:
        s.old.load_state_dict(s.net.state_dict())
    s.iter += 1
    q = s.net(obs_of(indices))
    act = torch.as_tensor(np.asarray(buf["act"])[indices].astype(np.int64), device=dev)
    loss = reference_loss(q, act, returns, tau, 1.0, min_q_weight)[0]
    s.opt.zero_grad()
    loss.backward()
    s.opt.step()
    return loss.item()
