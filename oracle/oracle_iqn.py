"""TEST INFRASTRUCTURE -- float64 numpy restatement of IQN's cosine embedding, feature product, target selection and loss rows
(loss, priorities, d loss / d q), and its update on plain torch networks with given fractions.

Only ``tests/`` and ``tools/`` may import this module; ``tianshou_b200`` never does.  It restates
tianshou/algorithm/modelfree/iqn.py and utils/net/discrete.py:126-216 without the framework around it:

  network: discrete.py:126-216 (cos(tau * pi * i) in fp32, ReLU(Linear(C, D)), feat * e, the ``last`` MLP on B * S rows)
  target : qrdqn.py:94-106 through IQNPolicy (iqn.py:72-100): the online arg-max of the sample means, the lagged network's
           quantiles of that action on its own fractions (the online ones when ``target_update_freq == 0``)
  loss   : iqn.py:156-183 (quantile-Huber loss with a fraction per row and sample, the priority), the gradient written out by hand
  lagged : dqn.py:277-286 (full copy when ``_iter % freq == 0``, BEFORE the step, after the targets were formed)

The kernels' layout is q[B][S][A] (sample-major); the reference's and ``IqnNet``'s is q[B, A, S].  The functions below take
whichever layout they say.  ``IqnNet`` with ``reference_loss`` makes ``iqn_update_torch``, the eager baseline of
tools/iqn_timing.py.

PINNING: tests/test_oracle_iqn.py replays tests/golden/iqn_ref_*.npz (outputs of the imported reference,
oracle/gen_golden_iqn.py) through ``iqn_update`` with the recorded fractions, and checks ``iqn_rows`` against float64 autograd of
the reference's ``[B, S_on, 1] x [B, 1, S_t]`` expression.
"""
from __future__ import annotations

import copy
import warnings
from collections.abc import Callable, Iterator

import numpy as np
import torch
from torch import nn

from oracle.oracle_discrete_bcq import cnn_trunk, mlp_trunk, obs_next_of
from oracle.oracle_offpolicy import compute_nstep_targets, mlp


# ------------------------------------------------------------------------------------------------ network pieces, float64
def cos_argument(taus: np.ndarray, C: int) -> np.ndarray:
    """The fp32 argument the reference forms: fl(tau * fl(fl32(pi) * i)), i = 1 .. C, shape [..., C] (discrete.py:144-156)."""
    i_pi = np.float32(np.pi) * np.arange(1, C + 1, dtype=np.float32)
    return np.asarray(taus, np.float32)[..., None] * i_pi


def cos_features(taus: np.ndarray, C: int) -> np.ndarray:
    """cos of that fp32 argument in float64."""
    return np.cos(cos_argument(taus, C).astype(np.float64))


def mix(feat: np.ndarray, e: np.ndarray, S: int) -> np.ndarray:
    """h[b * S + s] = feat[b] * e[b * S + s]   (discrete.py:211-214)."""
    feat, e = np.asarray(feat, np.float64), np.asarray(e, np.float64)
    return (feat[:, None, :] * e.reshape(feat.shape[0], S, -1)).reshape(e.shape)


def mix_backward(dh: np.ndarray, feat: np.ndarray, e: np.ndarray, S: int, trunk_act: str = "none",
                 trunk_out: np.ndarray | None = None) -> tuple[np.ndarray, np.ndarray]:
    """(dfeat [B, D], de_pre [B * S, D]): dfeat = sum_s dh * e times the derivative of the trunk's last activation ("none",
    "relu", "tanh") at its output; de_pre = dh * feat * 1[e > 0], e being the embedding's ReLU output."""
    dh, feat, e = (np.asarray(a, np.float64) for a in (dh, feat, e))
    B, D = feat.shape
    dfeat = (dh.reshape(B, S, D) * e.reshape(B, S, D)).sum(1)
    if trunk_act == "relu":
        dfeat = dfeat * (np.asarray(trunk_out) > 0)
    elif trunk_act == "tanh":
        y = np.asarray(trunk_out, np.float64)
        dfeat = dfeat * (1.0 - y * y)
    de_pre = (dh.reshape(B, S, D) * feat[:, None, :] * (e.reshape(B, S, D) > 0)).reshape(B * S, D)
    return dfeat, de_pre


# ------------------------------------------------------------------------------------------------ target and rows, float64
def iqn_select(q: np.ndarray) -> np.ndarray:
    """The policy's action on q[B][S][A]: the first arg-max of the sample means (qrdqn.py:18-20, iqn.py:97-98)."""
    return np.asarray(q, np.float64).mean(1).argmax(1)


def iqn_target(q_online: np.ndarray, q_next: np.ndarray) -> np.ndarray:
    """``q_next[b, :, a*]`` [B, S_next] with a* the online arg-max; both in the [B][S][A] layout."""
    a = iqn_select(q_online)
    return np.asarray(q_next)[np.arange(len(a)), :, a]


def iqn_rows(q: np.ndarray, act: np.ndarray, returns: np.ndarray, taus: np.ndarray, weight: np.ndarray | None) -> dict:
    """loss, d loss / d q [B, S_on, A] and the priorities [B] on q[B][S_on][A]   (iqn.py:156-183).

    With c_i = q[b, i, act], u_ij = returns[b, j] - c_i, h = smooth_l1(u), w_ij = |taus[b, i] - 1[u_ij <= 0]| (detached):
    qr_b = (1/S_on) sum_ij h_ij w_ij, prio_b = (1/S_on) sum_ij h_ij, loss = mean_b(weight_b qr_b)."""
    q, ret, tau = np.asarray(q, np.float64), np.asarray(returns, np.float64), np.asarray(taus, np.float64)
    B, S_on, _ = q.shape
    rows = np.arange(B)
    w = np.ones(B) if weight is None else np.asarray(weight, np.float64).reshape(-1)
    c = q[rows, :, act]                                 # [B, S_on] over i
    u = ret[:, None, :] - c[:, :, None]                 # [B, i, j]
    au = np.abs(u)
    h = np.where(au < 1.0, 0.5 * u * u, au - 0.5)
    wt = np.abs(tau[:, :, None] - (u <= 0.0))
    qr_b = (h * wt).sum(-1).mean(1)
    prio = h.sum(-1).mean(1)
    dq = np.zeros_like(q)
    dq[rows, :, act] = -(w[:, None] / (B * S_on)) * (wt * np.clip(u, -1.0, 1.0)).sum(-1)
    return dict(loss=float((w * qr_b).mean()), dq=dq, prio=prio, qr_b=qr_b)


def reference_loss(q: torch.Tensor, act: np.ndarray | torch.Tensor, returns: torch.Tensor, taus: torch.Tensor,
                   weight: torch.Tensor | float) -> tuple[torch.Tensor, torch.Tensor]:
    """(loss, prio): iqn.py:163-179 in torch on q[B, A, S_on] (the reference's layout), the ``[B, S_on, 1] x [B, 1, S_t]``
    broadcast written as the reference writes it (any dtype, any device)."""
    F = torch.nn.functional
    act = torch.as_tensor(act, device=q.device)
    curr_dist = q[torch.arange(len(act), device=q.device), act, :].unsqueeze(2)
    target_dist = returns.unsqueeze(1)
    with warnings.catch_warnings():
        warnings.filterwarnings("ignore", message="Using a target size")      # the broadcast is intended
        dist_diff = F.smooth_l1_loss(target_dist, curr_dist, reduction="none")
    huber_loss = (dist_diff * (taus.unsqueeze(2) - (target_dist - curr_dist).detach().le(0.0).to(q.dtype)).abs()).sum(-1).mean(1)
    return (huber_loss * weight).mean(), dist_diff.detach().abs().sum(-1).mean(1)


# ------------------------------------------------------------------------------------------------ networks
class IqnNet(nn.Module):
    """``ImplicitQuantileNetwork`` as plain modules in the reference's parameter order: ``preprocess`` (the trunk), ``last``,
    ``embed`` (Linear(C, D); ReLU after it).  ``forward(x, taus)`` -> q[B, A, S] on the given fractions."""

    def __init__(self, trunk: nn.Module, feat: int, last_hidden: tuple[int, ...], A: int, C: int):
        super().__init__()
        self.preprocess = trunk
        self.last = mlp([feat, *last_hidden, A], False)
        self.embed = nn.Linear(C, feat)
        self.C = C

    def forward(self, x: torch.Tensor, taus: torch.Tensor) -> torch.Tensor:
        feat = self.preprocess(x)
        B, S = taus.shape
        i_pi = np.pi * torch.arange(1, self.C + 1, dtype=taus.dtype, device=taus.device)
        e = torch.relu(self.embed(torch.cos(taus.view(B, S, 1) * i_pi).view(B * S, self.C)))
        h = (feat.unsqueeze(1) * e.view(B, S, -1)).view(B * S, -1)
        return self.last(h).view(B, S, -1).transpose(1, 2)


def net_from_cfg(g) -> IqnNet:
    """The network a golden file's ``cfg_*`` entries describe."""
    if str(g["cfg_kind"]) == "cnn":
        trunk, feat = cnn_trunk(4, int(g["cfg_H"]), int(g["cfg_W"]))
    else:
        trunk, feat = mlp_trunk(int(g["cfg_obs"]), tuple(int(x) for x in g["cfg_hidden"]), int(g["cfg_trunk_out"]))
    return IqnNet(trunk(), feat, tuple(int(x) for x in g["cfg_last"]), int(g["cfg_A"]), int(g["cfg_C"]))


# ------------------------------------------------------------------------------------------------ update
class IqnState:
    """The network, its lagged copy (None: ``target_update_freq == 0``), Adam and the iteration counter."""

    def __init__(self, net: IqnNet, lr: float, freq: int):
        self.net = net
        self.old = copy.deepcopy(net) if freq > 0 else None
        self.opt = torch.optim.Adam(net.parameters(), lr=lr)
        self.freq = freq
        self.iter = 0


def iqn_update(s: IqnState, obs_of: Callable[[np.ndarray], torch.Tensor], buf: dict, indices: np.ndarray,
               is_weight: np.ndarray | None, gamma: float, n_step: int, S_on: int, S_t: int, taus: Iterator[torch.Tensor]) -> dict:
    """One ``IQN.update`` on the sampled ``indices`` with the fractions taken from ``taus`` in the reference's draw order (the
    target's online forward, the lagged forward when there is one, the step's forward): the forwards in torch fp32, the rows in
    float64 numpy, their gradient pushed back through the network with autograd."""
    dev = next(s.net.parameters()).device

    def target_q(terminal: np.ndarray) -> torch.Tensor:
        x = obs_next_of(obs_of, buf, terminal, dev)
        q = s.net(x, next(taus)).transpose(1, 2)
        q_next = s.old(x, next(taus)).transpose(1, 2) if s.old is not None else q
        return torch.from_numpy(iqn_target(q.cpu().numpy(), q_next.cpu().numpy()))

    returns = compute_nstep_targets(buf, indices, target_q, gamma, n_step).reshape(len(indices), -1)
    assert returns.shape[1] == (S_t if s.old is not None else S_on)
    if s.old is not None and s.iter % s.freq == 0:
        s.old.load_state_dict(s.net.state_dict())
    s.iter += 1
    tau = next(taus)
    assert tau.shape == (len(indices), S_on)
    q = s.net(obs_of(indices), tau).transpose(1, 2)            # [B, S_on, A]
    act = np.asarray(buf["act"])[indices].astype(np.int64).reshape(-1)
    r = iqn_rows(q.detach().cpu().numpy(), act, returns, tau.cpu().numpy(), is_weight)
    s.opt.zero_grad()
    q.backward(torch.as_tensor(r["dq"], dtype=torch.float32, device=dev))
    s.opt.step()
    return dict(returns=returns, loss=r["loss"], prio=r["prio"])


def iqn_update_torch(s: IqnState, obs_of: Callable[[np.ndarray], torch.Tensor], buf: dict, indices: np.ndarray, gamma: float,
                     n_step: int, S_on: int, S_t: int) -> float:
    """The same update as the reference runs it in eager PyTorch: fractions from ``torch.rand`` on the network's device, the
    target there, the n-step return on the host (algorithm_base.py:721-817), the loss by ``reference_loss`` and autograd,
    torch's Adam.  Returns the loss."""
    dev = next(s.net.parameters()).device

    def target_q(terminal: np.ndarray) -> torch.Tensor:
        x = obs_next_of(obs_of, buf, terminal, dev)
        B = x.shape[0]
        q = s.net(x, torch.rand(B, S_on, device=dev))
        if s.old is None:
            return q[torch.arange(B, device=dev), q.mean(2).argmax(1), :].cpu()
        q_next = s.old(x, torch.rand(B, S_t, device=dev))
        return q_next[torch.arange(B, device=dev), q.mean(2).argmax(1), :].cpu()

    returns = torch.as_tensor(compute_nstep_targets(buf, indices, target_q, gamma, n_step).reshape(len(indices), -1), device=dev)
    if s.old is not None and s.iter % s.freq == 0:
        s.old.load_state_dict(s.net.state_dict())
    s.iter += 1
    tau = torch.rand(len(indices), S_on, device=dev)
    q = s.net(obs_of(indices), tau)
    act = torch.as_tensor(np.asarray(buf["act"])[indices].astype(np.int64), device=dev)
    loss = reference_loss(q, act, returns, tau, 1.0)[0]
    s.opt.zero_grad()
    loss.backward()
    s.opt.step()
    return loss.item()
