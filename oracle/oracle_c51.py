"""TEST INFRASTRUCTURE -- float64 numpy restatement of C51's softmax, expected values, target selection, projection,
cross-entropy, logit gradient and priorities, and its update on plain torch networks.

Only ``tests/`` and ``tools/`` may import this module; ``tianshou_b200`` never does.  It restates
tianshou/algorithm/modelfree/c51.py without the framework around it (no Batch / Policy / Collector):

  returns : c51.py:110-111 (the support repeated per row as the n-step target), algorithm_base.py:721-817
  lagged  : dqn.py:277-286 (full copy when ``_iter % freq == 0``), c51.py:143 -- BEFORE the target is formed
  target  : c51.py:113-136 (the lagged distribution at the online arg-max of the expected values, :62-63, at s_{t+1}: the
            batch's ``obs_next``; the clamp and the dense projection)
  loss    : c51.py:145-160 (cross-entropy with 1e-8 inside the log, the weighted mean, the unweighted priority), the gradient
            with respect to the raw logits written out by hand

``categorical_net`` is the plain layer chain of ``Net(softmax=True, num_atoms=N)`` / ``C51Net`` in the reference's parameter
order: ``logits`` returns the raw ``[B, A, N]`` output, ``forward`` the per-action softmax the reference's model returns.  With
``reference_loss`` (the reference's loss expression in torch) it makes ``c51_update_torch``, the eager baseline of
tools/c51_timing.py.

PINNING: tests/test_oracle_c51.py replays tests/golden/c51_ref_*.npz (outputs of the imported reference,
oracle/gen_golden_c51.py) through ``c51_update``, and checks ``c51_rows`` against float64 autograd of the reference's
expression.
"""
from __future__ import annotations

import copy
from collections.abc import Callable

import numpy as np
import torch
from torch import nn

from oracle.oracle_discrete_bcq import obs_next_of
from oracle.oracle_offpolicy import compute_nstep_targets, mlp, nature_cnn


def support(N: int, v_min: float, v_max: float) -> np.ndarray:
    """The reference's fp32 ``torch.linspace(v_min, v_max, N)`` on the CPU (c51.py:59-62)."""
    return torch.linspace(v_min, v_max, N).numpy()


# ------------------------------------------------------------------------------------------------ rows, float64
def softmax(x: np.ndarray) -> np.ndarray:
    """Softmax over the last axis (the atoms)."""
    x = np.asarray(x, np.float64)
    e = np.exp(x - x.max(-1, keepdims=True))
    return e / e.sum(-1, keepdims=True)


def c51_select(logits: np.ndarray, z: np.ndarray) -> np.ndarray:
    """The policy's action on raw ``[B, A, N]`` logits: the first arg-max of sum_k softmax(logits)_ak z_k (c51.py:62-63)."""
    return (softmax(logits) * np.asarray(z, np.float64)).sum(2).argmax(1)


def c51_target(logits_online: np.ndarray, logits_next: np.ndarray, z: np.ndarray) -> np.ndarray:
    """``softmax(logits_next[b, a*])`` with a* the online arg-max   (c51.py:113-124)."""
    a = c51_select(logits_online, z)
    return softmax(np.asarray(logits_next)[np.arange(len(a)), a, :])


def project(returns: np.ndarray, next_dist: np.ndarray, z: np.ndarray, v_min: float, v_max: float, delta_z: float) -> np.ndarray:
    """target_j = sum_k clamp(1 - |clamp(returns_k) - z_j| / delta_z, 0, 1) next_dist_k, ``[B, N]``   (c51.py:125-136)."""
    t = np.clip(np.asarray(returns, np.float64), v_min, v_max)
    z = np.asarray(z, np.float64)
    w = np.clip(1.0 - np.abs(t[:, None, :] - z[None, :, None]) / delta_z, 0.0, 1.0)       # [B, j, k]
    return (w * np.asarray(next_dist, np.float64)[:, None, :]).sum(-1)


def c51_rows(logits: np.ndarray, act: np.ndarray, returns: np.ndarray, z: np.ndarray, v_min: float, v_max: float, delta_z: float,
             next_dist: np.ndarray, weight: np.ndarray | None) -> dict:
    """loss, the per-row cross-entropy, d loss / d logits ``[B, A, N]`` and the priorities ``[B]`` (c51.py:145-160).

    With target from ``project`` and p = softmax(logits[b, act]): CE_b = -sum_j target_j log(p_j + 1e-8), loss =
    mean_b(weight_b CE_b), prio = CE_b.  With g_j = -(weight_b / B) target_j / (p_j + 1e-8), the taken block's gradient is
    p_k (g_k - sum_j p_j g_j) and every other block's 0."""
    logits = np.asarray(logits, np.float64)
    B, A, N = logits.shape
    rows = np.arange(B)
    w = np.ones(B) if weight is None else np.asarray(weight, np.float64).reshape(-1)
    target = project(returns, next_dist, z, v_min, v_max, delta_z)
    p = softmax(logits[rows, act, :])
    ce = -(target * np.log(p + 1e-8)).sum(1)
    g = -(w / B)[:, None] * target / (p + 1e-8)
    dl = np.zeros_like(logits)
    dl[rows, act, :] = p * (g - (p * g).sum(1, keepdims=True))
    return dict(loss=float((w * ce).mean()), ce=ce, dlogits=dl, prio=ce, target=target)


def reference_loss(curr_dist_all: torch.Tensor, act: np.ndarray | torch.Tensor, target_dist: torch.Tensor,
                   weight: torch.Tensor | float) -> tuple[torch.Tensor, torch.Tensor]:
    """(loss, cross_entropy): c51.py:150-154 in torch on the model's probabilities ``[B, A, N]`` (any dtype, any device)."""
    act = torch.as_tensor(act, device=curr_dist_all.device)
    curr_dist = curr_dist_all[torch.arange(len(act), device=curr_dist_all.device), act, :]
    cross_entropy = -(target_dist * torch.log(curr_dist + 1e-8)).sum(1)
    return (cross_entropy * weight).mean(), cross_entropy


def reference_target(next_dist: torch.Tensor, returns: torch.Tensor, z: torch.Tensor, v_min: float, v_max: float,
                     delta_z: float) -> torch.Tensor:
    """c51.py:125-136 in torch, the broadcast written as the reference writes it."""
    target_support = returns.clamp(v_min, v_max)
    target_dist = (1 - (target_support.unsqueeze(1) - z.view(1, -1, 1)).abs() / delta_z).clamp(0, 1) * next_dist.unsqueeze(1)
    return target_dist.sum(-1)


# ------------------------------------------------------------------------------------------------ networks
class CategoricalView(nn.Module):
    """A layer chain whose last Linear has A * N outputs: ``logits`` views it as ``[B, A, N]``, ``forward`` applies the softmax
    over each action's atoms."""

    def __init__(self, chain: nn.Sequential, A: int, N: int):
        super().__init__()
        self.chain, self.A, self.N = chain, A, N

    def logits(self, x: torch.Tensor) -> torch.Tensor:
        return self.chain(x).view(-1, self.A, self.N)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return self.logits(x).softmax(-1)


def categorical_net(kind: str, A: int, N: int, obs: int = 0, hidden: tuple[int, ...] = (), H: int = 0, W: int = 0) -> CategoricalView:
    """``Net(state_shape=obs, action_shape=A, hidden_sizes=hidden, softmax=True, num_atoms=N)`` or ``C51Net(c=4, h=H, w=W,
    action_shape=A, num_atoms=N)`` (common.py:298-369, atari_network.py:125-151)."""
    chain = nature_cnn(4, H, W, A * N) if kind == "cnn" else mlp([obs, *hidden, A * N], False)
    return CategoricalView(chain, A, N)


def net_from_cfg(g) -> CategoricalView:
    if str(g["cfg_kind"]) == "cnn":
        return categorical_net("cnn", int(g["cfg_A"]), int(g["cfg_N"]), H=int(g["cfg_H"]), W=int(g["cfg_W"]))
    return categorical_net("mlp", int(g["cfg_A"]), int(g["cfg_N"]), obs=int(g["cfg_obs"]), hidden=tuple(int(x) for x in g["cfg_hidden"]))


# ------------------------------------------------------------------------------------------------ update
class C51State:
    """The network, its lagged copy (None: ``target_update_freq == 0``), Adam, the iteration counter and the support."""

    def __init__(self, net: CategoricalView, lr: float, freq: int, v_min: float, v_max: float):
        self.net = net
        self.old = copy.deepcopy(net) if freq > 0 else None
        self.opt = torch.optim.Adam(net.parameters(), lr=lr)
        self.freq = freq
        self.iter = 0
        self.v_min, self.v_max = v_min, v_max
        self.z = support(net.N, v_min, v_max)
        self.delta_z = (v_max - v_min) / (net.N - 1)


def _returns(s: C51State, buf: dict, indices: np.ndarray, gamma: float, n_step: int) -> np.ndarray:
    z = torch.from_numpy(s.z)
    return compute_nstep_targets(buf, indices, lambda terminal: z.repeat(len(terminal), 1), gamma, n_step).reshape(-1, s.net.N)


def _tick(s: C51State) -> None:
    if s.old is not None and s.iter % s.freq == 0:
        s.old.load_state_dict(s.net.state_dict())
    s.iter += 1


def c51_update(s: C51State, obs_of: Callable[[np.ndarray], torch.Tensor], buf: dict, indices: np.ndarray, is_weight: np.ndarray | None,
               gamma: float, n_step: int, target_before_tick: bool = False) -> dict:
    """One ``C51.update`` on the sampled ``indices``: the forwards in torch fp32, the rows in float64 numpy, their gradient pushed
    back through the network with autograd.  ``target_before_tick`` forms the target before the lagged refresh (QR-DQN's
    order), which the reference does not do: gen_golden_c51.py uses it to show that its goldens tell the two apart."""
    dev = next(s.net.parameters()).device
    returns = _returns(s, buf, indices, gamma, n_step)

    def next_dist() -> np.ndarray:
        with torch.no_grad():
            x = obs_next_of(obs_of, buf, indices, dev)
            lo = s.net.logits(x)
            ln = s.old.logits(x) if s.old is not None else lo
        return c51_target(lo.cpu().numpy(), ln.cpu().numpy(), s.z)

    nd = next_dist() if target_before_tick else None
    _tick(s)
    if nd is None:
        nd = next_dist()
    logits = s.net.logits(obs_of(indices))
    act = np.asarray(buf["act"])[indices].astype(np.int64).reshape(-1)
    r = c51_rows(logits.detach().cpu().numpy(), act, returns, s.z, s.v_min, s.v_max, s.delta_z, nd, is_weight)
    s.opt.zero_grad()
    logits.backward(torch.as_tensor(r["dlogits"], dtype=torch.float32, device=dev))
    s.opt.step()
    return dict(returns=returns, loss=r["loss"], prio=r["prio"])


def c51_update_torch(s: C51State, obs_of: Callable[[np.ndarray], torch.Tensor], buf: dict, indices: np.ndarray, gamma: float,
                     n_step: int) -> float:
    """The same update as the reference runs it in eager PyTorch: the n-step return on the host (algorithm_base.py:721-817), the
    lagged refresh, the target on the network's device, the loss by ``reference_loss`` and autograd, torch's Adam.  Returns
    the loss."""
    dev = next(s.net.parameters()).device
    z = torch.as_tensor(s.z, device=dev)
    returns = torch.as_tensor(_returns(s, buf, indices, gamma, n_step), device=dev)
    _tick(s)
    with torch.no_grad():
        x = obs_next_of(obs_of, buf, indices, dev)
        dist = s.net(x)
        a = (dist * z).sum(2).argmax(1)
        nd = (s.old(x) if s.old is not None else dist)[torch.arange(len(indices), device=dev), a, :]
        target = reference_target(nd, returns, z, s.v_min, s.v_max, s.delta_z)
    curr = s.net(obs_of(indices))
    act = torch.as_tensor(np.asarray(buf["act"])[indices].astype(np.int64), device=dev)
    loss = reference_loss(curr, act, target, 1.0)[0]
    s.opt.zero_grad()
    loss.backward()
    s.opt.step()
    return loss.item()
