"""TEST INFRASTRUCTURE -- float64 numpy restatement of discrete BCQ's target, losses and loss gradients, and its update on
plain torch networks.

Only ``tests/`` and ``tools/`` may import this module; ``tianshou_b200`` never does.  It restates
tianshou/algorithm/imitation/discrete_bcq.py without the framework around it (no Batch / Policy / Collector):

  target : discrete_bcq.py:115-118 (the imitator's mask on the arg-max), :228-234, algorithm_base.py:721-817 (n-step)
  loss   : discrete_bcq.py:244-252 (smooth-L1 + NLL + logit penalty), the gradients written out by hand
  lagged : discrete_bcq.py:240-242 (full copy when ``_iter % freq == 0``, BEFORE the step)

``TwoHeadNets`` is the two-heads-on-one-trunk layout every reference use of discrete BCQ / CRR builds, in the reference's
parameter order; it is also the eager baseline of tools/discrete_offline_timing.py.

PINNING: tests/test_oracle_discrete_bcq.py replays tests/golden/dbcq_ref_*.npz (outputs of the imported reference,
oracle/gen_golden_discrete_bcq.py) through ``discrete_bcq_update``.
"""
from __future__ import annotations

import copy
from collections.abc import Callable

import numpy as np
import torch
from torch import nn

from oracle.oracle_offpolicy import compute_nstep_targets, mlp, nature_cnn, next_index

FLT_MAX = np.float32(np.finfo(np.float32).max)


# ------------------------------------------------------------------------------------------------ rows, float64
def log_softmax(z: np.ndarray) -> np.ndarray:
    z = np.asarray(z, np.float64)
    m = z.max(-1, keepdims=True)
    return z - (m + np.log(np.exp(z - m).sum(-1, keepdims=True)))


def bcq_select(q: np.ndarray, logits: np.ndarray, log_tau: float) -> np.ndarray:
    """DiscreteBCQPolicy's action (discrete_bcq.py:115-118).  The masked values are formed in float32, as torch forms them
    (``q - finfo.max * mask``), so ties among them fall as they do there; the first maximum wins."""
    q, logits = np.asarray(q, np.float32), np.asarray(logits, np.float32)
    mask = ((logits - logits.max(-1, keepdims=True)) < np.float32(log_tau)).astype(np.float32)
    return (q - FLT_MAX * mask).argmax(-1)


def bcq_target(q_online: np.ndarray, logits: np.ndarray, q_old: np.ndarray, log_tau: float) -> np.ndarray:
    """Q_old(s', argmax over the kept actions of Q(s', .))   (discrete_bcq.py:228-234)."""
    a = bcq_select(q_online, logits, log_tau)
    return np.asarray(q_old)[np.arange(len(a)), a]


def bcq_rows(q: np.ndarray, logits: np.ndarray, act: np.ndarray, returns: np.ndarray, penalty: float) -> dict:
    """(loss, q_loss, i_loss, reg_loss) and d loss / d q, d loss / d logits   (discrete_bcq.py:244-252)."""
    q, z, ret = np.asarray(q, np.float64), np.asarray(logits, np.float64), np.asarray(returns, np.float64).reshape(-1)
    B, A = q.shape
    rows = np.arange(B)
    td = q[rows, act] - ret
    small = np.abs(td) < 1.0
    q_loss = np.where(small, 0.5 * td * td, np.abs(td) - 0.5).mean()
    lp = log_softmax(z)
    i_loss = -lp[rows, act].mean()
    reg = (z * z).mean()
    hit = np.zeros((B, A))
    hit[rows, act] = 1.0
    dq = hit * (np.where(small, td, np.sign(td)) / B)[:, None]
    dlogits = (np.exp(lp) - hit) / B + 2.0 * penalty * z / (B * A)
    return dict(losses=np.array([q_loss + i_loss + penalty * reg, q_loss, i_loss, reg]), dq=dq, dlogits=dlogits)


# ------------------------------------------------------------------------------------------------ networks
class TwoHeadNets(nn.Module):
    """Heads ``a`` and ``b`` (trunk + ``last`` MLP each).  ``parameters()`` gives trunk a, last a, (trunk b,) last b: the order of
    the reference's ``policy.parameters()`` (BCQ: model, imitator) and ``ModuleList([policy, critic]).parameters()`` (CRR)."""

    def __init__(self, trunk: Callable[[], nn.Module], feat: int, last_hidden: tuple[int, ...], outs: tuple[int, int], shared: bool):
        super().__init__()
        self.trunk_a = trunk()
        self.last_a = mlp([feat, *last_hidden, outs[0]], False)
        self.trunk_b = self.trunk_a if shared else trunk()
        self.last_b = mlp([feat, *last_hidden, outs[1]], False)
        self.shared = shared

    def a(self, x: torch.Tensor) -> torch.Tensor:
        return self.last_a(self.trunk_a(x))

    def b(self, x: torch.Tensor) -> torch.Tensor:
        return self.last_b(self.trunk_b(x))

    def both(self, x: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
        if self.shared:
            h = self.trunk_a(x)
            return self.last_a(h), self.last_b(h)
        return self.a(x), self.b(x)

    def head_a_parameters(self) -> list[nn.Parameter]:
        return [*self.trunk_a.parameters(), *self.last_a.parameters()]

    def head_b_parameters(self) -> list[nn.Parameter]:
        return [*self.trunk_b.parameters(), *self.last_b.parameters()]


def mlp_trunk(obs: int, hidden: tuple[int, ...], out: int = 0) -> tuple[Callable[[], nn.Module], int]:
    """``Net(state_shape=obs, hidden_sizes=hidden)`` (ReLU after every layer) or, with ``out``,
    ``Net(state_shape=obs, action_shape=out, hidden_sizes=hidden)`` (a last Linear without activation)."""
    if out:
        return (lambda: mlp([obs, *hidden, out], False)), out
    return (lambda: mlp([obs, *hidden], True)), hidden[-1]


def cnn_trunk(c: int, h: int, w: int) -> tuple[Callable[[], nn.Module], int]:
    """``DQNet(c, h, w, features_only=True)``: the three convolutions and the Flatten (atari_network.py:77-111)."""
    with torch.no_grad():
        feat = int(np.prod(nature_cnn(c, h, w, 1)[0](torch.zeros(1, c, h, w)).shape[1:]))
    return (lambda: nature_cnn(c, h, w, 1)[0]), feat


def nets_from_cfg(g, outs: tuple[int, int]) -> TwoHeadNets:
    """The networks a golden file's ``cfg_*`` entries describe."""
    last_hidden = tuple(int(x) for x in g["cfg_last_hidden"])
    if str(g["cfg_kind"]) == "cnn":
        trunk, feat = cnn_trunk(4, int(g["cfg_H"]), int(g["cfg_W"]))
    else:
        trunk, feat = mlp_trunk(int(g["cfg_obs"]), tuple(int(x) for x in g["cfg_hidden"]), int(g["cfg_trunk_out"]))
    return TwoHeadNets(trunk, feat, last_hidden, outs, bool(g["cfg_shared"]))


def obs_next_of(obs_of: Callable[[np.ndarray], torch.Tensor], buf: dict, idx: np.ndarray, device) -> torch.Tensor:
    """``buffer[idx].obs_next``: the stored column, or obs[next(idx)] when it is not stored (buffer_base.py:627-629)."""
    if "obs_next" in buf:
        return torch.as_tensor(buf["obs_next"][idx], dtype=torch.float32, device=device)
    return obs_of(next_index(idx, buf["offset"], buf["done"], buf["last_index"], buf["lengths"]))


# ------------------------------------------------------------------------------------------------ update
class BcqState:
    """Networks, lagged copy of head a (the Q model), Adam and the iteration counter."""

    def __init__(self, nets: TwoHeadNets, lr: float):
        self.nets = nets
        self.old = copy.deepcopy(nets)          # only its head a is read
        self.opt = torch.optim.Adam(nets.parameters(), lr=lr)
        self.iter = 0


def discrete_bcq_update(s: BcqState, obs_of: Callable[[np.ndarray], torch.Tensor], buf: dict, indices: np.ndarray, gamma: float,
                        n_step: int, freq: int, log_tau: float, penalty: float) -> dict:
    """One ``DiscreteBCQ.update`` on the sampled ``indices``: the forwards in torch fp32, the rows in float64 numpy, their
    gradients pushed back through the networks with autograd."""
    dev = next(s.nets.parameters()).device

    def target_q(terminal: np.ndarray) -> torch.Tensor:
        x = obs_next_of(obs_of, buf, terminal, dev)
        q, z = s.nets.both(x)
        return torch.from_numpy(bcq_target(q.cpu().numpy(), z.cpu().numpy(), s.old.a(x).cpu().numpy(), log_tau))

    returns = compute_nstep_targets(buf, indices, target_q, gamma, n_step).reshape(-1)
    if s.iter % freq == 0:
        s.old.load_state_dict(s.nets.state_dict())
    s.iter += 1
    q, z = s.nets.both(obs_of(indices))
    act = np.asarray(buf["act"])[indices].astype(np.int64).reshape(-1)
    r = bcq_rows(q.detach().cpu().numpy(), z.detach().cpu().numpy(), act, returns, penalty)
    s.opt.zero_grad()
    torch.autograd.backward([q, z], [torch.as_tensor(r["dq"], dtype=torch.float32, device=dev),
                                     torch.as_tensor(r["dlogits"], dtype=torch.float32, device=dev)])
    s.opt.step()
    return dict(returns=returns, losses=r["losses"])
