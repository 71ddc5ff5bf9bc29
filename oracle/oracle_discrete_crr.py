"""TEST INFRASTRUCTURE -- float64 numpy restatement of discrete CRR's target, losses and loss gradients, and its update on
plain torch networks (the two-head layout of ``oracle_discrete_bcq.TwoHeadNets``: head a = actor, head b = critic).

Only ``tests/`` and ``tools/`` may import this module; ``tianshou_b200`` never does.  It restates
tianshou/algorithm/imitation/discrete_crr.py:125-167 without the framework around it.  The gradients are written out by hand
and are the reference's AUTOGRAD gradients: the advantage is not detached, so in ``"exp"`` mode the coefficient carries
gradient into q and the logits wherever the clamp passes; and ``-log_prob`` ``[B]`` times the coefficient ``[B, 1]`` broadcasts to
``[B, B]``, so the actor loss is the product of the two means.

PINNING: tests/test_oracle_discrete_crr.py replays tests/golden/dcrr_ref_*.npz (outputs of the imported reference,
oracle/gen_golden_discrete_crr.py) through ``discrete_crr_update``.
"""
from __future__ import annotations

import copy
from collections.abc import Callable

import numpy as np
import torch

from oracle.oracle_discrete_bcq import TwoHeadNets, log_softmax, obs_next_of


def crr_rows(q: np.ndarray, logits: np.ndarray, act: np.ndarray, q_old: np.ndarray, logits_old: np.ndarray, rew: np.ndarray,
             done: np.ndarray, gamma: float, mode: str, beta: float, bound: float, min_q_weight: float) -> dict:
    """(loss, actor_loss, critic_loss, cql_loss), the one-step target, the advantage and d loss / d q, d loss / d logits."""
    q, z = np.asarray(q, np.float64), np.asarray(logits, np.float64)
    B, A = q.shape
    rows = np.arange(B)
    eq = (np.exp(log_softmax(logits_old)) * np.asarray(q_old, np.float64)).sum(-1)
    eq[np.asarray(done).reshape(-1) > 0] = 0.0
    target = np.asarray(rew, np.float64).reshape(-1) + gamma * eq
    qa = q[rows, act]
    err = qa - target
    lp = log_softmax(z)
    p = np.exp(lp)
    S = (p * q).sum(-1)
    adv = qa - S
    g = np.zeros(B)
    if mode == "binary":
        coef = (adv > 0).astype(np.float64)
    elif mode == "exp":
        with np.errstate(over="ignore"):
            e = np.exp(adv / beta)
        coef = np.clip(e, 0.0, bound)
        passes = (e >= 0.0) & (e <= bound)
        g[passes] = (e / beta)[passes]
    else:
        coef = np.ones(B)
    lpq = log_softmax(q)
    # -log_prob [B] times the coefficient [B, 1] broadcasts to [B, B] (discrete_crr.py:155): the mean of the outer product
    nbar, cbar = (-lp[rows, act]).mean(), coef.mean()
    g *= nbar
    actor, critic, cql = nbar * cbar, 0.5 * (err * err).mean(), (-lpq[rows, act]).mean()
    hit = np.zeros((B, A))
    hit[rows, act] = 1.0
    dq = (hit * err[:, None] + g[:, None] * (hit - p) + min_q_weight * (np.exp(lpq) - hit)) / B
    dlogits = (cbar * (p - hit) - g[:, None] * p * (q - S[:, None])) / B
    return dict(losses=np.array([actor + critic + min_q_weight * cql, actor, critic, cql]), target=target, adv=adv, coef=coef,
                dq=dq, dlogits=dlogits)


class CrrState:
    """Networks, their lagged copy (``freq == 0``: the online networks themselves), Adam and the iteration counter."""

    def __init__(self, nets: TwoHeadNets, lr: float, freq: int):
        self.nets = nets
        self.freq = freq
        self.old = copy.deepcopy(nets) if freq > 0 else nets
        self.opt = torch.optim.Adam(nets.parameters(), lr=lr)
        self.iter = 0


def discrete_crr_update(s: CrrState, obs_of: Callable[[np.ndarray], torch.Tensor], buf: dict, indices: np.ndarray, gamma: float,
                        mode: str, beta: float, bound: float, min_q_weight: float) -> dict:
    """One ``DiscreteCRR.update`` on the sampled ``indices``: the lagged copy when ``iter % freq == 0``, the step, then
    ``iter`` advances (discrete_crr.py:129-160)."""
    dev = next(s.nets.parameters()).device
    if s.freq > 0 and s.iter % s.freq == 0:
        s.old.load_state_dict(s.nets.state_dict())
    z, q = s.nets.both(obs_of(indices))
    with torch.no_grad():
        zo, qo = s.old.both(obs_next_of(obs_of, buf, indices, dev))
    act = np.asarray(buf["act"])[indices].astype(np.int64).reshape(-1)
    r = crr_rows(q.detach().cpu().numpy(), z.detach().cpu().numpy(), act, qo.cpu().numpy(), zo.cpu().numpy(),
                 np.asarray(buf["rew"])[indices].astype(np.float32), np.asarray(buf["done"])[indices], gamma, mode, beta, bound,
                 min_q_weight)
    s.opt.zero_grad()
    torch.autograd.backward([q, z], [torch.as_tensor(r["dq"], dtype=torch.float32, device=dev),
                                     torch.as_tensor(r["dlogits"], dtype=torch.float32, device=dev)])
    s.opt.step()
    s.iter += 1
    return r
