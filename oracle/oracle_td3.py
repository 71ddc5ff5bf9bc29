"""TEST INFRASTRUCTURE -- eager-PyTorch restatement of the reference's TD3 and TD3+BC updates (CPU or GPU, autograd).

Only ``tests/`` and ``tools/`` may import this module; ``tianshou_b200`` never does.  It restates
tianshou/algorithm/modelfree/td3.py:190-226 and imitation/td3_bc.py:102-127 without the framework around it (no Batch / Policy /
Collector), on top of the n-step helpers of ``oracle_offpolicy``:

  actor              : utils/net/continuous.py:84 (max_action * tanh(last(preprocess(s))))
  target             : td3.py:94-102 (min of the lagged critics), :190-202 (smoothing noise), ddpg.py:327-339 + the n-step return
  critic steps       : ddpg.py:267-285 (weighted MSE, Adam);  batch.weight = (td1 + td2) / 2 (td3.py:212)
  actor step         : td3.py:214-219 (-mean Q1(s, pi(s))) or td3_bc.py:113-120 (lmbda = alpha / mean|Q|, + F.mse_loss)
  Polyak             : utils/lagged_network.py:8-18 on the lagged critics AND the lagged actor, on actor steps only

The target noise comes from ``noise_fn(shape)`` (the reference calls ``torch.randn``).  It is also the eager baseline of
tools/td3_timing.py.

PINNING: tests/test_oracle_td3.py replays tests/golden/td3_ref_*.npz (outputs of the imported reference,
oracle/gen_golden_td3.py) through ``td3_update``.
"""
from __future__ import annotations

import copy
from collections.abc import Callable

import numpy as np
import torch
import torch.nn.functional as F
from torch import nn

from oracle.oracle_offpolicy import mlp, next_index, nstep_return


def nstep_targets(buf: dict, indices: np.ndarray, target_q_fn: Callable[[np.ndarray], torch.Tensor], gamma: float,
                  n_step: int) -> np.ndarray:
    """``Algorithm.compute_nstep_return`` (algorithm_base.py:721-817) on one plain buffer.  ``buf``: rew, done, terminated, offset,
    last_index, lengths (what ``ReplayBuffer.next`` reads) and ``unfinished`` (``ReplayBuffer.unfinished_index()``).  The two
    differ on a ``from_data`` buffer: its ``last_index`` stays [0] while the unfinished slot is the one before the insertion
    index."""
    chain = [indices]
    for _ in range(n_step - 1):
        chain.append(next_index(chain[-1], buf["offset"], buf["done"], buf["last_index"], buf["lengths"]))
    chain = np.stack(chain)
    terminal = chain[-1]
    with torch.no_grad():
        tq = target_q_fn(terminal)
    tq = tq.numpy().reshape(len(indices), -1) * (~buf["terminated"][terminal]).reshape(-1, 1)
    end_flag = buf["done"].copy()
    end_flag[np.asarray(buf["unfinished"], dtype=np.int64)] = True
    return nstep_return(buf["rew"], end_flag, tq, chain, gamma, n_step).astype(np.float32)


class Td3Nets:
    """Same parameter order as the reference modules' ``parameters()``: actor = preprocess trunk, last; critic = trunk, last."""

    def __init__(self, obs: int, act: int, hidden: tuple[int, ...], max_action: float = 1.0):
        self.a = nn.Sequential(mlp([obs, *hidden], True), nn.Linear(hidden[-1], act))
        self.c = [nn.Sequential(mlp([obs + act, *hidden], True), nn.Linear(hidden[-1], 1)) for _ in range(2)]
        self.a_old = copy.deepcopy(self.a)
        self.c_old = [copy.deepcopy(c) for c in self.c]
        self.max_action = max_action

    def modules(self) -> list[nn.Module]:
        return [self.a, *self.c, self.a_old, *self.c_old]

    def pi(self, obs: torch.Tensor, old: bool = False) -> torch.Tensor:
        return self.max_action * torch.tanh((self.a_old if old else self.a)(obs))


def actor_objective(nets: Td3Nets, obs: torch.Tensor, act: torch.Tensor, bc_alpha: float | None = None) -> torch.Tensor:
    """TD3's actor loss ``-mean(Q1(s, pi(s)))`` (td3.py:216) or, with ``bc_alpha``, TD3+BC's
    ``-lmbda * mean(q) + F.mse_loss(pi(s), a)`` with ``lmbda = alpha / mean|q|`` detached (td3_bc.py:114-117)."""
    pi = nets.pi(obs)
    q = nets.c[0](torch.cat([obs, pi], dim=1))
    if bc_alpha is None:
        return -q.mean()
    lmbda = bc_alpha / q.abs().mean().detach()
    return -lmbda * q.mean() + F.mse_loss(pi, act)


def td3_update(nets: Td3Nets, opts: list[torch.optim.Optimizer], buf: dict, indices: np.ndarray,
               noise_fn: Callable[[tuple[int, int]], torch.Tensor], *, gamma: float, n_step: int, tau: float, policy_noise: float,
               noise_clip: float, actor_step: bool, is_weight: torch.Tensor | None = None, bc_alpha: float | None = None) -> dict:
    """One ``TD3._update_with_batch`` (or ``TD3BC``'s with ``bc_alpha``) after the n-step target on the sampled ``indices``.
    ``opts`` = (actor, critic1, critic2) Adam; ``buf``: the whole-buffer arrays ``nstep_targets`` reads plus obs, act,
    obs_next; ``actor_step``: ``_cnt % update_actor_freq == 0``.  The networks' dtype sets the arithmetic."""
    dtype = nets.a[-1].weight.dtype
    dev = nets.a[-1].weight.device

    def target_q(terminal: np.ndarray) -> torch.Tensor:
        obs_next = torch.as_tensor(buf["obs_next"][terminal], device=dev).to(dtype)
        a = nets.pi(obs_next, old=True)
        noise = noise_fn(tuple(a.shape)).to(dev, dtype) * policy_noise
        if noise_clip > 0.0:
            noise = noise.clamp(-noise_clip, noise_clip)
        a = a + noise
        x = torch.cat([obs_next, a], dim=1)
        return torch.min(nets.c_old[0](x), nets.c_old[1](x)).cpu()

    returns = torch.from_numpy(nstep_targets(buf, indices, target_q, gamma, n_step)).flatten().to(dev, dtype)
    obs = torch.as_tensor(buf["obs"][indices], device=dev).to(dtype)
    act = torch.as_tensor(buf["act"][indices], device=dev).to(dtype)
    weight = 1.0 if is_weight is None else is_weight.to(dev, dtype)
    losses, tds = [], []
    for k in range(2):
        td = nets.c[k](torch.cat([obs, act], dim=1)).flatten() - returns
        loss = (td.pow(2) * weight).mean()
        opts[1 + k].zero_grad(); loss.backward(); opts[1 + k].step()
        losses.append(float(loss.detach())); tds.append(td.detach())
    actor_loss = None
    if actor_step:
        loss = actor_objective(nets, obs, act, bc_alpha)
        opts[0].zero_grad(); loss.backward(); opts[0].step()
        actor_loss = float(loss.detach())
        with torch.no_grad():
            for tgt, src in ((nets.c_old[0], nets.c[0]), (nets.c_old[1], nets.c[1]), (nets.a_old, nets.a)):
                for t, s in zip(tgt.parameters(), src.parameters(), strict=True):
                    t.copy_(tau * s + (1 - tau) * t)
    return dict(returns=returns.detach(), actor_loss=actor_loss, critic1_loss=losses[0], critic2_loss=losses[1],
                weight=((tds[0] + tds[1]) / 2.0))
