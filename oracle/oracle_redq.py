"""TEST INFRASTRUCTURE -- eager-PyTorch restatement of the reference's REDQ update (CPU or GPU, autograd).

Only ``tests/`` and ``tools/`` may import this module; ``tianshou_b200`` never does.  It restates
tianshou/algorithm/modelfree/redq.py:254-304 without the framework around it (no Batch / Policy / Collector), on top of the
n-step helper of ``oracle_td3``:

  actor        : utils/net/continuous.py (conditioned sigma, unbounded mu), redq.py:103-131 (rsample, tanh, the log-prob
                 correction)
  ensemble     : utils/net/common.py:518-550 (x @ W_e + b_e per member; the first layer reads the shared [B, in] input)
  target       : redq.py:254-269 ({min | mean} over the drawn subset of the lagged ensemble, minus alpha * log pi)
  critic step  : redq.py:273-279 (mean(td^2 * w) over members and rows, one Adam step; batch.weight = mean_e td)
  actor step   : redq.py:285-293 (mean(alpha * log pi - mean_e Q)), then alpha.update(-log pi)
  Polyak       : utils/lagged_network.py:8-18 on the lagged ensemble, every update

The rsample noise comes from ``noise_fn(shape)``; the subset is given.  It is also the eager baseline of tools/redq_timing.py.

PINNING: tests/test_oracle_redq.py replays tests/golden/redq_ref_*.npz (outputs of the imported reference,
oracle/gen_golden_redq.py) through ``redq_update``.
"""
from __future__ import annotations

import copy
from collections.abc import Callable

import numpy as np
import torch
from torch import nn

from oracle.oracle_offpolicy import mlp
from oracle.oracle_td3 import nstep_targets

SIGMA_MIN, SIGMA_MAX = -20.0, 2.0
_EPS = float(np.finfo(np.float32).eps)


class Ensemble(nn.Module):
    """An EnsembleLinear chain with ReLU between its layers: parameters W_0, b_0, W_1, b_1, ... ([E, in, out], [E, 1, out])."""

    def __init__(self, E: int, dims: list[int]):
        super().__init__()
        self.params = nn.ParameterList()
        for i, o in zip(dims[:-1], dims[1:]):
            k = np.sqrt(1.0 / i)
            self.params.append(nn.Parameter(torch.rand(E, i, o) * 2 * k - k))
            self.params.append(nn.Parameter(torch.rand(E, 1, o) * 2 * k - k))

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        n = len(self.params) // 2
        for j in range(n):
            x = torch.matmul(x, self.params[2 * j]) + self.params[2 * j + 1]
            if j < n - 1:
                x = torch.relu(x)
        return x


class RedqNets:
    """Same parameter order as the reference modules' ``parameters()``: actor = preprocess trunk, mu, sigma; critic = the
    ensemble chain."""

    def __init__(self, obs: int, act: int, hidden: tuple[int, ...], E: int):
        self.trunk = mlp([obs, *hidden], True)
        self.mu = nn.Linear(hidden[-1], act)
        self.sigma = nn.Linear(hidden[-1], act)
        self.actor = nn.ModuleList([self.trunk, self.mu, self.sigma])
        self.critic = Ensemble(E, [obs + act, *hidden, 1])
        self.critic_old = copy.deepcopy(self.critic)
        self.E = E

    def modules(self) -> list[nn.Module]:
        return [self.actor, self.critic, self.critic_old]

    def policy(self, obs: torch.Tensor, noise: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
        """(tanh-squashed action, corrected log pi) of the rsample ``mu + sigma * noise`` (redq.py:109-123)."""
        h = self.trunk(obs)
        loc = self.mu(h)
        scale = torch.clamp(self.sigma(h), min=SIGMA_MIN, max=SIGMA_MAX).exp()
        x = loc + noise * scale
        log_prob = torch.distributions.Independent(torch.distributions.Normal(loc, scale), 1).log_prob(x).unsqueeze(-1)
        act = torch.tanh(x)
        return act, log_prob - torch.log(1 - act.pow(2) + _EPS).sum(-1, keepdim=True)


class FixedAlpha:
    def __init__(self, value: float):
        self.value = value

    def update(self, entropy: torch.Tensor) -> float | None:
        return None


class AutoAlpha:
    """sac.py:168-215: log_alpha with its own Adam."""

    def __init__(self, target_entropy: float, log_alpha: float, lr: float, dtype: torch.dtype = torch.float32):
        self.target_entropy = target_entropy
        self.log_alpha = torch.tensor(log_alpha, dtype=dtype, requires_grad=True)
        self.opt = torch.optim.Adam([self.log_alpha], lr=lr)

    @property
    def value(self) -> float:
        return self.log_alpha.detach().exp().item()

    def update(self, entropy: torch.Tensor) -> float:
        loss = -(self.log_alpha * (self.target_entropy - entropy.to(self.log_alpha.dtype))).mean()
        self.opt.zero_grad(); loss.backward(); self.opt.step()
        return loss.item()


def target_q_values(nets: RedqNets, obs_next: torch.Tensor, noise: torch.Tensor, subset: np.ndarray, target_mode: str,
                    alpha: float) -> torch.Tensor:
    """``_target_q_compute_value`` (redq.py:254-269) at a' ~ pi(.|s') with the given noise and subset."""
    a, logp = nets.policy(obs_next, noise)
    qs = nets.critic_old(torch.cat([obs_next, a], dim=1))[torch.as_tensor(np.asarray(subset, dtype=np.int64))]
    tq = torch.min(qs, dim=0)[0] if target_mode == "min" else torch.mean(qs, dim=0)
    return tq - alpha * logp


def actor_objective(nets: RedqNets, obs: torch.Tensor, noise: torch.Tensor, alpha: float) -> tuple[torch.Tensor, torch.Tensor]:
    """(actor loss, log pi) of redq.py:285-288."""
    a, logp = nets.policy(obs, noise)
    qa = nets.critic(torch.cat([obs, a], dim=1)).mean(dim=0).flatten()
    return (alpha * logp.flatten() - qa).mean(), logp


def redq_update(nets: RedqNets, opts: list[torch.optim.Optimizer], alpha, buf: dict, indices: np.ndarray,
                noise_fn: Callable[[tuple[int, int]], torch.Tensor], subset: np.ndarray, *, gamma: float, n_step: int, tau: float,
                target_mode: str, actor_step: bool, is_weight: torch.Tensor | None = None) -> dict:
    """One ``REDQ.update`` after the index draw on the sampled ``indices``: the n-step target (drawing the rsample noise of
    pi(.|s') from ``noise_fn``), the ensemble step, on ``actor_step`` the actor step (its noise drawn next) and ``alpha.update``,
    and Polyak.  ``opts`` = (actor, critic) Adam; ``alpha``: ``FixedAlpha`` / ``AutoAlpha``.  The networks' dtype sets the
    arithmetic."""
    dtype = nets.mu.weight.dtype
    dev = nets.mu.weight.device
    A = nets.mu.out_features

    def target_q(terminal: np.ndarray) -> torch.Tensor:
        obs_next = torch.as_tensor(buf["obs_next"][terminal], device=dev).to(dtype)
        noise = noise_fn((len(terminal), A)).to(dev, dtype)
        return target_q_values(nets, obs_next, noise, subset, target_mode, float(alpha.value)).cpu()

    returns = torch.from_numpy(nstep_targets(buf, indices, target_q, gamma, n_step)).flatten().to(dev, dtype)
    obs = torch.as_tensor(buf["obs"][indices], device=dev).to(dtype)
    act = torch.as_tensor(buf["act"][indices], device=dev).to(dtype)
    weight = 1.0 if is_weight is None else is_weight.to(dev, dtype)
    td = nets.critic(torch.cat([obs, act], dim=1)).flatten(1) - returns
    critic_loss = (td.pow(2) * weight).mean()
    opts[1].zero_grad(); critic_loss.backward(); opts[1].step()
    out = dict(returns=returns.detach(), critic_loss=float(critic_loss.detach()), weight=td.detach().mean(dim=0),
               actor_loss=None, alpha_loss=None)
    if actor_step:
        noise = noise_fn((len(indices), A)).to(dev, dtype)
        loss, logp = actor_objective(nets, obs, noise, float(alpha.value))
        opts[0].zero_grad(); loss.backward(); opts[0].step()
        out["alpha_loss"] = alpha.update(-logp.detach())
        out["actor_loss"] = float(loss.detach())
    with torch.no_grad():
        for t, s in zip(nets.critic_old.parameters(), nets.critic.parameters(), strict=True):
            t.copy_(tau * s + (1 - tau) * t)
    return out
