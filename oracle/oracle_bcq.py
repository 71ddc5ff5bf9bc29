"""TEST INFRASTRUCTURE -- eager-PyTorch restatement of the reference's BCQ update and policy (CPU or GPU, autograd).

Only ``tests/`` and ``tools/`` may import this module; ``tianshou_b200`` never does.  It restates
tianshou/algorithm/imitation/bcq.py:91-116 and :188-263 and utils/net/continuous.py:378-490 without the framework around it (no
Batch / Policy / Collector):

  VAE step           : bcq.py:201-208 (mse(a, recon) + KL / 2, z = mean + std * eps, log_std clamped to [-4, 15])
  target             : bcq.py:211-237 (s' repeated N times, decoded with CPU latents clamped to +-0.5 and NOT perturbed,
                       lmbda * min + (1 - lmbda) * max of the lagged critics, the max over the N samples, one step with done)
  critic steps       : bcq.py:239-245 (plain F.mse_loss, Adam)
  actor step         : bcq.py:247-253 (-mean Q1(s, perturb(s, decode(s))) against the updated critic 1; an MLP preprocess's
                       ``[0]`` is its row 0, which perturbs every row)
  Polyak             : utils/lagged_network.py:8-18 on the lagged perturbation network and both lagged critics
  policy             : bcq.py:100-116 (per observation S decoded, perturbed actions; the first argmax of critic 1)

The VAE's eps comes from ``eps_fn(shape)`` (the reference calls ``torch.randn_like`` on the networks' device); the decode latents
are ``torch.randn`` on torch's CPU generator, as in the reference.  It is also the eager baseline of tools/bcq_timing.py.

PINNING: tests/test_oracle_bcq.py replays tests/golden/bcq_ref_*.npz (outputs of the imported reference, oracle/gen_golden_bcq.py)
through ``bcq_update`` and ``bcq_policy``.
"""
from __future__ import annotations

import copy
from collections.abc import Callable

import numpy as np
import torch
import torch.nn.functional as F
from torch import nn

from oracle.oracle_offpolicy import mlp


class BcqNets:
    """Same parameter order as the reference modules' ``parameters()``: perturbation = preprocess chain; critic = trunk, last;
    VAE = encoder, mean, log_std, decoder."""

    def __init__(self, obs: int, act: int, hidden: tuple[int, ...], vae_hidden: tuple[int, ...], latent: int,
                 max_action: float = 1.0, phi: float = 0.05, per_row: bool = False):
        self.p = nn.Sequential(mlp([obs + act, *hidden], True), nn.Linear(hidden[-1], act))
        self.c = [nn.Sequential(mlp([obs + act, *hidden], True), nn.Linear(hidden[-1], 1)) for _ in range(2)]
        self.enc = mlp([obs + act, *vae_hidden], True)
        self.mean, self.log_std = nn.Linear(vae_hidden[-1], latent), nn.Linear(vae_hidden[-1], latent)
        self.dec = nn.Sequential(mlp([obs + latent, *vae_hidden], True), nn.Linear(vae_hidden[-1], act))
        self.p_old = copy.deepcopy(self.p)
        self.c_old = [copy.deepcopy(c) for c in self.c]
        self.max_action, self.phi, self.per_row, self.latent = max_action, phi, per_row, latent

    def vae_modules(self) -> list[nn.Module]:
        return [self.enc, self.mean, self.log_std, self.dec]

    def vae_parameters(self) -> list[nn.Parameter]:
        return [p for m in self.vae_modules() for p in m.parameters()]

    def modules(self) -> list[nn.Module]:
        return [self.p, *self.c, *self.vae_modules(), self.p_old, *self.c_old]

    def decode(self, s: torch.Tensor, z: torch.Tensor | None = None) -> torch.Tensor:
        if z is None:
            z = torch.randn(s.shape[:-1] + (self.latent,)).to(s.device, s.dtype).clamp(-0.5, 0.5)
        return self.max_action * torch.tanh(self.dec(torch.cat([s, z], -1)))

    def perturb(self, s: torch.Tensor, a: torch.Tensor, old: bool = False) -> torch.Tensor:
        logits = (self.p_old if old else self.p)(torch.cat([s, a], -1))
        if not self.per_row:
            logits = logits[0]
        noise = self.phi * self.max_action * torch.tanh(logits)
        return (noise + a).clamp(-self.max_action, self.max_action)


def vae_objective(nets: BcqNets, obs: torch.Tensor, act: torch.Tensor, eps: torch.Tensor) -> torch.Tensor:
    """``mse(a, recon) + KL / 2`` (bcq.py:202-206) with the given standard-normal ``eps``."""
    h = nets.enc(torch.cat([obs, act], -1))
    mean, std = nets.mean(h), torch.exp(nets.log_std(h).clamp(-4, 15))
    recon = nets.decode(obs, mean + std * eps)
    kl = (-torch.log(std) + (std.pow(2) + mean.pow(2) - 1) / 2).mean()
    return F.mse_loss(act, recon) + kl / 2


def bcq_update(nets: BcqNets, opts: list[torch.optim.Optimizer], batch: dict[str, torch.Tensor],
               eps_fn: Callable[[tuple[int, ...]], torch.Tensor], *, gamma: float, tau: float, lmbda: float, N: int) -> dict:
    """One ``BCQ._update_with_batch`` on ``batch`` (obs, act, obs_next, rew, done as tensors of the networks' dtype / device;
    done bool).  ``opts`` = (perturbation, critic 1, critic 2, vae) Adam.  Returns the four losses and the target."""
    obs, act = batch["obs"], batch["act"]
    B = obs.shape[0]
    eps = eps_fn((B, nets.latent)).to(obs.device, obs.dtype)
    vae_loss = vae_objective(nets, obs, act, eps)
    opts[3].zero_grad(); vae_loss.backward(); opts[3].step()
    with torch.no_grad():
        obs_next = batch["obs_next"].repeat_interleave(N, dim=0)
        act_next = nets.decode(obs_next)
        x = torch.cat([obs_next, act_next], -1)
        q1, q2 = nets.c_old[0](x), nets.c_old[1](x)
        q = lmbda * torch.min(q1, q2) + (1 - lmbda) * torch.max(q1, q2)
        q = q.reshape(B, -1).max(dim=1)[0].reshape(-1, 1)
        target = batch["rew"].reshape(-1, 1) + torch.logical_not(batch["done"]).reshape(-1, 1) * gamma * q
    losses = []
    for k in range(2):
        loss = F.mse_loss(nets.c[k](torch.cat([obs, act], -1)), target)
        opts[1 + k].zero_grad(); loss.backward(); opts[1 + k].step()
        losses.append(float(loss.detach()))
    perturbed = nets.perturb(obs, nets.decode(obs))
    actor_loss = -nets.c[0](torch.cat([obs, perturbed], -1)).mean()
    opts[0].zero_grad(); actor_loss.backward(); opts[0].step()
    with torch.no_grad():
        for tgt, src in ((nets.p_old, nets.p), (nets.c_old[0], nets.c[0]), (nets.c_old[1], nets.c[1])):
            for t, s in zip(tgt.parameters(), src.parameters(), strict=True):
                t.copy_(tau * s + (1 - tau) * t)
    return dict(actor_loss=float(actor_loss.detach()), critic1_loss=losses[0], critic2_loss=losses[1],
                vae_loss=float(vae_loss.detach()), target=target.detach())


def bcq_policy(nets: BcqNets, obs: torch.Tensor, S: int) -> np.ndarray:
    """``BCQPolicy.forward`` (bcq.py:100-116): the reference's loop over the observations."""
    out = []
    with torch.no_grad():
        for o in obs:
            s = o.reshape(1, -1).repeat(S, 1)
            a = nets.perturb(s, nets.decode(s))
            q = nets.c[0](torch.cat([s, a], -1))
            out.append(a[q.argmax(0)].cpu().numpy().flatten())
    return np.array(out)
