"""TEST INFRASTRUCTURE -- eager-PyTorch restatement of the reference's discrete SAC update (CPU or GPU, autograd).

Only ``tests/`` and ``tools/`` may import this module; ``tianshou_b200`` never does.  It restates
tianshou/algorithm/modelfree/discrete_sac.py:147-196 without the framework around it (no Batch / Policy / Collector), on
top of the n-step, index and NatureCNN helpers of ``oracle_offpolicy``:

  target : discrete_sac.py:147-155 (sum_a pi(a|s') min(Q1', Q2')(s', a) + alpha H), ddpg.py:327-339, algorithm_base.py:721-817
  critics: discrete_sac.py:158-174, actor: :176-184, alpha: sac.py:203-215, Polyak: utils/lagged_network.py:8-18

The reference's policy calls ``dist.sample()`` once in the target and once for the actor loss and discards both draws; this
restatement draws them too (``Categorical.sample``), so the torch generator of the device it runs on advances as the
reference's does.  It is also the eager baseline of tools/discrete_sac_timing.py.

PINNING: tests/test_oracle_discrete_sac.py replays tests/golden/dsac_ref_*.npz (outputs of the imported reference,
oracle/gen_golden_discrete_sac.py) through ``discrete_sac_update``.
"""
from __future__ import annotations

from collections.abc import Callable
from dataclasses import dataclass

import numpy as np
import torch
from torch import nn
from torch.distributions import Categorical

from oracle.oracle_offpolicy import compute_nstep_targets, mlp, nature_cnn, next_index, stacked_obs


def mlp_head_net(obs: int, hidden: tuple[int, ...], out: int, last_hidden: tuple[int, ...] = ()) -> nn.Sequential:
    """``DiscreteActor`` / ``DiscreteCritic`` on ``Net(state_shape=obs, hidden_sizes=hidden)``: trunk, then the ``last`` MLP.
    Same parameter order as the reference module's ``parameters()``."""
    return nn.Sequential(mlp([obs, *hidden], True), mlp([hidden[-1], *last_hidden, out], False))


def cnn_head_net(c: int, h: int, w: int, feat: int, out: int) -> nn.Sequential:
    """The same heads on ``DQNet(c, h, w, features_only=True, output_dim_added_layer=feat)`` (atari_network.py:77-111)."""
    conv = nature_cnn(c, h, w, 1)[0]
    with torch.no_grad():
        n = int(np.prod(conv(torch.zeros(1, c, h, w)).shape[1:]))
    return nn.Sequential(nn.Sequential(conv, nn.Linear(n, feat), nn.ReLU()), nn.Linear(feat, out))


GOLDEN_VIEW_MAX = 2048


def seeded_params(mod: nn.Module, seed: int) -> None:
    """Deterministic initial weights from numpy's PCG64 stream: every tensor in ``parameters()`` order uniform in
    +-1/sqrt(fan_in) (a bias: +-1/sqrt(its length)).  The compact goldens store the seed instead of the initial tensors."""
    rng = np.random.default_rng(seed)
    with torch.no_grad():
        for p in mod.parameters():
            fan_in = int(np.prod(p.shape[1:])) if p.dim() > 1 else p.numel()
            b = 1.0 / np.sqrt(fan_in)
            p.copy_(torch.from_numpy(rng.uniform(-b, b, tuple(p.shape)).astype(np.float32)))


def golden_view(t: np.ndarray | torch.Tensor) -> np.ndarray:
    """The elements of a parameter tensor a compact golden stores: the flat tensor at a fixed stride that keeps at most
    ``GOLDEN_VIEW_MAX`` of them (every element of a smaller tensor)."""
    flat = (t.detach().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)).reshape(-1)
    return flat[::max(1, -(-flat.size // GOLDEN_VIEW_MAX))].copy()


@dataclass
class AutoAlphaState:
    """``AutoAlpha`` (sac.py:168-215): log_alpha, its target entropy and its torch optimiser."""

    log_alpha: nn.Parameter
    target_entropy: float
    optim: torch.optim.Optimizer

    @property
    def value(self) -> float:
        return self.log_alpha.detach().exp().item()

    def update(self, entropy: torch.Tensor) -> float:
        loss = -(self.log_alpha * (self.target_entropy - entropy)).mean()
        self.optim.zero_grad(); loss.backward(); self.optim.step()
        return loss.item()


def flat_obs(rows: np.ndarray, device: torch.device | str) -> Callable[[np.ndarray], torch.Tensor]:
    """Observation reader of a buffer with flat fp32 rows."""
    return lambda idx: torch.as_tensor(rows[idx], dtype=torch.float32, device=device)


def frame_obs(buf: dict, stack: int, denom: float, device: torch.device | str) -> Callable[[np.ndarray], torch.Tensor]:
    """Observation reader of a frame-stacking buffer: uint8 frames stacked through prev(), divided by ``denom`` in float64
    as numpy does (atari_network.py:48-55), then fp32."""
    return lambda idx: torch.as_tensor(stacked_obs(buf["obs"], idx, buf, stack) / denom, dtype=torch.float32, device=device)


def discrete_sac_update(actor: nn.Module, critics: list[nn.Module], critics_old: list[nn.Module], opts: list[torch.optim.Optimizer],
                        obs_of: Callable[[np.ndarray], torch.Tensor], buf: dict, indices: np.ndarray, is_weight: np.ndarray | None,
                        gamma: float, n_step: int, alpha: float | AutoAlphaState, tau: float, obs_next_stored: bool) -> dict:
    """One ``DiscreteSAC.update`` on the sampled ``indices``.  ``opts`` = (actor, critic1, critic2) Adam; ``obs_of(idx)`` reads
    observations at buffer slots; ``obs_next_stored``: the buffer keeps obs_next (``buf["obs_next"]``), else
    obs_next = obs[next(i)].  Returns the n-step returns, the priority-update TD errors, the losses and the alpha results."""
    dev = next(actor.parameters()).device
    alpha_v = alpha if isinstance(alpha, float) else alpha.value

    def target_q(terminal: np.ndarray) -> torch.Tensor:
        if obs_next_stored:
            s = torch.as_tensor(buf["obs_next"][terminal], dtype=torch.float32, device=dev)
        else:
            s = obs_of(next_index(terminal, buf["offset"], buf["done"], buf["last_index"], buf["lengths"]))
        dist = Categorical(logits=actor(s))
        dist.sample()                                       # the policy's discarded draw (discrete_sac.py:74-79)
        q = dist.probs * torch.min(critics_old[0](s), critics_old[1](s))
        return (q.sum(dim=-1) + alpha_v * dist.entropy()).cpu()

    returns = torch.from_numpy(compute_nstep_targets(buf, indices, target_q, gamma, n_step)).flatten().to(dev)
    obs = obs_of(indices)
    act = torch.as_tensor(np.asarray(buf["act"])[indices], dtype=torch.long, device=dev).view(-1, 1)
    weight = 1.0 if is_weight is None else torch.as_tensor(is_weight, dtype=torch.float32, device=dev)
    losses, tds = [], []
    for k in range(2):
        td = critics[k](obs).gather(1, act).flatten() - returns
        loss = (td.pow(2) * weight).mean()
        opts[1 + k].zero_grad(); loss.backward(); opts[1 + k].step()
        losses.append(loss.detach()); tds.append(td.detach())
    dist = Categorical(logits=actor(obs))
    dist.sample()
    entropy = dist.entropy()
    with torch.no_grad():
        q = torch.min(critics[0](obs), critics[1](obs))
    actor_loss = -(alpha_v * entropy + (dist.probs * q).sum(dim=-1)).mean()
    opts[0].zero_grad(); actor_loss.backward(); opts[0].step()
    alpha_loss = None if isinstance(alpha, float) else alpha.update(entropy.detach())
    with torch.no_grad():
        for k in range(2):
            for t, s in zip(critics_old[k].parameters(), critics[k].parameters(), strict=True):
                t.copy_(tau * s + (1 - tau) * t)
    l = torch.stack([actor_loss.detach(), *losses]).cpu().numpy()
    return dict(returns=returns.cpu().numpy(), weight=((tds[0] + tds[1]) / 2.0).cpu().numpy(), losses=l.astype(np.float64),
                alpha=alpha_v if isinstance(alpha, float) else alpha.value, alpha_loss=alpha_loss)
