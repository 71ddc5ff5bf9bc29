"""TEST INFRASTRUCTURE -- eager-PyTorch restatement of the reference's CQL update (CPU or GPU, autograd).

Only ``tests/`` and ``tools/`` may import this module; ``tianshou_b200`` never does.  It restates
tianshou/algorithm/imitation/cql.py:243-400 without the framework around it (no Batch / Policy / Collector), on top of the
tanh-Gaussian actor / critic modules of ``oracle_offpolicy``:

  calibration returns : cql.py:243-266 + algorithm_base.py:653-719 (Monte-Carlo return of ``sample(0)``, stored positionally)
  actor / alpha       : cql.py:208-216, 274-279;  target: :282-292;  blocks: :303-346;  penalty: :348-365
  Lagrange multiplier : cql.py:367-381;  critic steps: :383-388 (clip_grad_norm_ + Adam);  Polyak: utils/lagged_network.py:8-18

The four ``rsample`` draws come from ``noise_fn`` in the reference's order (actor step, target, current-pi, next-pi); the
random actions are drawn where the reference draws them, ``torch.FloatTensor(B * R, A).uniform_(-min_action, max_action)`` on
torch's CPU generator.  It is also the eager baseline of tools/cql_timing.py.

PINNING: tests/test_oracle_cql.py replays tests/golden/cql_ref_*.npz (outputs of the imported reference,
oracle/gen_golden_cql.py) through ``cql_update`` and ``calibration_returns``.
"""
from __future__ import annotations

from collections.abc import Callable

import numpy as np
import torch
from torch import nn

from oracle.oracle_offpolicy import SacNets


def sample_all_order(size: int, insertion_idx: int) -> np.ndarray:
    """``ReplayBuffer.sample_indices(0)`` of a plain buffer (buffer_base.py:519-525): oldest first."""
    return np.concatenate([np.arange(insertion_idx, size), np.arange(insertion_idx)]).astype(np.int64)


def calibration_returns(rew: np.ndarray, terminated: np.ndarray, truncated: np.ndarray, done: np.ndarray, size: int,
                        insertion_idx: int, gamma: float) -> np.ndarray:
    """``CQL.process_buffer`` on a plain ``ReplayBuffer``: the discounted return-to-go of every transition of ``sample(0)``
    (``_gae`` with zero values and lambda 1, segment ends terminated | truncated | the unfinished last slot), element i of the
    sampled order at position i -- not at the slot it belongs to."""
    idx = sample_all_order(size, insertion_idx)
    end = np.logical_or(terminated[idx], truncated[idx])
    last = (insertion_idx - 1) % size
    if not done[last]:
        end[idx == last] = True
    r = np.asarray(rew, dtype=np.float64)[idx]
    out = np.zeros(len(idx))
    g = 0.0
    for i in range(len(idx) - 1, -1, -1):
        g = r[i] + (0.0 if end[i] else gamma) * g
        out[i] = g
    return out


def cql_nets(obs: int, act: int, hidden: tuple[int, ...]) -> SacNets:
    """Actor (trunk, mu, sigma) and two critics with the reference modules' ``parameters()`` order."""
    return SacNets(obs, act, hidden)


def cql_update(nets: SacNets, opts: list[torch.optim.Optimizer], alpha, multiplier: tuple[torch.Tensor, torch.optim.Optimizer] | None,
               batch: dict, noise_fn: Callable[[tuple[int, int]], torch.Tensor], *, gamma: float, tau: float, temperature: float,
               cql_weight: float, num_repeat_actions: int, lagrange_threshold: float, min_action: float, max_action: float,
               alpha_min: float, alpha_max: float, max_grad_norm: float) -> dict:
    """One ``CQL._update_with_batch`` (cql.py:268-400).  ``opts`` = (actor, critic1, critic2) Adam; ``alpha`` a float or an
    ``oracle_discrete_sac.AutoAlphaState``; ``multiplier`` = (cql_log_alpha leaf, its Adam) or None (``with_lagrange=False``);
    ``batch``: fp32 tensors obs, act, rew, done, obs_next and ``calibration_returns`` (None: uncalibrated)."""
    obs, act, rew, done, obs_next = (batch[k] for k in ("obs", "act", "rew", "done", "obs_next"))
    dev = obs.device
    B, A, R = obs.shape[0], act.shape[-1], num_repeat_actions
    a_v = alpha if isinstance(alpha, float) else alpha.value

    def policy(o: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
        return nets.policy(o, noise_fn((o.shape[0], A)).to(dev))

    def q(k: int, o: torch.Tensor, a: torch.Tensor) -> torch.Tensor:
        return nets.c[k](torch.cat([o, a], dim=1))

    act_pred, log_pi = policy(obs)
    actor_loss = (a_v * log_pi - torch.min(q(0, obs, act_pred), q(1, obs, act_pred))).mean()
    opts[0].zero_grad(); actor_loss.backward(); opts[0].step()
    alpha_loss = None if isinstance(alpha, float) else alpha.update(-log_pi.detach())
    a_v = alpha if isinstance(alpha, float) else alpha.value

    with torch.no_grad():
        act_next, new_log_pi = policy(obs_next)
        x = torch.cat([obs_next, act_next], dim=1)
        target_q = torch.min(nets.c_old[0](x), nets.c_old[1](x)) - a_v * new_log_pi
        target_q = (rew + torch.logical_not(done) * gamma * target_q.flatten()).float().to(obs.dtype)   # fp64 runs: widen back
    current_q = [q(k, obs, act).flatten() for k in range(2)]
    losses = [torch.nn.functional.mse_loss(cq, target_q) for cq in current_q]

    random_actions = torch.FloatTensor(B * R, A).uniform_(-min_action, max_action).to(dev, obs.dtype)
    tmp_obs = obs.unsqueeze(1).repeat(1, R, 1).view(B * R, -1)
    tmp_obs_next = obs_next.unsqueeze(1).repeat(1, R, 1).view(B * R, -1)
    blocks: list[list[torch.Tensor]] = [[], []]          # per critic: random, current-pi, next-pi
    a_c, lp_c = policy(tmp_obs)
    a_x, lp_x = policy(tmp_obs_next)
    rand_logp = np.log(0.5 ** A)
    for k in range(2):
        blocks[k] = [q(k, tmp_obs, random_actions) - rand_logp, q(k, tmp_obs, a_c) - lp_c.detach(), q(k, tmp_obs, a_x) - lp_x.detach()]
    cal = batch.get("calibration_returns")
    if cal is not None:
        ret = cal.unsqueeze(1).repeat((1, R)).view(-1, 1)
        blocks = [[torch.max(v, ret) for v in bl] for bl in blocks]
    scaled = []
    for k in range(2):
        cat = torch.cat(blocks[k], 1)
        scaled.append(torch.logsumexp(cat / temperature, dim=1).mean() * cql_weight * temperature - current_q[k].mean() * cql_weight)
    cql_alpha = cql_alpha_loss = None
    if multiplier is not None:
        log_alpha, la_opt = multiplier
        cql_alpha = torch.clamp(log_alpha.exp(), alpha_min, alpha_max)
        scaled = [cql_alpha * (s - lagrange_threshold) for s in scaled]
        la_opt.zero_grad()
        cql_alpha_loss = -(scaled[0] + scaled[1]) * 0.5
        cql_alpha_loss.backward(retain_graph=True)
        la_opt.step()
    losses = [losses[k] + scaled[k] for k in range(2)]
    for k in range(2):
        opts[1 + k].zero_grad()
        losses[k].backward(retain_graph=k == 0)
        nn.utils.clip_grad_norm_(nets.c[k].parameters(), max_norm=max_grad_norm)
        opts[1 + k].step()
    with torch.no_grad():
        for k in range(2):
            for t, s in zip(nets.c_old[k].parameters(), nets.c[k].parameters(), strict=True):
                t.copy_(tau * s + (1 - tau) * t)
    f = lambda t: None if t is None else float(t.detach().reshape(-1)[0])
    return dict(actor_loss=f(actor_loss), critic1_loss=f(losses[0]), critic2_loss=f(losses[1]),
                alpha=a_v, alpha_loss=alpha_loss, cql_alpha=f(cql_alpha), cql_alpha_loss=f(cql_alpha_loss), target=target_q.detach())
