"""TEST INFRASTRUCTURE -- eager-PyTorch restatement of the reference's BDQN update (CPU or GPU, autograd).

Only ``tests/`` and ``tools/`` may import this module; ``tianshou_b200`` never does.  It restates
tianshou/algorithm/modelfree/bdqn.py:126-224 without the framework around it (no Batch / Policy / Collector):

  network : utils/net/common.py:661-674 (value + (scores - scores.mean(2)) of a BranchingNet-shaped module: ``common``,
            ``value``, ``branches``)
  target  : bdqn.py:126-175 (always discounted by 0.99: ``_preprocess_batch`` (:177-184) calls ``_compute_return`` without
            the algorithm's ``gamma``, so the keyword's default applies; a*_k the per-branch arg-max of the online network when double, else of the lagged one; the branch
            mean, the reward and (1 - end) in numpy; end = done, and True at every unfinished episode's last slot)
  loss    : bdqn.py:177-196 (the returns repeated over [B, nb, A] and masked to each branch's chosen action; at B = 1 the
            reference's ``.squeeze()`` broadcasts them to [nb, nb, A]); one optimiser step; batch.weight = the signed td sum

It is also the eager baseline of tools/bdqn_timing.py.

PINNING: tests/test_oracle_bdqn.py replays tests/golden/bdqn_ref_*.npz (outputs of the imported reference,
oracle/gen_golden_bdqn.py) through ``bdqn_update``.
"""
from __future__ import annotations

import numpy as np
import torch
from torch import nn

TARGET_GAMMA = 0.99         # the default of ``_compute_return``'s ``gamma``, the only discount the reference's target uses


def q_values(net: nn.Module, obs: torch.Tensor) -> torch.Tensor:
    """[B, nb, A] Q-values of a BranchingNet-shaped module."""
    h = net.common.model(obs)
    v = net.value.model(h).unsqueeze(1)
    s = torch.stack([b.model(h) for b in net.branches], 1)
    return v + (s - s.mean(2, keepdim=True))


def bdqn_targets(net: nn.Module, net_old: nn.Module | None, obs_next: torch.Tensor, rew: np.ndarray, end: np.ndarray, *,
                 gamma: float, is_double: bool) -> torch.Tensor:
    """``_compute_return`` (bdqn.py:144-175): the returns as the loss reads them, [B, nb, A] (or [nb, nb, A] at B = 1)."""
    with torch.no_grad():
        online = q_values(net, obs_next)
        target_q = q_values(net_old, obs_next) if net_old is not None else online
        act = online.argmax(-1, keepdim=True) if is_double else target_q.max(-1).indices.unsqueeze(-1)
        tq = torch.gather(target_q, -1, act).squeeze()
    tq_np = tq.cpu().numpy()
    nb, A = online.shape[1], online.shape[2]
    mean_tq = np.mean(tq_np, -1) if len(tq_np.shape) > 1 else tq_np
    y = rew + gamma * mean_tq * (1 - end)
    y = np.repeat(np.repeat(y[..., None], nb, axis=-1)[..., None], A, axis=-1)
    return torch.as_tensor(y).to(tq.dtype).to(tq.device)


def bdqn_loss(net: nn.Module, obs: torch.Tensor, act: torch.Tensor, returns: torch.Tensor,
              weight: torch.Tensor | float = 1.0) -> tuple[torch.Tensor, torch.Tensor]:
    """(loss, signed td sum per row) of ``_update_with_batch`` (bdqn.py:177-196)."""
    q = q_values(net, obs)
    act_mask = torch.zeros_like(q).scatter_(-1, act.long().unsqueeze(-1), 1)
    td = returns * act_mask - q * act_mask
    loss = (td.pow(2).sum(-1).mean(-1) * weight).mean()
    return loss, td.sum(-1).sum(-1)


def bdqn_update(net: nn.Module, opt: torch.optim.Optimizer, net_old: nn.Module | None, buf: dict, end: np.ndarray,
                indices: np.ndarray, *, is_double: bool, is_weight: np.ndarray | None = None,
                refresh: bool = False) -> dict:
    """One ``BDQN.update`` after the index draw, on the sampled ``indices``: the target, then (``refresh``) the lagged network's
    full copy at the start of ``_update_with_batch``, then the step.  ``buf`` holds the buffer's ``obs`` / ``act`` / ``rew`` /
    ``obs_next`` columns, ``end`` its end flags.  The network's dtype sets the arithmetic."""
    p = next(net.parameters())
    dtype, dev = p.dtype, p.device
    obs_next = torch.as_tensor(buf["obs_next"][indices], device=dev).to(dtype)
    returns = bdqn_targets(net, net_old, obs_next, buf["rew"][indices], end[indices], gamma=TARGET_GAMMA,
                           is_double=is_double)
    if refresh:
        net_old.load_state_dict(net.state_dict())
    obs = torch.as_tensor(buf["obs"][indices], device=dev).to(dtype)
    act = torch.as_tensor(np.asarray(buf["act"][indices], dtype=np.int64), device=dev)
    weight = 1.0 if is_weight is None else torch.as_tensor(is_weight, device=dev).to(dtype)
    loss, td_sum = bdqn_loss(net, obs, act, returns, weight)
    opt.zero_grad(); loss.backward(); opt.step()
    return dict(returns=returns, loss=float(loss.detach()), td_sum=td_sum.detach())
