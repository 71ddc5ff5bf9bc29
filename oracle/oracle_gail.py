"""TEST INFRASTRUCTURE -- eager-PyTorch restatement of GAIL's discriminator half (the reference's gail.py:193-248 semantics,
written independently): the reward pass over the rollout rows and the discriminator's Adam steps over chunks of one
permutation, each against its own expert rows.

Pinned to the reference's goldens by tests/test_oracle_gail.py (CPU); tools/gail_timing.py runs it on the GPU as the
eager-PyTorch context of the CUDA path.  Never imported by the product package.
"""
from __future__ import annotations

import numpy as np
import torch
from torch import nn


def disc_net(obs: int, act: int, hidden: tuple[int, ...], activation: type[nn.Module]) -> nn.Sequential:
    """Linear / activation chain on concat(obs, act) ending in one linear logit (parameter order of
    ContinuousCritic(preprocess_net=Net(concat=True)))."""
    dims = (obs + act, *hidden)
    return nn.Sequential(*[m for i in range(len(hidden)) for m in (nn.Linear(dims[i], dims[i + 1]), activation())],
                         nn.Linear(dims[-1], 1))


def step_bounds(n: int, disc_update_num: int) -> list[tuple[int, int]]:
    """Row ranges of the discriminator steps: chunks of n // disc_update_num, a short remainder merged into the last one."""
    size = n // disc_update_num
    assert size >= 1, f"{n} rows cannot make {disc_update_num} chunks"
    starts = list(range(0, n, size))
    if n % size and len(starts) > 1:
        starts.pop()
    return [(lo, starts[i + 1] if i + 1 < len(starts) else n) for i, lo in enumerate(starts)]


def _neg_logsigmoid(x: torch.Tensor) -> torch.Tensor:
    return -torch.nn.functional.logsigmoid(x)


def rewards(disc: nn.Module, obs: torch.Tensor, act: torch.Tensor) -> torch.Tensor:
    """Per-row reward -log(1 - sigmoid(D(s, a))) = -logsigmoid(-D), evaluated in the discriminator's dtype."""
    with torch.no_grad():
        return _neg_logsigmoid(-disc(torch.cat([obs, act], 1))).reshape(-1)


def disc_update(disc: nn.Module, opt: torch.optim.Optimizer, obs: torch.Tensor, act: torch.Tensor, order: np.ndarray,
                exp_obs: torch.Tensor, exp_act: torch.Tensor, disc_update_num: int) -> dict[str, list[float]]:
    """One Adam step per chunk of ``order``; step s uses expert rows [s * size, (s + 1) * size) of exp_obs / exp_act."""
    n = obs.shape[0]
    size = n // disc_update_num
    res: dict[str, list[float]] = {"loss": [], "acc_pi": [], "acc_exp": [], "margin_pi": [], "margin_exp": []}
    for s, (lo, hi) in enumerate(step_bounds(n, disc_update_num)):
        idx = torch.as_tensor(order[lo:hi])
        pi = disc(torch.cat([obs[idx], act[idx]], 1)).reshape(-1)
        ex = disc(torch.cat([exp_obs[s * size:(s + 1) * size], exp_act[s * size:(s + 1) * size]], 1)).reshape(-1)
        # policy rows are pushed towards D < 0, expert rows towards D > 0
        loss = _neg_logsigmoid(-pi).mean() + _neg_logsigmoid(ex).mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
        res["loss"].append(float(loss.detach()))
        res["acc_pi"].append(float((pi < 0).float().mean()))
        res["acc_exp"].append(float((ex > 0).float().mean()))
        res["margin_pi"].append(float(pi.detach().abs().min()))
        res["margin_exp"].append(float(ex.detach().abs().min()))
    return res
