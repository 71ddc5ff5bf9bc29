"""TEST INFRASTRUCTURE -- eager-PyTorch restatement of the NPG / TRPO update loop (the reference's npg.py:140-224 and
trpo.py:131-200 semantics, written independently): autograd double backward for the Fisher-vector products, a plain
conjugate gradient, the natural step or the backtracking line search, and the critic's Adam steps.

Pinned to the reference's goldens by tests/test_oracle_npg.py (CPU); tools/npg_trpo_timing.py runs it on the GPU as the
eager-PyTorch context of the CUDA path.  Never imported by the product package.
"""
from __future__ import annotations

import math

import torch
from torch import nn
from torch.distributions import Categorical, Independent, Normal, kl_divergence


class Actor(nn.Module):
    """Linear / activation trunk + linear head; Gaussian heads own a state-independent log-std registered first (the
    parameter order of ContinuousActorProbabilistic)."""

    def __init__(self, obs: int, act: int, hidden: tuple[int, ...], activation: type[nn.Module], categorical: bool) -> None:
        super().__init__()
        if not categorical:
            self.sigma_param = nn.Parameter(torch.zeros(act, 1))
        self.categorical = categorical
        dims = (obs, *hidden)
        self.trunk = nn.Sequential(*[m for i in range(len(hidden)) for m in (nn.Linear(dims[i], dims[i + 1]), activation())])
        self.head = nn.Linear(dims[-1], act)

    def dist(self, obs: torch.Tensor) -> torch.distributions.Distribution:
        out = self.head(self.trunk(obs))
        if self.categorical:
            return Categorical(probs=torch.softmax(out, -1))
        return Independent(Normal(out, self.sigma_param.reshape(-1).exp().expand_as(out)), 1)


def critic_net(obs: int, hidden: tuple[int, ...], activation: type[nn.Module]) -> nn.Sequential:
    dims = (obs, *hidden)
    return nn.Sequential(*[m for i in range(len(hidden)) for m in (nn.Linear(dims[i], dims[i + 1]), activation())],
                         nn.Linear(dims[-1], 1))


def _flat(ts) -> torch.Tensor:
    return torch.cat([t.reshape(-1) for t in ts])


def _load_flat(params: list[nn.Parameter], flat: torch.Tensor) -> None:
    off = 0
    for p in params:
        p.data.copy_(flat[off:off + p.numel()].view_as(p))
        off += p.numel()


def bounds(n: int, size: int) -> list[tuple[int, int]]:
    """Batch.split(size, merge_last=True) cut points."""
    out = []
    for lo in range(0, n, size):
        if n % size and lo + 2 * size >= n:
            out.append((lo, n))
            break
        out.append((lo, min(lo + size, n)))
    return out


def update(actor: Actor, critic: nn.Module, critic_opt: torch.optim.Optimizer, data: dict, perms, batch_size: int | None, *,
           trpo: bool, optim_critic_iters: int, trust_region_size: float = 0.5, max_kl: float = 0.01, backtrack_coeff: float = 0.8,
           max_backtracks: int = 10, damping: float = 0.1, cg_steps: int = 10, residual_tol: float = 1e-10) -> dict:
    """One ``_update_with_batch`` on preprocessed rows ``data`` (obs, act, adv, returns, logp_old tensors) in the minibatch
    orders ``perms``.  Returns per-minibatch actor_loss / vf_loss / kl / step_size / cg_iters and the warning messages."""
    params = list(actor.parameters())
    n = data["obs"].shape[0]
    res: dict = {"actor_loss": [], "vf_loss": [], "kl": [], "step_size": [], "cg_iters": [], "warnings": []}
    for perm in perms:
        for lo, hi in bounds(n, batch_size or n):
            idx = torch.as_tensor(perm[lo:hi])
            obs, act, adv, ret, lpo = (data[k][idx] for k in ("obs", "act", "adv", "returns", "logp_old"))

            def surrogate(dist: torch.distributions.Distribution) -> torch.Tensor:
                lp = dist.log_prob(act)
                return -(((lp - lpo).exp() if trpo else lp) * adv).mean()

            dist = actor.dist(obs)
            loss = surrogate(dist)
            grad = _flat(torch.autograd.grad(loss, params, retain_graph=True)).detach()
            with torch.no_grad():
                old = actor.dist(obs)
            kl_grad = _flat(torch.autograd.grad(kl_divergence(old, dist).mean(), params, create_graph=True))

            def fisher(v: torch.Tensor) -> torch.Tensor:
                return _flat(torch.autograd.grad((kl_grad * v).sum(), params, retain_graph=True)).detach() + damping * v

            # conjugate gradient on fisher(x) = grad, x0 = 0
            x, r, p = torch.zeros_like(grad), grad.clone(), grad.clone()
            rr, iters = r.dot(r), 0
            for _ in range(cg_steps):
                z = fisher(p)
                alpha = rr / p.dot(z)
                x, r = x + alpha * p, r - alpha * z
                iters += 1
                rr_new = r.dot(r)
                if rr_new < residual_tol:
                    break
                p, rr = r + rr_new / rr * p, rr_new
            direction = -x
            theta = _flat(p.data for p in params)
            kl_val = 0.0
            step = float(torch.sqrt(2 * max_kl / (direction * fisher(direction)).sum())) if trpo else float("nan")
            with torch.no_grad():
                if not trpo:
                    _load_flat(params, theta + trust_region_size * direction)
                    kl_val = float(kl_divergence(old, actor.dist(obs)).mean())
                else:
                    for i in range(max_backtracks):
                        _load_flat(params, theta + step * direction)
                        new = actor.dist(obs)
                        kl_val = float(kl_divergence(old, new).mean())
                        if kl_val < max_kl and float(surrogate(new)) < float(loss):
                            if i > 0:
                                res["warnings"].append(f"Backtracking to step {i}.")
                            break
                        if i == max_backtracks - 1:
                            _load_flat(params, theta)
                            step = 0.0
                            res["warnings"].append("Line search failed! It seems hyperparamters are poor and need to be changed.")
                        else:
                            step = float(torch.tensor(step, dtype=torch.float32) * backtrack_coeff)
            vf = math.nan
            for _ in range(optim_critic_iters):
                vf_loss = torch.nn.functional.mse_loss(ret, critic(obs).flatten())
                critic_opt.zero_grad()
                vf_loss.backward()
                critic_opt.step()
                vf = float(vf_loss.detach())
            res["actor_loss"].append(float(loss.detach()))
            res["vf_loss"].append(vf)
            res["kl"].append(kl_val)
            res["step_size"].append(step)
            res["cg_iters"].append(iters)
    return res
