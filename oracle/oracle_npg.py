"""TEST INFRASTRUCTURE -- eager-PyTorch restatement of the NPG / TRPO update loop (the reference's npg.py:140-224 and
trpo.py:131-200 semantics, written independently): autograd double backward for the Fisher-vector products, a plain
conjugate gradient, the natural step or the backtracking line search, and the critic's Adam steps.

Pinned to the reference's goldens by tests/test_oracle_npg.py (CPU); tools/npg_trpo_timing.py runs it on the GPU as the
eager-PyTorch context of the CUDA path.  The per-minibatch pieces (surrogate rows, Fisher-vector product, one CG iteration, the TRPO step size, the critic
loss) are the float64 teacher of tests/test_npg_steps_gpu.py.  Never imported by the product package.
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


def surrogate_rows(dist: torch.distributions.Distribution, act: torch.Tensor, adv: torch.Tensor, lpo: torch.Tensor,
                   trpo: bool) -> torch.Tensor:
    """Per-row surrogate loss: -logp * adv (NPG) or -exp(logp - logp_old) * adv (TRPO); their mean is the actor loss."""
    lp = dist.log_prob(act)
    return -(((lp - lpo).exp() if trpo else lp) * adv)


def fisher_product(actor: Actor, obs: torch.Tensor, v: torch.Tensor) -> torch.Tensor:
    """F v without damping: d/dtheta (dKL/dtheta . v) of KL(old || new).mean() at old = new (npg.py:189-200)."""
    params = list(actor.parameters())
    dist = actor.dist(obs)
    with torch.no_grad():
        old = actor.dist(obs)
    kl_grad = _flat(torch.autograd.grad(kl_divergence(old, dist).mean(), params, create_graph=True))
    return _flat(torch.autograd.grad((kl_grad * v).sum(), params)).detach()


def cg_iteration(x: torch.Tensor, r: torch.Tensor, p: torch.Tensor, rr: torch.Tensor, z: torch.Tensor, damping: float,
                 residual_tol: float) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor, bool]:
    """One conjugate-gradient iteration (npg.py:212-223) with z = F p (damping added here): (x, r, p, r.r, converged)."""
    z = z + damping * p
    alpha = rr / p.dot(z)
    x, r = x + alpha * p, r - alpha * z
    rr_new = r.dot(r)
    if rr_new < residual_tol:
        return x, r, p, rr_new, True
    return x, r, r + rr_new / rr * p, rr_new, False


def step_size(x: torch.Tensor, fx: torch.Tensor, damping: float, max_kl: float) -> torch.Tensor:
    """trpo.py:152-159 for the search direction s = -x: sqrt(2 max_kl / (s . MVP(s))) = sqrt(2 max_kl / (x . (F x + damping x)))."""
    return torch.sqrt(2 * max_kl / (x * (fx + damping * x)).sum())


def critic_loss(critic: nn.Module, obs: torch.Tensor, ret: torch.Tensor) -> torch.Tensor:
    """F.mse_loss(returns, critic(obs)) (npg.py:175-179)."""
    return torch.nn.functional.mse_loss(ret, critic(obs).flatten())


def minibatch(actor: Actor, critic: nn.Module, critic_opt: torch.optim.Optimizer, obs: torch.Tensor, act: torch.Tensor,
              adv: torch.Tensor, ret: torch.Tensor, lpo: torch.Tensor, *, trpo: bool, optim_critic_iters: int,
              trust_region_size: float = 0.5, max_kl: float = 0.01, backtrack_coeff: float = 0.8, max_backtracks: int = 10,
              damping: float = 0.1, cg_steps: int = 10, residual_tol: float = 1e-10) -> dict:
    """One minibatch of npg.py:140-187 / trpo.py:131-200, updating ``actor`` and ``critic`` in place: actor_loss, vf_loss,
    kl, step_size, cg_iters and the warnings it raises."""
    params = list(actor.parameters())
    warnings: list[str] = []
    dist = actor.dist(obs)
    loss = surrogate_rows(dist, act, adv, lpo, trpo).mean()
    grad = _flat(torch.autograd.grad(loss, params)).detach()
    with torch.no_grad():
        old = actor.dist(obs)
    # conjugate gradient on fisher(x) + damping x = grad, x0 = 0
    x, r, p = torch.zeros_like(grad), grad.clone(), grad.clone()
    rr, iters = r.dot(r), 0
    for _ in range(cg_steps):
        x, r, p, rr, done = cg_iteration(x, r, p, rr, fisher_product(actor, obs, p), damping, residual_tol)
        iters += 1
        if done:
            break
    theta = _flat(q.data for q in params)
    kl_val = 0.0
    step = float(step_size(x, fisher_product(actor, obs, x), damping, max_kl)) if trpo else float("nan")
    with torch.no_grad():
        if not trpo:
            _load_flat(params, theta - trust_region_size * x)
            kl_val = float(kl_divergence(old, actor.dist(obs)).mean())
        else:
            for i in range(max_backtracks):
                _load_flat(params, theta - step * x)
                new = actor.dist(obs)
                kl_val = float(kl_divergence(old, new).mean())
                if kl_val < max_kl and float(surrogate_rows(new, act, adv, lpo, trpo).mean()) < float(loss):
                    if i > 0:
                        warnings.append(f"Backtracking to step {i}.")
                    break
                if i == max_backtracks - 1:
                    _load_flat(params, theta)
                    step = 0.0
                    warnings.append("Line search failed! It seems hyperparamters are poor and need to be changed.")
                else:
                    step = float(torch.tensor(step, dtype=torch.float32) * backtrack_coeff)
    vf = math.nan
    for _ in range(optim_critic_iters):
        vf_loss = critic_loss(critic, obs, ret)
        critic_opt.zero_grad()
        vf_loss.backward()
        critic_opt.step()
        vf = float(vf_loss.detach())
    return {"actor_loss": float(loss.detach()), "vf_loss": vf, "kl": kl_val, "step_size": step, "cg_iters": iters,
            "warnings": warnings}


def update(actor: Actor, critic: nn.Module, critic_opt: torch.optim.Optimizer, data: dict, perms, batch_size: int | None,
           **kw) -> dict:
    """One ``_update_with_batch`` on preprocessed rows ``data`` (obs, act, adv, returns, logp_old tensors) in the minibatch
    orders ``perms``; ``kw`` as ``minibatch``.  Returns per-minibatch actor_loss / vf_loss / kl / step_size / cg_iters and
    the warning messages."""
    n = data["obs"].shape[0]
    res: dict = {"actor_loss": [], "vf_loss": [], "kl": [], "step_size": [], "cg_iters": [], "warnings": []}
    for perm in perms:
        for lo, hi in bounds(n, batch_size or n):
            idx = torch.as_tensor(perm[lo:hi])
            out = minibatch(actor, critic, critic_opt, *(data[k][idx] for k in ("obs", "act", "adv", "returns", "logp_old")),
                            **kw)
            res["warnings"] += out.pop("warnings")
            for k, v in out.items():
                res[k].append(v)
    return res
