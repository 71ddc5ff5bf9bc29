"""TEST INFRASTRUCTURE -- numpy restatement of clip_grad_norm_ + torch.optim.RMSprop and the actor-critic update loop
that steps with it (the on-policy device update with ``ts_ppo_hparams.optimizer = TS_OPT_RMSPROP``).

Kept beside ``oracle_np`` rather than in it so that the Adam restatement the existing goldens pin stays as it is; the
loss, value pass and GAE are ``oracle_np``'s own."""
from __future__ import annotations

import numpy as np

from oracle import oracle_np as onp

F = np.float32


def clip_rmsprop_step(p, grads, sq, step, hp):
    """clip_grad_norm_ + torch.optim.RMSprop single-tensor step without momentum / centering (algorithm_base.py:496-500;
    torch/optim/rmsprop.py ``_single_tensor_rmsprop``).  In place on p and sq (square_avg); returns (step+1, grad_norm).
    No bias correction; 1 - alpha is formed in double and rounded once, as torch passes addcmul's value."""
    total = np.sqrt(sum(float((g.astype(np.float64) ** 2).sum()) for g in grads.values()))
    coef = F(1.0)
    if hp["max_grad_norm"]:
        coef = F(min(hp["max_grad_norm"] / (F(total) + F(1e-6)), 1.0))
    alpha, w_sq, lr, eps = F(hp["alpha"]), F(1.0 - hp["alpha"]), F(hp["lr"]), F(hp["eps"])
    for k in (onp.PARAM_ORDER if set(grads) == set(onp.PARAM_ORDER) else list(grads)):
        g = (grads[k] * coef).astype(F)
        if hp.get("weight_decay"):
            g = g + F(hp["weight_decay"]) * p[k]
        sq[k] *= alpha                                  # square_avg.mul_(alpha).addcmul_(grad, grad, value=1 - alpha)
        sq[k] += w_sq * g * g
        avg = np.sqrt(sq[k]) + eps                      # square_avg.sqrt().add_(eps)
        p[k] -= lr * (g / avg)                          # param.addcdiv_(grad, avg, value=-lr)
    return step + 1, total


def optimizer_step(p, grads, state, step, hp):
    """One optimiser step of either kind: ``hp["optimizer"] == "rmsprop"`` -> ``clip_rmsprop_step`` on state["square_avg"],
    else ``oracle_np.clip_adam_step`` on state["exp_avg"] / state["exp_avg_sq"]."""
    if hp.get("optimizer") == "rmsprop":
        return clip_rmsprop_step(p, grads, state["square_avg"], step, hp)
    return onp.clip_adam_step(p, grads, state["exp_avg"], state["exp_avg_sq"], step, hp)


def init_state(p, hp):
    zeros = lambda: {k: np.zeros_like(v) for k, v in p.items()}      # noqa: E731
    return {"square_avg": zeros()} if hp.get("optimizer") == "rmsprop" else {"exp_avg": zeros(), "exp_avg_sq": zeros()}


def ppo_update(p, state, step, rollout, perms, batch_size, repeat, hp, rms, gamma, lam, recompute_adv):
    """``oracle_np.ppo_update`` (Gaussian tanh actor-critic, PPO or A2C loss) with the optimiser chosen by ``hp``."""
    v_s, returns, adv = onp.add_returns_and_advantages(p, rollout, rms, gamma, lam)
    mu, sigma, _, _ = onp.actor_forward(p, rollout["obs"])
    logp_old = onp.normal_logp(rollout["act"].astype(F), mu, sigma)
    first = dict(v_s=v_s.copy(), returns=returns.copy(), adv=adv.copy(), logp_old=logp_old.copy())
    n = len(adv)
    losses, norms = [], []
    for r in range(repeat):
        if recompute_adv and r > 0:
            v_s, returns, adv = onp.add_returns_and_advantages(p, rollout, rms, gamma, lam)
        for lo, hi in onp.minibatch_bounds(n, batch_size or n):
            idx = perms[r][lo:hi]
            mb = dict(obs=rollout["obs"][idx], act=rollout["act"][idx], adv=adv[idx], returns=returns[idx],
                      logp_old=logp_old[idx], v_s=v_s[idx])
            grads, ls = onp.ppo_minibatch_grad(p, mb, hp)
            step, norm = optimizer_step(p, grads, state, step, hp)
            losses.append(ls)
            norms.append(norm)
    return dict(first=first, losses=np.array(losses), grad_norms=np.array(norms), step=step, v_s=v_s, returns=returns,
                adv=adv)
