"""TEST INFRASTRUCTURE -- float64 numpy restatement of FQF's fraction proposal, target selection and fraction loss rows (the W1
fraction loss, the entropy, d loss / d z), and its update on plain torch networks.

Only ``tests/`` and ``tools/`` may import this module; ``tianshou_b200`` never does.  It restates
tianshou/algorithm/modelfree/fqf.py and utils/net/discrete.py:219-314 without the framework around it:

  fractions: discrete.py:219-252 (Categorical(logits=z): softmax, cumsum padded with 0, midpoints, the clamped entropy)
  network  : IQN's (oracle_iqn.IqnNet) at tau_hats, and without gradient at taus[:, 1:-1]
  target   : fqf.py:94-98 and :178-193: the first arg-max of sum_n (taus[n+1] - taus[n]) q[n], the lagged network's quantiles of
             that action at the ONLINE tau_hats (the online ones when ``target_update_freq == 0``)
  losses   : the quantile loss is oracle_iqn.iqn_rows with tau_hats; the fraction loss fqf.py:221-247 with its strict sign tests
  steps    : the fraction optimiser (Adam or RMSprop) on the fraction net only, the main Adam on the quantile network only
  lagged   : dqn.py:277-286 (full copy of the quantile network when ``_iter % freq == 0``, before the step)

The kernels' layout is q[B][N][A] (sample-major); the reference's is q[B, A, N].  ``FqfState`` with ``fqf_update_torch`` is the
eager baseline of tools/fqf_timing.py.

PINNING: tests/test_oracle_fqf.py replays tests/golden/fqf_ref_*.npz (outputs of the imported reference,
oracle/gen_golden_fqf.py) through ``fqf_update`` and checks ``fractions`` / ``fraction_rows`` against float64 autograd of the
reference's expressions.
"""
from __future__ import annotations

import copy
from collections.abc import Callable

import numpy as np
import torch
from torch import nn

from oracle import oracle_iqn as oi
from oracle.oracle_discrete_bcq import obs_next_of
from oracle.oracle_offpolicy import compute_nstep_targets

FRACTION_INIT_SCALE = 4.0     # the goldens' fraction weights: 4x seeded_params' range, so the proposed widths are far from uniform


def seed_fraction_net(lin: nn.Linear, seed: int) -> None:
    """The goldens' fraction weights: uniform in +-4/sqrt(D), bias uniform in +-4/sqrt(N), from numpy's PCG64 stream."""
    rng = np.random.default_rng(seed)
    with torch.no_grad():
        for p in (lin.weight, lin.bias):
            fan_in = int(p.shape[1]) if p.dim() > 1 else p.numel()
            b = FRACTION_INIT_SCALE / np.sqrt(fan_in)
            p.copy_(torch.from_numpy(rng.uniform(-b, b, tuple(p.shape)).astype(np.float32)))


# ------------------------------------------------------------------------------------------------ fractions, float64
def fractions(z: np.ndarray) -> dict:
    """The proposal from the fraction net's output z [B, N]: p = softmax(z), logp = max(z - logsumexp(z), finfo.min) (the
    entropy's clamp: an underflowed p gives 0, not NaN), H = -sum logp * p, taus [B, N + 1] = (0, cumsum p), tau_hats the
    midpoints, inner = taus[:, 1:-1]."""
    z = np.asarray(z, np.float64)
    m = z.max(1, keepdims=True)
    e = np.exp(z - m)
    s = e.sum(1, keepdims=True)
    l = np.maximum(z - (m + np.log(s)), np.finfo(np.float32).min)
    p = e / s
    taus = np.concatenate([np.zeros((z.shape[0], 1)), np.cumsum(p, 1)], 1)
    return dict(p=p, logp=l, H=-(l * p).sum(1), taus=taus, tau_hats=(taus[:, :-1] + taus[:, 1:]) / 2, inner=taus[:, 1:-1])


def fqf_select(q: np.ndarray, taus: np.ndarray) -> np.ndarray:
    """The policy's action on q[B][N][A]: the first arg-max of sum_n (taus[n+1] - taus[n]) q[n]   (fqf.py:94-98)."""
    w = np.diff(np.asarray(taus, np.float64), axis=1)
    return (w[:, :, None] * np.asarray(q, np.float64)).sum(1).argmax(1)


def fqf_target(q_online: np.ndarray, taus: np.ndarray, q_next: np.ndarray) -> np.ndarray:
    """``q_next[b, :, a*]`` [B, N] with a* the online fraction-weighted arg-max; [B][N][A] layout."""
    a = fqf_select(q_online, taus)
    return np.asarray(q_next)[np.arange(len(a)), :, a]


def gradient_of_taus(h: np.ndarray, c: np.ndarray) -> np.ndarray:
    """g [B, N - 1] from the chosen action's quantiles at tau_hats h [B, N] and at taus[:, 1:-1] c [B, N - 1], with the
    reference's strict sign tests (fqf.py:229-243)."""
    v1, v2 = c - h[:, :-1], c - h[:, 1:]
    s1 = c > np.concatenate([h[:, :1], c[:, :-1]], 1)
    s2 = c < np.concatenate([c[:, 1:], h[:, -1:]], 1)
    return np.where(s1, v1, -v1) + np.where(s2, v2, -v2)


def fraction_rows(q_hat: np.ndarray, q_tau: np.ndarray, act: np.ndarray, fr: dict, ent_coef: float) -> dict:
    """fraction_loss, entropy_loss, their total ``fraction_loss - ent_coef * entropy_loss`` and its gradient dz [B, N] at the
    fraction net's output, on q_hat [B][N][A] and q_tau [B][N-1][A] and the proposal ``fr`` (``fractions``' dict).
    dz_bj = (1/B) p_j ((G_j - sum_k p_k G_k) + ent_coef (logp_j + H_b)), G_j = sum_{i > j} g_i over the taus index i."""
    B = q_hat.shape[0]
    rows = np.arange(B)
    h = np.asarray(q_hat, np.float64)[rows, :, act]
    c = np.asarray(q_tau, np.float64)[rows, :, act]
    g = gradient_of_taus(h, c)
    frac_b = (g * fr["taus"][:, 1:-1]).sum(1)
    G = np.concatenate([np.cumsum(g[:, ::-1], 1)[:, ::-1], np.zeros((B, 1))], 1)    # G_j = sum_{i >= j} g[:, i]
    p = fr["p"]
    S = (p * G).sum(1, keepdims=True)
    dz = p * ((G - S) + ent_coef * (fr["logp"] + fr["H"][:, None])) / B
    fl, el = float(frac_b.mean()), float(fr["H"].mean())
    return dict(g=g, frac_b=frac_b, fraction_loss=fl, entropy_loss=el, total=fl - ent_coef * el, dz=dz)


def reference_fraction_loss(z: torch.Tensor, sa_quantile_hats: torch.Tensor, sa_quantiles: torch.Tensor,
                            ent_coef: float) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """(fraction_entropy_loss, fraction_loss, entropy_loss): discrete.py:242-252 and fqf.py:221-247 in torch, as the reference
    writes them, from the fraction net's output z [B, N] and the chosen action's quantiles at tau_hats [B, N] and at
    taus[:, 1:-1] [B, N - 1] (any dtype)."""
    dist = torch.distributions.Categorical(logits=z)
    taus = torch.nn.functional.pad(torch.cumsum(dist.probs, dim=1), (1, 0))
    entropies = dist.entropy()
    with torch.no_grad():
        values_1 = sa_quantiles - sa_quantile_hats[:, :-1]
        signs_1 = sa_quantiles > torch.cat([sa_quantile_hats[:, :1], sa_quantiles[:, :-1]], dim=1)
        values_2 = sa_quantiles - sa_quantile_hats[:, 1:]
        signs_2 = sa_quantiles < torch.cat([sa_quantiles[:, 1:], sa_quantile_hats[:, -1:]], dim=1)
        gradient_of_taus = torch.where(signs_1, values_1, -values_1) + torch.where(signs_2, values_2, -values_2)
    fraction_loss = (gradient_of_taus * taus[:, 1:-1]).sum(1).mean()
    entropy_loss = entropies.mean()
    return fraction_loss - ent_coef * entropy_loss, fraction_loss, entropy_loss


# ------------------------------------------------------------------------------------------------ update
class FqfState:
    """The quantile network (``oracle_iqn.IqnNet``), its lagged copy (None: ``target_update_freq == 0``), the fraction net
    ``Linear(D, N)``, Adam on the network, Adam or RMSprop on the fraction net and the iteration counter."""

    def __init__(self, net: oi.IqnNet, frac: nn.Linear, lr: float, frac_opt: str, frac_lr: float, freq: int):
        self.net, self.frac = net, frac
        self.old = copy.deepcopy(net) if freq > 0 else None
        self.opt = torch.optim.Adam(net.parameters(), lr=lr)
        cls = torch.optim.RMSprop if frac_opt == "rmsprop" else torch.optim.Adam
        self.fopt = cls(frac.parameters(), lr=frac_lr)
        self.freq = freq
        self.iter = 0


def _trunk_and_quantiles(net: oi.IqnNet, x: torch.Tensor, taus: torch.Tensor, feat: torch.Tensor | None = None):
    """(feat, q [B, A, S]) of ``net`` at the fractions ``taus`` (the trunk's ``feat`` when already computed)."""
    feat = net.preprocess(x) if feat is None else feat
    B, S = taus.shape
    i_pi = np.pi * torch.arange(1, net.C + 1, dtype=taus.dtype, device=taus.device)
    e = torch.relu(net.embed(torch.cos(taus.view(B, S, 1) * i_pi).view(B * S, net.C)))
    h = (feat.unsqueeze(1) * e.view(B, S, -1)).view(B * S, -1)
    return feat, net.last(h).view(B, S, -1).transpose(1, 2)


def _propose(frac: nn.Linear, feat: torch.Tensor) -> tuple[torch.Tensor, dict, dict]:
    """z, its proposal in float64 (for the fraction loss) and the fractions the network is evaluated at: ``taus``, ``tau_hats``
    and ``inner`` formed in fp32 as the reference forms them (discrete.py:242-249), so that the quantile network sees the
    reference's fractions bit for bit."""
    z = frac(feat.detach())
    with torch.no_grad():
        taus = torch.nn.functional.pad(torch.cumsum(torch.distributions.Categorical(logits=z).probs, dim=1), (1, 0))
    at = dict(taus=taus, tau_hats=(taus[:, :-1] + taus[:, 1:]) / 2.0, inner=taus[:, 1:-1].contiguous())
    return z, fractions(z.detach().cpu().numpy()), at


def fqf_update(s: FqfState, obs_of: Callable[[np.ndarray], torch.Tensor], buf: dict, indices: np.ndarray,
               is_weight: np.ndarray | None, gamma: float, n_step: int, ent_coef: float) -> dict:
    """One ``FQF.update`` on the sampled ``indices``: the forwards in torch fp32, the proposal, the target, the loss rows and
    the fraction gradient in float64 numpy, the gradients pushed back through the networks with autograd."""
    dev = next(s.net.parameters()).device

    def target_q(terminal: np.ndarray) -> torch.Tensor:
        x = obs_next_of(obs_of, buf, terminal, dev)
        with torch.no_grad():
            feat = s.net.preprocess(x)
            _, _, at = _propose(s.frac, feat)
            th = at["tau_hats"]
            q = _trunk_and_quantiles(s.net, x, th, feat)[1].transpose(1, 2)
            q_next = _trunk_and_quantiles(s.old, x, th)[1].transpose(1, 2) if s.old is not None else q
        return torch.from_numpy(fqf_target(q.cpu().numpy(), at["taus"].cpu().numpy(), q_next.cpu().numpy()))

    returns = compute_nstep_targets(buf, indices, target_q, gamma, n_step).reshape(len(indices), -1)
    if s.old is not None and s.iter % s.freq == 0:
        s.old.load_state_dict(s.net.state_dict())
    s.iter += 1
    x = obs_of(indices)
    feat = s.net.preprocess(x)
    z, fr, at = _propose(s.frac, feat)
    q = _trunk_and_quantiles(s.net, x, at["tau_hats"], feat)[1].transpose(1, 2)        # [B, N, A]
    with torch.no_grad():
        q_tau = _trunk_and_quantiles(s.net, x, at["inner"], feat)[1].transpose(1, 2)
    act = np.asarray(buf["act"])[indices].astype(np.int64).reshape(-1)
    qd = q.detach().cpu().numpy()
    r = oi.iqn_rows(qd, act, returns, at["tau_hats"].cpu().numpy(), is_weight)
    fl = fraction_rows(qd, q_tau.cpu().numpy(), act, fr, ent_coef)
    s.fopt.zero_grad()
    z.backward(torch.as_tensor(fl["dz"], dtype=torch.float32, device=dev))
    s.fopt.step()
    s.opt.zero_grad()
    q.backward(torch.as_tensor(r["dq"], dtype=torch.float32, device=dev))
    s.opt.step()
    return dict(returns=returns, losses=np.array([r["loss"] + fl["total"], r["loss"], fl["fraction_loss"], fl["entropy_loss"]]),
                prio=r["prio"])


def fqf_update_torch(s: FqfState, obs_of: Callable[[np.ndarray], torch.Tensor], buf: dict, indices: np.ndarray, gamma: float,
                     n_step: int, ent_coef: float) -> float:
    """The same update as the reference runs it in eager PyTorch: the proposal, the target and the losses in torch on the
    networks' device, the n-step return on the host (algorithm_base.py:721-817), autograd and torch's optimisers.  Returns the
    loss."""
    dev = next(s.net.parameters()).device

    def propose(z):
        dist = torch.distributions.Categorical(logits=z)
        taus = torch.nn.functional.pad(torch.cumsum(dist.probs, dim=1), (1, 0))
        return taus, (taus[:, :-1] + taus[:, 1:]).detach() / 2.0, dist.entropy()

    def target_q(terminal: np.ndarray) -> torch.Tensor:
        x = obs_next_of(obs_of, buf, terminal, dev)
        with torch.no_grad():
            feat = s.net.preprocess(x)
            taus, th, _ = propose(s.frac(feat))
            q = _trunk_and_quantiles(s.net, x, th, feat)[1]
            a = ((taus[:, 1:] - taus[:, :-1]).unsqueeze(1) * q).sum(2).max(1)[1]
            q_next = _trunk_and_quantiles(s.old, x, th)[1] if s.old is not None else q
            return q_next[torch.arange(len(a), device=dev), a, :].cpu()

    returns = torch.as_tensor(compute_nstep_targets(buf, indices, target_q, gamma, n_step).reshape(len(indices), -1), device=dev)
    if s.old is not None and s.iter % s.freq == 0:
        s.old.load_state_dict(s.net.state_dict())
    s.iter += 1
    x = obs_of(indices)
    feat = s.net.preprocess(x)
    z = s.frac(feat.detach())
    taus, th, _ = propose(z.detach())
    q = _trunk_and_quantiles(s.net, x, th, feat)[1]
    with torch.no_grad():
        q_tau = _trunk_and_quantiles(s.net, x, taus[:, 1:-1], feat)[1]
    act = torch.as_tensor(np.asarray(buf["act"])[indices].astype(np.int64), device=dev)
    rows = torch.arange(len(act), device=dev)
    loss = oi.reference_loss(q, act, returns, th, 1.0)[0]
    floss = reference_fraction_loss(z, q[rows, act, :].detach(), q_tau[rows, act, :], ent_coef)[0]
    s.fopt.zero_grad()
    floss.backward()
    s.fopt.step()
    s.opt.zero_grad()
    loss.backward()
    s.opt.step()
    return loss.item() + floss.item()
