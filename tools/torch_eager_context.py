"""CONTEXT ONLY (never the target, never on the product path): the same PPO ``update()`` written the way the reference writes
it -- stock PyTorch modules, autograd, ``clip_grad_norm_``, ``torch.optim.Adam``, one minibatch at a time (ppo.py:164-224,
a2c.py:115-153) -- but with every tensor on the GPU and the chunked 256-row no-grad passes replaced by full-batch forwards.
SURVEY 2.3 names this number as part of the bar ("what moving the reference's own code to the GPU would give").

    python tools/torch_eager_context.py [--envs 4096] [--steps 2]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np
import torch
from torch import nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def run(E: int = 4096, T: int = 128, bs: int = 16384, repeat: int = 10, steps: int = 2, device: str = "cuda:0") -> dict:
    from tianshou_b200.synthetic import synth_rollout
    dev = torch.device(device)
    O, A = 17, 6
    torch.manual_seed(0)

    def trunk():
        return nn.Sequential(nn.Linear(O, 64), nn.Tanh(), nn.Linear(64, 64), nn.Tanh())

    actor, mu, critic = trunk().to(dev), nn.Linear(64, A).to(dev), nn.Sequential(trunk(), nn.Linear(64, 1)).to(dev)
    logstd = nn.Parameter(torch.full((A,), -0.5, device=dev))
    params = [*actor.parameters(), *mu.parameters(), logstd, *critic.parameters()]
    opt = torch.optim.Adam(params, lr=3e-4)
    cols: dict[str, list] = {k: [] for k in ("obs", "act", "rew", "terminated", "truncated", "obs_next")}
    for s in synth_rollout(np.random.default_rng(0), E, T, O, A):
        for k in cols:
            cols[k].append(s[k])
    host = {k: np.stack(v, axis=1).reshape(E * T, *v[0].shape[1:]) for k, v in cols.items()}
    N = E * T

    def dist(o):
        return torch.distributions.Independent(torch.distributions.Normal(mu(actor(o)), logstd.exp()), 1)

    def gae(v_s, v_next, rew, term, end):       # the reverse scan stays a host loop in the reference (numba); here: per-env torch loop over T
        delta = rew + 0.99 * v_next * (~term) - v_s
        adv = torch.zeros_like(delta)
        d2, e2, a2 = delta.view(E, T), end.view(E, T), adv.view(E, T)
        run_ = torch.zeros(E, device=dev, dtype=delta.dtype)
        for t in range(T - 1, -1, -1):
            run_ = d2[:, t] + 0.99 * 0.95 * (~e2[:, t]) * run_
            a2[:, t] = run_
        return adv

    def update():
        d = {k: torch.from_numpy(v).to(dev, non_blocking=True) for k, v in host.items()}
        obs, obs_next, act = d["obs"].float(), d["obs_next"].float(), d["act"].float()
        rew, term = d["rew"], d["terminated"]
        end = term | d["truncated"]
        end.view(E, T)[:, -1] = True
        with torch.no_grad():
            logp_old = dist(obs).log_prob(act)
        for r in range(repeat):
            with torch.no_grad():
                v_s, v_next = critic(obs).flatten().double(), critic(obs_next).flatten().double()
                adv = gae(v_s, v_next, rew, term, end)
                ret = (adv + v_s).float()
                adv, v_s32 = adv.float(), v_s.float()
            perm = torch.from_numpy(np.random.permutation(N)).to(dev)
            for lo in range(0, N, bs):
                idx = perm[lo:lo + bs]
                dd = dist(obs[idx])
                ratio = (dd.log_prob(act[idx]) - logp_old[idx]).exp()
                a = adv[idx]
                clip_loss = -torch.min(ratio * a, ratio.clamp(0.8, 1.2) * a).mean()
                v = critic(obs[idx]).flatten()
                v_clip = v_s32[idx] + (v - v_s32[idx]).clamp(-0.2, 0.2)
                vf = torch.max((ret[idx] - v).pow(2), (ret[idx] - v_clip).pow(2)).mean()
                loss = clip_loss + 0.25 * vf
                opt.zero_grad()
                loss.backward()
                nn.utils.clip_grad_norm_(params, 0.5)
                opt.step()
                _ = (loss.item(), clip_loss.item(), vf.item())        # the reference's per-step .item() calls

    update()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        update()
    torch.cuda.synchronize()
    dt = (time.perf_counter() - t0) / steps
    return {"value": N / dt, "unit": "transitions/s", "ms_per_update": 1e3 * dt, "what": "stock PyTorch eager + autograd + torch.optim.Adam on the "
            f"{torch.cuda.get_device_name()}, {E} envs x {T} steps, minibatch {bs}, repeat {repeat}, return scaling omitted, full-batch no-grad passes: context only"}


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=2)
    a = ap.parse_args()
    print(json.dumps(run(E=a.envs, steps=a.steps)))
