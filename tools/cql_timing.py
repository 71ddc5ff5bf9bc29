"""Time ``CQL.update()`` on one GPU next to the eager-PyTorch restatement of the reference's update (oracle/oracle_cql.py) on
the same GPU, the same buffer and the same initial weights, in the same call.

    python tools/cql_timing.py [--reps 21] [--out timing.json]

Workloads (examples/offline/d4rl_cql.py defaults: [256, 256] networks, batch 256, num_repeat_actions 10, Lagrange,
calibrated): ``hopper`` (obs 11, act 3) and ``halfcheetah`` (obs 17, act 6), each on a 100k-transition ``from_data`` buffer
with the device mirror on.  Each number is the median wall time of ``--reps`` updates after three warm-up updates, with a device
synchronise inside the timed region, and its 10th-90th percentile range.  The eager update includes the index draw and the
upload of the sampled rows.  Prints the card name and power limit with the numbers.  Needs a CUDA device.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DEV = "cuda:0"
WORKLOADS = {"hopper": (11, 3), "halfcheetah": (17, 6)}


class _Box:
    def __init__(self, dim: int) -> None:
        self.shape = (dim,)
        self.low = -np.ones(dim, np.float32)
        self.high = np.ones(dim, np.float32)


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return {"name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip()}


def _time_ms(fn, reps: int, warmup: int = 3) -> list[float]:
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        out.append((time.perf_counter() - t0) * 1e3)
    return out


def run(name: str, reps: int) -> dict:
    from oracle.oracle_cql import cql_nets, cql_update
    from tianshou_b200.algorithm import CQL, AdamOptimizerFactory
    from tianshou_b200.algorithm.modelfree.sac import SACPolicy
    from tianshou_b200.data import ReplayBuffer
    from tianshou_b200.utils import policy_within_training_step
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.continuous import ContinuousActorProbabilistic, ContinuousCritic
    O, A = WORKLOADS[name]
    H, B, R, n = (256, 256), 256, 10, 100_000
    rng = np.random.default_rng(0)
    term = rng.random(n) < 1e-3
    trunc = np.zeros(n, bool)
    trunc[999::1000] = True
    trunc &= ~term
    data = (rng.standard_normal((n, O)).astype(np.float32), np.tanh(rng.standard_normal((n, A))).astype(np.float32),
            rng.standard_normal(n), term, trunc, term | trunc, rng.standard_normal((n, O)).astype(np.float32))
    torch.manual_seed(0)
    actor = ContinuousActorProbabilistic(preprocess_net=Net(state_shape=(O,), hidden_sizes=H), action_shape=(A,), unbounded=True,
                                         conditioned_sigma=True).to(DEV)
    crit = ContinuousCritic(preprocess_net=Net(state_shape=(O,), action_shape=(A,), hidden_sizes=H, concat=True)).to(DEV)
    nets = cql_nets(O, A, H)
    src = [*actor.preprocess.parameters(), *actor.mu.parameters(), *actor.sigma.parameters()]
    with torch.no_grad():
        for p, q in zip(nets.actor_params(), src, strict=True):
            p.copy_(q.detach().cpu())
        for k in range(2):
            for p, q in zip(nets.c[k].parameters(), crit.parameters(), strict=True):
                p.copy_(q.detach().cpu())
            nets.c_old[k].load_state_dict(nets.c[k].state_dict())
    algo = CQL(policy=SACPolicy(actor=actor, action_space=_Box(A)), policy_optim=AdamOptimizerFactory(lr=1e-4), critic=crit,
               critic_optim=AdamOptimizerFactory(lr=3e-4), num_repeat_actions=R)
    buf = ReplayBuffer.from_data(*data)
    buf.enable_device_mirror()
    buf.sync_device_mirror()
    buf = algo.process_buffer(buf)

    def device_update():
        with policy_within_training_step(algo.policy):
            algo.update(buf, B)

    for m in (nets.a_trunk, nets.a_mu, nets.a_sigma, *nets.c, *nets.c_old):
        m.to(DEV)
    opts = [torch.optim.Adam(nets.actor_params(), lr=1e-4), torch.optim.Adam(nets.c[0].parameters(), lr=3e-4),
            torch.optim.Adam(nets.c[1].parameters(), lr=3e-4)]
    la = torch.tensor([0.0], requires_grad=True, device=DEV)
    mult = (la, torch.optim.Adam([la], lr=1e-4))
    cal = np.asarray(buf._meta["calibration_returns"])
    host = {k: np.asarray(v) for k, v in zip(("obs", "act", "rew", "terminated", "truncated", "done", "obs_next"), data, strict=True)}
    eager_rs = np.random.RandomState(1)
    noise = lambda shape: torch.randn(shape, device=DEV)

    def eager_update():
        idx = eager_rs.choice(n, B)
        t = lambda a: torch.as_tensor(a[idx], dtype=torch.float32).to(DEV)
        batch = dict(obs=t(host["obs"]), act=t(host["act"]), rew=t(host["rew"]), done=t(host["done"].astype(np.float32)),
                     obs_next=t(host["obs_next"]), calibration_returns=t(cal))
        r = cql_update(nets, opts, 0.2, mult, batch, noise, gamma=0.99, tau=0.005, temperature=1.0, cql_weight=1.0,
                       num_repeat_actions=R, lagrange_threshold=10.0, min_action=-1.0, max_action=1.0, alpha_min=0.0, alpha_max=1e6,
                       max_grad_norm=1.0)
        float(r["critic1_loss"])

    d = _time_ms(device_update, reps)
    e = _time_ms(eager_update, reps)
    pct = lambda x: [float(np.percentile(x, 10)), float(np.percentile(x, 90))]
    return {"workload": name, "obs": O, "act": A, "batch": B, "num_repeat_actions": R, "device_ms": float(np.median(d)),
            "device_p10_p90": pct(d), "eager_ms": float(np.median(e)), "eager_p10_p90": pct(e),
            "speedup": float(np.median(e) / np.median(d))}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=21)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    out = {"card": card(), "results": [run(w, args.reps) for w in WORKLOADS]}
    print(json.dumps(out["card"]))
    for r in out["results"]:
        print(f"{r['workload']:12s} device {r['device_ms']:8.3f} ms (p10-p90 {r['device_p10_p90'][0]:.3f}-{r['device_p10_p90'][1]:.3f})"
              f"   eager {r['eager_ms']:8.3f} ms (p10-p90 {r['eager_p10_p90'][0]:.3f}-{r['eager_p10_p90'][1]:.3f})   x{r['speedup']:.2f}")
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
