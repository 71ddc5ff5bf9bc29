"""Time ``TD3.update()`` / ``TD3BC.update()`` on one GPU next to the eager-PyTorch restatement of the reference's update
(oracle/oracle_td3.py) on the same GPU, the same buffer and the same initial weights, in the same call.

    python tools/td3_timing.py [--reps 21] [--out timing.json]

Workloads ([256, 256] networks, batch 256, obs 17, act 6, update_actor_freq 2):
  ``mujoco_td3``  : examples/mujoco/mujoco_td3.py -- TD3, n = 1, on a 100k-slot buffer with the device mirror on
  ``d4rl_td3_bc`` : examples/offline/d4rl_td3_bc.py -- TD3+BC, n = 3, on a 100k-transition ``from_data`` buffer with the mirror on
Actor-step and critic-only updates are reported separately: each number is the median wall time of ``--reps`` updates of that
kind after four warm-up updates, with a device synchronise inside the timed region, and its 10th-90th percentile range.  The
eager update includes the index draw, the host n-step return (as the reference computes it) and the upload of the sampled rows.
Prints the card name and power limit with the numbers.  Needs a CUDA device.
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
WORKLOADS = {"mujoco_td3": dict(algo="td3", n_step=1), "d4rl_td3_bc": dict(algo="bc", n_step=3)}


class _Box:
    def __init__(self, dim: int) -> None:
        self.shape = (dim,)
        self.low = -np.ones(dim, np.float32)
        self.high = np.ones(dim, np.float32)


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return {"name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip()}


def _time_split_ms(fn, is_actor_step, reps: int, warmup: int = 4) -> tuple[list[float], list[float]]:
    """Wall times of ``fn`` split by ``is_actor_step()`` (read before the call), ``reps`` of each kind."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    actor, critic = [], []
    while len(actor) < reps or len(critic) < reps:
        kind = actor if is_actor_step() else critic
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        kind.append((time.perf_counter() - t0) * 1e3)
    return actor[:reps], critic[:reps]


def run(name: str, reps: int) -> dict:
    from oracle.oracle_td3 import Td3Nets, td3_update
    from tianshou_b200.algorithm import TD3, TD3BC, AdamOptimizerFactory
    from tianshou_b200.algorithm.modelfree.ddpg import ContinuousDeterministicPolicy
    from tianshou_b200.data import ReplayBuffer
    from tianshou_b200.utils import policy_within_training_step
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.continuous import ContinuousActorDeterministic, ContinuousCritic
    w = WORKLOADS[name]
    O, A, H, B, N, n_step, freq = 17, 6, (256, 256), 256, 100_000, w["n_step"], 2
    rng = np.random.default_rng(0)
    term = rng.random(N) < 1e-3
    trunc = np.zeros(N, bool)
    trunc[999::1000] = True
    trunc &= ~term
    data = (rng.standard_normal((N, O)).astype(np.float32), np.tanh(rng.standard_normal((N, A))).astype(np.float32),
            rng.standard_normal(N), term, trunc, term | trunc, rng.standard_normal((N, O)).astype(np.float32))
    torch.manual_seed(0)
    actor = ContinuousActorDeterministic(preprocess_net=Net(state_shape=(O,), hidden_sizes=H), action_shape=(A,)).to(DEV)
    crit = ContinuousCritic(preprocess_net=Net(state_shape=(O,), action_shape=(A,), hidden_sizes=H, concat=True)).to(DEV)
    nets = Td3Nets(O, A, H)
    with torch.no_grad():
        for p, q in zip(nets.a.parameters(), actor.parameters(), strict=True):
            p.copy_(q.detach().cpu())
        for k in range(2):
            for p, q in zip(nets.c[k].parameters(), crit.parameters(), strict=True):
                p.copy_(q.detach().cpu())
            nets.c_old[k].load_state_dict(nets.c[k].state_dict())
        nets.a_old.load_state_dict(nets.a.state_dict())
    kw = dict(policy=ContinuousDeterministicPolicy(actor=actor, action_space=_Box(A)), policy_optim=AdamOptimizerFactory(lr=3e-4),
              critic=crit, critic_optim=AdamOptimizerFactory(lr=3e-4), update_actor_freq=freq, n_step_return_horizon=n_step)
    algo = TD3BC(alpha=2.5, **kw) if w["algo"] == "bc" else TD3(**kw)
    buf = ReplayBuffer.from_data(*data)
    buf.enable_device_mirror()
    buf.sync_device_mirror()

    def device_update():
        with policy_within_training_step(algo.policy):
            algo.update(buf, B)

    for m in nets.modules():
        m.to(DEV)
    opts = [torch.optim.Adam(nets.a.parameters(), lr=3e-4), torch.optim.Adam(nets.c[0].parameters(), lr=3e-4),
            torch.optim.Adam(nets.c[1].parameters(), lr=3e-4)]
    host = {k: np.asarray(v) for k, v in zip(("obs", "act", "rew", "terminated", "truncated", "done", "obs_next"), data, strict=True)}
    host.update(offset=np.array([0, N]), last_index=np.asarray(buf.last_index), lengths=np.array([N]),
                unfinished=[] if host["done"][N - 1] else [N - 1])
    eager_rs = np.random.RandomState(1)
    eager_cnt = [0]

    def eager_update():
        idx = eager_rs.choice(N, B)
        r = td3_update(nets, opts, host, idx, lambda shape: torch.randn(shape, device=DEV), gamma=0.99, n_step=n_step, tau=0.005,
                       policy_noise=0.2, noise_clip=0.5, actor_step=eager_cnt[0] % freq == 0,
                       bc_alpha=2.5 if w["algo"] == "bc" else None)
        eager_cnt[0] += 1
        float(r["critic1_loss"])

    da, dc = _time_split_ms(device_update, lambda: algo._cnt % freq == 0, reps)
    ea, ec = _time_split_ms(eager_update, lambda: eager_cnt[0] % freq == 0, reps)
    pct = lambda x: [float(np.percentile(x, 10)), float(np.percentile(x, 90))]
    out = {"workload": name, "obs": O, "act": A, "batch": B, "n_step": n_step, "update_actor_freq": freq}
    for kind, d, e in (("actor_step", da, ea), ("critic_only", dc, ec)):
        out[kind] = {"device_ms": float(np.median(d)), "device_p10_p90": pct(d), "eager_ms": float(np.median(e)),
                     "eager_p10_p90": pct(e), "speedup": float(np.median(e) / np.median(d))}
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=21)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    out = {"card": card(), "results": [run(w, args.reps) for w in WORKLOADS]}
    print(json.dumps(out["card"]))
    for r in out["results"]:
        for kind in ("actor_step", "critic_only"):
            x = r[kind]
            print(f"{r['workload']:12s} {kind:12s} device {x['device_ms']:8.3f} ms (p10-p90 {x['device_p10_p90'][0]:.3f}-"
                  f"{x['device_p10_p90'][1]:.3f})   eager {x['eager_ms']:8.3f} ms (p10-p90 {x['eager_p10_p90'][0]:.3f}-"
                  f"{x['eager_p10_p90'][1]:.3f})   x{x['speedup']:.2f}")
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
