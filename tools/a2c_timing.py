"""Time A2C.update() on one GPU with torch.optim.RMSprop (examples/mujoco/mujoco_a2c.py's optimiser) and with Adam, the two
alternating update by update on the same inputs.

    python tools/a2c_timing.py [--reps 21] [--out timing.json]

Workloads: mujoco_a2c (16 envs x 5 steps = 80 transitions per collect, the whole batch as one minibatch, one repetition; obs 17 /
act 6, tanh [64, 64] actor and critic stand in for the environment) and a 4096 x 128 rollout with minibatch 16384.  Times are
medians of CUDA-event spans of ``--reps`` updates per optimiser after two warm-up updates of each.  Prints the card name and
power limit with the numbers.  Needs a CUDA device.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

WORKLOADS = [("mujoco_a2c_16x5", 16, 5, None), ("rollout_4096x128", 4096, 128, 16384)]     # name, envs, steps, minibatch
O, A = 17, 6


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return {"name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip()}


def build(kind: str, dev: str):
    from tianshou_b200.algorithm import A2C, AdamOptimizerFactory, ProbabilisticActorPolicy
    from tianshou_b200.algorithm.optim import RMSpropOptimizerFactory
    from ts_testutil import Box, build_actor_critic, gaussian_dist
    actor, critic = build_actor_critic(O, A, dev)
    policy = ProbabilisticActorPolicy(actor=actor, dist_fn=gaussian_dist, action_scaling=True, action_bound_method="clip",
                                      action_space=Box(A))
    optim = RMSpropOptimizerFactory(lr=7e-4, eps=1e-5, alpha=0.99) if kind == "rmsprop" else AdamOptimizerFactory(lr=7e-4)
    return A2C(policy=policy, critic=critic, optim=optim, max_grad_norm=0.5, vf_coef=0.5, ent_coef=0.01, gae_lambda=0.95,
               gamma=0.99, return_scaling=True)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=21)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("a2c_timing.py needs a CUDA device")
    from tianshou_b200.data import Batch, VectorReplayBuffer
    from tianshou_b200.utils import policy_within_training_step
    from ts_testutil import synth_rollout
    dev = "cuda:0"
    result = {"card": card(), "workloads": {}}
    for name, E, T, bs in WORKLOADS:
        buf = VectorReplayBuffer(E * T, E, device=dev)
        for s in synth_rollout(np.random.default_rng(0), E, T, O, A, p_term=0.01, trunc_len=1000):
            buf.add(Batch(**s), buffer_ids=np.arange(E))
        algos = {k: build(k, dev) for k in ("rmsprop", "adam")}

        def update(k):
            with policy_within_training_step(algos[k].policy):
                algos[k].update(buffer=buf, batch_size=bs, repeat=1)

        for _ in range(2):
            for k in algos:
                update(k)
        times = {k: [] for k in algos}
        for _ in range(args.reps):
            for k in algos:                       # alternating: both see the same host and GPU conditions
                t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                t0.record()
                update(k)
                t1.record()
                torch.cuda.synchronize()
                times[k].append(t0.elapsed_time(t1))
        result["workloads"][name] = {
            "rows": E * T, "minibatch": bs or E * T,
            **{f"{k}_ms_median": float(np.median(v)) for k, v in times.items()},
            **{f"{k}_ms_p10_p90": [float(np.percentile(v, 10)), float(np.percentile(v, 90))] for k, v in times.items()},
        }
    print(json.dumps(result, indent=1))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
