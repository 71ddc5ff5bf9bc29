"""Time ``DiscreteBCQ.update()`` and ``DiscreteCRR.update()`` on one GPU next to the same update in eager PyTorch
(oracle/oracle_discrete_bcq.py, oracle_discrete_crr.py: torch forwards and autograd backward around the loss rows) on the same
GPU, the same buffer and the same initial weights, in the same call.

    python tools/discrete_offline_timing.py [--reps 21] [--out timing.json]

Workloads, each for both algorithms:
  cartpole_mlp : the test_discrete_bcq.py / test_discrete_crr.py shape -- obs 4, 2 actions, one Net to 64 under both heads, heads
                 [64, 64], batch 64 (BCQ: 3-step returns), a uniform 20000-slot buffer of 10 environments with stored obs_next.
  atari_cnn    : the atari_bcq.py / atari_crr.py shape -- one DQNet(4, 84, 84, features_only=True) behind
                 ScaledObsInputActionReprNet under both heads, heads [512], 6 actions, batch 32, a 100k-slot buffer of uint8
                 single frames (stack_num 4) with the device mirror on.
Device and eager updates alternate; each number is the median wall time of ``--reps`` updates of each after three warm-up
updates of each, with a device synchronise inside the timed region.  The eager update includes what the reference's update does
on the host: the index draw, the frame-stack gather and the upload.  Prints the card's name and power limit, read in the same
run (query only).  Fails without a CUDA device.
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


class _Discrete:
    def __init__(self, n: int) -> None:
        self.n = n
        self.shape = ()


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return {"name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip()}


def _setup(workload: str, algo_name: str):
    from oracle import oracle_discrete_bcq as odb
    from oracle import oracle_discrete_crr as odc
    from oracle import oracle_discrete_sac as ods
    from tianshou_b200.algorithm import (AdamOptimizerFactory, DiscreteActorPolicy, DiscreteBCQ, DiscreteBCQPolicy, DiscreteCRR)
    from tianshou_b200.data import Batch, VectorReplayBuffer
    from tianshou_b200.env.atari import DQNet, ScaledObsInputActionReprNet
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.discrete import DiscreteActor, DiscreteCritic
    torch.manual_seed(0)
    rng = np.random.default_rng(0)
    if workload == "cartpole_mlp":
        A, E, size, B, last, lr = 2, 10, 20000, 64, (64, 64), 3e-4
        trunk = Net(state_shape=(4,), action_shape=64)
        mk, feat = odb.mlp_trunk(4, (), 64)
        buf = VectorReplayBuffer(size, E, device=DEV)
        for _ in range(size // E):
            buf.add(Batch(obs=rng.standard_normal((E, 4)).astype(np.float32), act=rng.integers(0, A, E), rew=rng.standard_normal(E),
                          terminated=rng.random(E) < 0.02, truncated=np.zeros(E, bool),
                          obs_next=rng.standard_normal((E, 4)).astype(np.float32)), buffer_ids=np.arange(E))
    else:
        A, E, size, B, last, lr = 6, 10, 100_000, 32, (512,), 6.25e-5
        trunk = ScaledObsInputActionReprNet(DQNet(4, 84, 84, A, features_only=True))
        mk, feat = odb.cnn_trunk(4, 84, 84)
        buf = VectorReplayBuffer(size, E, stack_num=4, ignore_obs_next=True, save_only_last_obs=True, device=DEV, device_mirror=True)
        for _ in range(size // E):
            st = np.repeat(rng.integers(0, 256, (E, 1, 84, 84), dtype=np.uint8), 4, axis=1)
            buf.add(Batch(obs=st, act=rng.integers(0, A, E), rew=rng.standard_normal(E), terminated=rng.random(E) < 0.01,
                          truncated=np.zeros(E, bool), obs_next=st), buffer_ids=np.arange(E))
    a = DiscreteActor(preprocess_net=trunk, action_shape=A, hidden_sizes=last, softmax_output=False).to(DEV)
    if algo_name == "bcq":
        b = DiscreteActor(preprocess_net=trunk, action_shape=A, hidden_sizes=last, softmax_output=False).to(DEV)
    else:
        b = DiscreteCritic(preprocess_net=trunk, hidden_sizes=last, last_size=A).to(DEV)
    nets = odb.TwoHeadNets(mk, feat, last, (A, A), True).to(DEV)
    with torch.no_grad():
        for p, q in zip(torch.nn.ModuleList([a, b]).parameters(), nets.parameters(), strict=True):
            q.copy_(p)
    view = dict(obs=np.asarray(buf.obs), act=np.asarray(buf.act), rew=np.asarray(buf.rew), done=np.asarray(buf.done),
                terminated=np.asarray(buf.terminated), offset=np.asarray(buf._extend_offset), last_index=buf.last_index,
                lengths=buf._sizes)
    if workload == "cartpole_mlp":
        view["obs_next"] = np.asarray(buf.obs_next)
        obs_of = ods.flat_obs(view["obs"], DEV)
    else:
        obs_of = ods.frame_obs(view, 4, 255.0, DEV)
    if algo_name == "bcq":
        n_step = 3 if workload == "cartpole_mlp" else 1
        policy = DiscreteBCQPolicy(model=a, imitator=b, action_space=_Discrete(A), target_update_freq=8000, unlikely_action_threshold=0.3)
        algo = DiscreteBCQ(policy=policy, optim=AdamOptimizerFactory(lr=lr), gamma=0.99, n_step_return_horizon=n_step,
                           target_update_freq=8000)
        state = odb.BcqState(nets, lr)
        eager = lambda idx: odb.discrete_bcq_update(state, obs_of, view, idx, 0.99, n_step, 8000, float(np.log(0.3)), 1e-2)
    else:
        algo = DiscreteCRR(policy=DiscreteActorPolicy(actor=a, action_space=_Discrete(A)), critic=b, optim=AdamOptimizerFactory(lr=lr),
                           gamma=0.99, target_update_freq=8000)
        state = odc.CrrState(nets, lr, 8000)
        eager = lambda idx: odc.discrete_crr_update(state, obs_of, view, idx, 0.99, "exp", 1.0, 20.0, 10.0)
    return algo, buf, eager, B


def run(workload: str, algo_name: str, reps: int, warmup: int = 3) -> dict:
    from tianshou_b200.utils import policy_within_training_step
    algo, buf, eager, B = _setup(workload, algo_name)

    def device_update():
        with policy_within_training_step(algo.policy):
            algo.update(buffer=buf, sample_size=B)

    def eager_update():
        eager(buf.sample_indices(B))

    np.random.seed(0)
    times = {"device": [], "eager": []}
    for i in range(warmup + reps):
        for name, fn in (("device", device_update), ("eager", eager_update)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            if i >= warmup:
                times[name].append((time.perf_counter() - t0) * 1e3)
    d, e = float(np.median(times["device"])), float(np.median(times["eager"]))
    return {"workload": workload, "algorithm": algo_name, "batch": B, "reps": reps, "device_ms": d, "eager_ms": e, "speedup": e / d,
            "device_all_ms": times["device"], "eager_all_ms": times["eager"]}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=21)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/discrete_offline_timing.py needs a CUDA device: a time measured anywhere else says nothing")
    out = {"card": card(), "results": [run(w, a, args.reps) for w in ("cartpole_mlp", "atari_cnn") for a in ("bcq", "crr")]}
    print(json.dumps(out["card"]))
    for r in out["results"]:
        print(f"{r['workload']:13s} {r['algorithm']} device {r['device_ms']:8.3f} ms ({min(r['device_all_ms']):.3f} - {max(r['device_all_ms']):.3f})"
              f"   eager {r['eager_ms']:8.3f} ms ({min(r['eager_all_ms']):.3f} - {max(r['eager_all_ms']):.3f})   x{r['speedup']:.2f}")
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
