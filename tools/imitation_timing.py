"""Time ``OfflineImitationLearning.update()`` / ``OffPolicyImitationLearning.update()`` on one GPU next to the same update in eager
PyTorch (the batch read through the buffer's ``__getitem__`` as the reference reads it, the actor's torch forward, the reference's
loss, autograd and torch's Adam) on the same GPU, the same buffer and the same initial weights, in the same call.

    python tools/imitation_timing.py [--reps 21] [--out timing.json]

Workloads:
  d4rl_il   obs 17, 6 actions, ``ContinuousActorDeterministic`` over ``Net([256, 256], action_shape=6)``, batch 256, a 100k-slot
            mirrored buffer (examples/offline/d4rl_il.py);
  a2c_il    obs 4, ``DiscreteActor`` over ``Net([64, 64])`` (softmax output), 2 actions, batch 64 (test/discrete/test_a2c_with_il.py);
  atari_il  ``DQNet``, 4 x 84 x 84 uint8 stacks, 6 actions, batch 32, a 100k-slot mirrored buffer (examples/offline/atari_il.py).
Device and eager updates alternate; each number is the median wall time of ``--reps`` updates of each (with min and max) after
three warm-up updates of each, with a device synchronise inside the timed region.  ``launches`` counts the kernel launches of
one device update through the project's library.  Prints the card's name, power limit and max SM clock, read in the same run
(query only).  Fails without a CUDA device.
"""
from __future__ import annotations

import argparse
import copy
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DEV = "cuda:0"


class _Discrete:
    def __init__(self, n: int) -> None:
        self.n = n
        self.shape = ()


class _Box:
    def __init__(self, dim: int, m: float) -> None:
        self.shape = (dim,)
        self.low, self.high = -m * np.ones(dim, np.float32), m * np.ones(dim, np.float32)


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return {"name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip()}


def _setup(workload: str):
    from tianshou_b200.algorithm import AdamOptimizerFactory
    from tianshou_b200.algorithm.imitation import ImitationPolicy, OfflineImitationLearning, OffPolicyImitationLearning
    from tianshou_b200.data import Batch, VectorReplayBuffer
    from tianshou_b200.env.atari.atari_network import DQNet
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.continuous import ContinuousActorDeterministic
    from tianshou_b200.utils.net.discrete import DiscreteActor
    torch.manual_seed(0)
    rng = np.random.default_rng(0)
    if workload == "d4rl_il":
        B, E, size, lr = 256, 10, 100_000, 1e-4
        actor = ContinuousActorDeterministic(preprocess_net=Net(state_shape=(17,), action_shape=(6,), hidden_sizes=[256, 256]),
                                             action_shape=(6,), max_action=1.0).to(DEV)
        space, Algo = _Box(6, 1.0), OfflineImitationLearning
        buf = VectorReplayBuffer(size, E, device=DEV, device_mirror=True)
        for _ in range(size // E):
            o = rng.standard_normal((E, 17)).astype(np.float32)
            buf.add(Batch(obs=o, act=rng.uniform(-1, 1, (E, 6)).astype(np.float32), rew=rng.standard_normal(E),
                          terminated=rng.random(E) < 0.001, truncated=np.zeros(E, bool), obs_next=o), buffer_ids=np.arange(E))
    elif workload == "a2c_il":
        B, E, size, lr = 64, 16, 20_000, 1e-3
        actor = DiscreteActor(preprocess_net=Net(state_shape=(4,), hidden_sizes=[64, 64]), action_shape=2).to(DEV)
        space, Algo = _Discrete(2), OffPolicyImitationLearning
        buf = VectorReplayBuffer(size, E, device=DEV)
        for _ in range(size // E):
            o = rng.standard_normal((E, 4)).astype(np.float32)
            buf.add(Batch(obs=o, act=rng.integers(0, 2, E), rew=rng.standard_normal(E), terminated=rng.random(E) < 0.02,
                          truncated=np.zeros(E, bool), obs_next=o), buffer_ids=np.arange(E))
    else:
        B, E, size, lr = 32, 10, 100_000, 1e-4
        actor = DQNet(c=4, h=84, w=84, action_shape=6).to(DEV)
        space, Algo = _Discrete(6), OfflineImitationLearning
        buf = VectorReplayBuffer(size, E, stack_num=4, ignore_obs_next=True, save_only_last_obs=True, device=DEV, device_mirror=True)
        for _ in range(size // E):
            st = np.repeat(rng.integers(0, 256, (E, 1, 84, 84), dtype=np.uint8), 4, axis=1)
            buf.add(Batch(obs=st, act=rng.integers(0, 6, E), rew=rng.standard_normal(E), terminated=rng.random(E) < 0.01,
                          truncated=np.zeros(E, bool), obs_next=st), buffer_ids=np.arange(E))
    ref = copy.deepcopy(actor)
    opt = torch.optim.Adam(ref.parameters(), lr=lr)
    algo = Algo(policy=ImitationPolicy(actor=actor, action_space=space), optim=AdamOptimizerFactory(lr=lr))
    continuous = workload == "d4rl_il"

    def eager(idx: np.ndarray) -> float:
        batch = buf[idx]
        out = ref(batch.obs)[0]
        if continuous:
            loss = F.mse_loss(out, torch.as_tensor(batch.act, dtype=torch.float32, device=DEV))
        else:
            loss = F.nll_loss(F.log_softmax(out, dim=-1), torch.as_tensor(batch.act, dtype=torch.long, device=DEV))
        opt.zero_grad()
        loss.backward()
        opt.step()
        return float(loss.item())

    return algo, buf, eager, B


def run(workload: str, reps: int, warmup: int = 3) -> dict:
    from tianshou_b200 import _cabi
    from tianshou_b200.utils import policy_within_training_step
    algo, buf, eager, B = _setup(workload)
    launches = []

    def device_update():
        _cabi.reset_launch_count()
        with policy_within_training_step(algo.policy):
            algo.update(buffer=buf, sample_size=B)
        launches.append(_cabi.launch_count())

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
    return {"workload": workload, "batch": B, "reps": reps, "device_ms": d, "eager_ms": e, "speedup": e / d,
            "launches": int(np.median(launches)), "device_all_ms": times["device"], "eager_all_ms": times["eager"]}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=21)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/imitation_timing.py needs a CUDA device: a time measured anywhere else says nothing")
    out = {"card": card(), "results": [run(w, args.reps) for w in ("d4rl_il", "a2c_il", "atari_il")]}
    print(json.dumps(out["card"]))
    for r in out["results"]:
        print(f"{r['workload']:10s} device {r['device_ms']:8.3f} ms ({min(r['device_all_ms']):.3f} - {max(r['device_all_ms']):.3f})"
              f"   eager {r['eager_ms']:8.3f} ms ({min(r['eager_all_ms']):.3f} - {max(r['eager_all_ms']):.3f})   x{r['speedup']:.2f}"
              f"   {r['launches']} launches per device update")
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
