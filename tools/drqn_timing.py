"""Time ``DQN.update()`` with a ``Recurrent`` model (DRQN) on one GPU next to the same update in eager PyTorch (the reference's
network with cuDNN's LSTM, the stacked batch read on the host as the reference's buffer reads it, the reference's loss, autograd
and torch's Adam) on the same GPU, the same buffer and the same initial weights, in the same call.

    python tools/drqn_timing.py [--reps 21] [--out timing.json]

Workload: the test_drqn.py shape -- obs 4, 2 actions, ``Recurrent(layer_num=2, hidden 128)``, a 20000-slot buffer of 16
environments with ``stack_num=4`` and ``ignore_obs_next=True``, batch 128, 3-step returns, gamma 0.95, target_update_freq 320.
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

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DEV = "cuda:0"
A, E, SIZE, B, S, N_STEP, FREQ, LR, GAMMA = 2, 16, 20000, 128, 4, 3, 320, 1e-3, 0.95


class _Discrete:
    def __init__(self, n: int) -> None:
        self.n = n
        self.shape = ()


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return {"name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip()}


def _setup():
    from oracle.oracle_offpolicy import compute_nstep_targets, next_index, stacked_obs
    from tianshou_b200.algorithm import DQN, AdamOptimizerFactory
    from tianshou_b200.algorithm.modelfree.dqn import DiscreteQLearningPolicy
    from tianshou_b200.data import Batch, VectorReplayBuffer
    from tianshou_b200.utils.net.common import Recurrent
    torch.manual_seed(0)
    rng = np.random.default_rng(0)
    model = Recurrent(layer_num=2, state_shape=4, action_shape=A).to(DEV)
    ref = copy.deepcopy(model)
    ref_old = copy.deepcopy(model)
    opt = torch.optim.Adam(ref.parameters(), lr=LR)
    algo = DQN(policy=DiscreteQLearningPolicy(model=model, action_space=_Discrete(A)), optim=AdamOptimizerFactory(lr=LR),
               gamma=GAMMA, n_step_return_horizon=N_STEP, target_update_freq=FREQ)
    buf = VectorReplayBuffer(SIZE, E, stack_num=S, ignore_obs_next=True, device=DEV)
    for _ in range(SIZE // E):
        o = rng.standard_normal((E, 4)).astype(np.float32)
        buf.add(Batch(obs=o, act=rng.integers(0, A, E), rew=rng.standard_normal(E), terminated=rng.random(E) < 0.02,
                      truncated=np.zeros(E, bool), obs_next=o), buffer_ids=np.arange(E))
    view = dict(obs=np.asarray(buf.obs), act=np.asarray(buf.act), rew=np.asarray(buf.rew), done=np.asarray(buf.done),
                terminated=np.asarray(buf.terminated), offset=np.asarray(buf._extend_offset), last_index=buf.last_index,
                lengths=buf._sizes)
    read = lambda idx: torch.as_tensor(stacked_obs(view["obs"], idx, view, S), device=DEV)
    it = [0]

    def eager(idx: np.ndarray) -> float:
        def target_q(terminal: np.ndarray) -> torch.Tensor:
            x = read(next_index(terminal, view["offset"], view["done"], view["last_index"], view["lengths"]))
            q_on, q_old = ref(x)[0], ref_old(x)[0]
            return q_old[torch.arange(len(terminal), device=DEV), q_on.argmax(dim=1)].cpu()

        returns = torch.as_tensor(compute_nstep_targets(view, idx, target_q, GAMMA, N_STEP), device=DEV).flatten()
        if it[0] % FREQ == 0:
            ref_old.load_state_dict(ref.state_dict())
        it[0] += 1
        q = ref(read(idx))[0][torch.arange(len(idx), device=DEV), torch.as_tensor(view["act"][idx], device=DEV)]
        loss = (returns - q).pow(2).mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
        return float(loss.item())

    return algo, buf, eager


def run(reps: int, warmup: int = 3) -> dict:
    from tianshou_b200 import _cabi
    from tianshou_b200.utils import policy_within_training_step
    algo, buf, eager = _setup()
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
    return {"workload": "test_drqn", "batch": B, "reps": reps, "device_ms": d, "eager_ms": e, "speedup": e / d,
            "launches": int(np.median(launches)), "device_all_ms": times["device"], "eager_all_ms": times["eager"]}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=21)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/drqn_timing.py needs a CUDA device: a time measured anywhere else says nothing")
    out = {"card": card(), "results": [run(args.reps)]}
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
