"""Time ``RainbowDQN.update()`` on one GPU next to the same update in eager PyTorch (oracle/oracle_rainbow.py
``rainbow_update_torch``: torch's noise draws, the reference's dueling, projection and loss expressions, autograd and torch's
Adam) on the same GPU, the same buffer and the same initial weights, in the same call; and the noise draws alone.

    python tools/rainbow_timing.py [--reps 21] [--out timing.json]

Workloads:
  cartpole_rainbow : the test_rainbow.py shape -- obs 4, 2 actions, ``Net(softmax=True, num_atoms=51)`` [128] * 4 with noisy
                     dueling heads (``noisy_std`` 0.1), batch 64, 3-step returns, target_update_freq 320, a uniform 20000-slot
                     buffer of 10 environments with stored obs_next.
  atari_rainbow    : the atari_rainbow.py shape -- ``RainbowNet`` (noisy, dueling) behind ScaledObsInputActionReprNet, 4 x 84 x 84
                     uint8 stacks, 6 actions, 51 atoms, batch 32, 3-step returns, target_update_freq 500, a 100k-slot buffer of
                     single frames (stack_num 4) with the device mirror on.
Device and eager updates alternate; each number is the median wall time of ``--reps`` updates of each (with min and max) after
three warm-up updates of each, with a device synchronise inside the timed region.  ``noise_ms`` is the median time of the device
update's two ``_sample_noise`` calls (online and lagged network, torch's ``randn`` per noisy layer), synchronised, measured
apart from the updates.  Prints the card's name, power limit and max SM clock, read in the same run (query only).  Fails
without a CUDA device.
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
N_ATOMS, V_MIN, V_MAX = 51, -10.0, 10.0


class _Discrete:
    def __init__(self, n: int) -> None:
        self.n = n
        self.shape = ()


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return {"name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip()}


def _setup(workload: str):
    from oracle import oracle_discrete_sac as ods
    from oracle import oracle_rainbow as orb
    from tianshou_b200.algorithm import AdamOptimizerFactory, C51Policy, RainbowDQN
    from tianshou_b200.data import Batch, VectorReplayBuffer
    from tianshou_b200.env.atari import RainbowNet, ScaledObsInputActionReprNet
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.discrete import NoisyLinear
    torch.manual_seed(0)
    rng = np.random.default_rng(0)
    N = N_ATOMS
    if workload == "cartpole_rainbow":
        A, E, size, B, n_step, freq, lr, gamma = 2, 10, 20000, 64, 3, 320, 1e-3, 0.99

        def noisy(x: int, y: int) -> NoisyLinear:
            return NoisyLinear(x, y, 0.1)

        model = Net(state_shape=(4,), action_shape=A, hidden_sizes=(128,) * 4, softmax=True, num_atoms=N,
                    dueling_param=({"linear_layer": noisy}, {"linear_layer": noisy})).to(DEV)
        ref = orb.rainbow_net(dict(kind="mlp", obs=4, hidden=(128,) * 4, q_hidden=(), v_hidden=(), trunk_noisy=False, v_noisy=True,
                                   A=A, N=N))
        buf = VectorReplayBuffer(size, E, device=DEV)
        for _ in range(size // E):
            buf.add(Batch(obs=rng.standard_normal((E, 4)).astype(np.float32), act=rng.integers(0, A, E), rew=rng.standard_normal(E),
                          terminated=rng.random(E) < 0.02, truncated=np.zeros(E, bool),
                          obs_next=rng.standard_normal((E, 4)).astype(np.float32)), buffer_ids=np.arange(E))
    else:
        A, E, size, B, n_step, freq, lr, gamma = 6, 10, 100_000, 32, 3, 500, 0.0000625, 0.99
        model = ScaledObsInputActionReprNet(RainbowNet(c=4, h=84, w=84, action_shape=A, num_atoms=N, noisy_std=0.1)).to(DEV)
        ref = orb.rainbow_net(dict(kind="cnn", H=84, W=84, noisy=True, dueling=True, A=A, N=N))
        buf = VectorReplayBuffer(size, E, stack_num=4, ignore_obs_next=True, save_only_last_obs=True, device=DEV, device_mirror=True)
        for _ in range(size // E):
            st = np.repeat(rng.integers(0, 256, (E, 1, 84, 84), dtype=np.uint8), 4, axis=1)
            buf.add(Batch(obs=st, act=rng.integers(0, A, E), rew=rng.standard_normal(E), terminated=rng.random(E) < 0.01,
                          truncated=np.zeros(E, bool), obs_next=st), buffer_ids=np.arange(E))
    ref = ref.to(DEV)
    with torch.no_grad():
        for p, q in zip(model.parameters(), ref.parameters(), strict=True):
            q.copy_(p)
    policy = C51Policy(model=model, action_space=_Discrete(A), num_atoms=N, v_min=V_MIN, v_max=V_MAX)
    algo = RainbowDQN(policy=policy, optim=AdamOptimizerFactory(lr=lr), gamma=gamma, n_step_return_horizon=n_step,
                      target_update_freq=freq)
    view = dict(obs=np.asarray(buf.obs), act=np.asarray(buf.act), rew=np.asarray(buf.rew), done=np.asarray(buf.done),
                terminated=np.asarray(buf.terminated), offset=np.asarray(buf._extend_offset), last_index=buf.last_index,
                lengths=buf._sizes)
    if workload == "cartpole_rainbow":
        view["obs_next"] = np.asarray(buf.obs_next)
        obs_of = ods.flat_obs(view["obs"], DEV)
    else:
        obs_of = ods.frame_obs(view, 4, 255.0, DEV)
    state = orb.RainbowState(ref, lr, freq, V_MIN, V_MAX)
    eager = lambda idx: orb.rainbow_update_torch(state, obs_of, view, idx, gamma, n_step)
    return algo, buf, eager, B


def run(workload: str, reps: int, warmup: int = 3) -> dict:
    from tianshou_b200.utils import policy_within_training_step
    algo, buf, eager, B = _setup(workload)

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
    noise = []
    for i in range(warmup + reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        with torch.no_grad():
            algo._sample_noise(algo.policy.model)
            algo._sample_noise(algo.model_old)
        torch.cuda.synchronize()
        if i >= warmup:
            noise.append((time.perf_counter() - t0) * 1e3)
    d, e = float(np.median(times["device"])), float(np.median(times["eager"]))
    return {"workload": workload, "batch": B, "reps": reps, "device_ms": d, "eager_ms": e, "speedup": e / d,
            "noise_ms": float(np.median(noise)), "device_all_ms": times["device"], "eager_all_ms": times["eager"]}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=21)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/rainbow_timing.py needs a CUDA device: a time measured anywhere else says nothing")
    out = {"card": card(), "results": [run(w, args.reps) for w in ("cartpole_rainbow", "atari_rainbow")]}
    print(json.dumps(out["card"]))
    for r in out["results"]:
        print(f"{r['workload']:16s} device {r['device_ms']:8.3f} ms ({min(r['device_all_ms']):.3f} - {max(r['device_all_ms']):.3f})"
              f"   eager {r['eager_ms']:8.3f} ms ({min(r['eager_all_ms']):.3f} - {max(r['eager_all_ms']):.3f})   x{r['speedup']:.2f}"
              f"   noise draws {r['noise_ms']:.3f} ms")
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
