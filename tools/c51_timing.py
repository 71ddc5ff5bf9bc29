"""Time ``C51.update()`` on one GPU next to the same update in eager PyTorch (oracle/oracle_c51.py ``c51_update_torch``: the
reference's projection and loss expressions, autograd and torch's Adam) on the same GPU, the same buffer and the same initial
weights, in the same call; and ``ts_c51_rows`` alone.

    python tools/c51_timing.py [--reps 21] [--launches 2000] [--out timing.json]

Workloads:
  cartpole_c51 : the test_c51.py shape -- obs 4, 2 actions, ``Net(softmax=True)`` [128] * 4, 51 atoms, batch 64, 3-step returns,
                 target_update_freq 320, a uniform 20000-slot buffer of 10 environments with stored obs_next.
  atari_c51    : the atari_c51.py shape -- ``C51Net`` behind ScaledObsInputActionReprNet, 4 x 84 x 84 uint8 stacks, 6 actions,
                 51 atoms, batch 32, 3-step returns, target_update_freq 500, a 100k-slot buffer of single frames (stack_num 4)
                 with the device mirror on.
Device and eager updates alternate; each number is the median wall time of ``--reps`` updates of each (with min and max) after
three warm-up updates of each, with a device synchronise inside the timed region.  The eager update includes what the
reference's update does on the host: the index draw, the frame-stack gather, the upload and the host n-step return.
``ts_c51_rows`` at B 32, A 6, N 51 is timed with CUDA events around ``--launches`` back-to-back launches.
Prints the card's name, power limit and max SM clock, read in the same run (query only).  Fails without a CUDA device.
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
    from oracle import oracle_c51 as oc
    from oracle import oracle_discrete_sac as ods
    from tianshou_b200.algorithm import C51, AdamOptimizerFactory, C51Policy
    from tianshou_b200.data import Batch, VectorReplayBuffer
    from tianshou_b200.env.atari import C51Net, ScaledObsInputActionReprNet
    from tianshou_b200.utils.net.common import Net
    torch.manual_seed(0)
    rng = np.random.default_rng(0)
    N = N_ATOMS
    if workload == "cartpole_c51":
        A, E, size, B, n_step, freq, lr, gamma = 2, 10, 20000, 64, 3, 320, 1e-3, 0.9
        model = Net(state_shape=(4,), action_shape=A, hidden_sizes=(128,) * 4, softmax=True, num_atoms=N).to(DEV)
        ref = oc.categorical_net("mlp", A, N, obs=4, hidden=(128,) * 4)
        buf = VectorReplayBuffer(size, E, device=DEV)
        for _ in range(size // E):
            buf.add(Batch(obs=rng.standard_normal((E, 4)).astype(np.float32), act=rng.integers(0, A, E), rew=rng.standard_normal(E),
                          terminated=rng.random(E) < 0.02, truncated=np.zeros(E, bool),
                          obs_next=rng.standard_normal((E, 4)).astype(np.float32)), buffer_ids=np.arange(E))
    else:
        A, E, size, B, n_step, freq, lr, gamma = 6, 10, 100_000, 32, 3, 500, 1e-4, 0.99
        model = ScaledObsInputActionReprNet(C51Net(c=4, h=84, w=84, action_shape=A, num_atoms=N)).to(DEV)
        ref = oc.categorical_net("cnn", A, N, H=84, W=84)
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
    algo = C51(policy=policy, optim=AdamOptimizerFactory(lr=lr), gamma=gamma, n_step_return_horizon=n_step, target_update_freq=freq)
    view = dict(obs=np.asarray(buf.obs), act=np.asarray(buf.act), rew=np.asarray(buf.rew), done=np.asarray(buf.done),
                terminated=np.asarray(buf.terminated), offset=np.asarray(buf._extend_offset), last_index=buf.last_index,
                lengths=buf._sizes)
    if workload == "cartpole_c51":
        view["obs_next"] = np.asarray(buf.obs_next)
        obs_of = ods.flat_obs(view["obs"], DEV)
    else:
        obs_of = ods.frame_obs(view, 4, 255.0, DEV)
    state = oc.C51State(ref, lr, freq, V_MIN, V_MAX)
    eager = lambda idx: oc.c51_update_torch(state, obs_of, view, idx, gamma, n_step)
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
    d, e = float(np.median(times["device"])), float(np.median(times["eager"]))
    return {"workload": workload, "batch": B, "reps": reps, "device_ms": d, "eager_ms": e, "speedup": e / d,
            "device_all_ms": times["device"], "eager_all_ms": times["eager"]}


def rows_kernel(launches: int, B: int = 32, A: int = 6, N: int = N_ATOMS) -> dict:
    """``ts_c51_rows`` alone: mean time per launch over ``launches`` back-to-back launches between two CUDA events."""
    from oracle import oracle_c51 as oc
    from tianshou_b200._cabi import call, ptr, stream_ptr
    g = torch.Generator(device="cpu").manual_seed(0)
    logits = (torch.randn(B, A, N, generator=g) * 2).to(DEV)
    act = torch.randint(0, A, (B,), generator=g).to(DEV)
    ret = (torch.randn(B, N, generator=g) * 8).to(DEV)
    z = torch.as_tensor(oc.support(N, V_MIN, V_MAX), device=DEV)
    nd = torch.randn(B, N, generator=g).softmax(-1).to(DEV)
    dl, prio, rows, losses = (torch.empty(B, A, N, device=DEV), torch.empty(B, device=DEV), torch.empty(3, B, device=DEV),
                              torch.empty(4, device=DEV))
    st = stream_ptr(torch.device(DEV))
    dz = (V_MAX - V_MIN) / (N - 1)
    args = (ptr(logits), ptr(act), ptr(ret), ptr(z), V_MIN, V_MAX, dz, ptr(nd), None, B, A, N, ptr(dl), ptr(prio), ptr(rows),
            ptr(losses), st)
    for _ in range(50):
        call("ts_c51_rows", *args)
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(launches):
        call("ts_c51_rows", *args)
    t1.record()
    torch.cuda.synchronize()
    return {"B": B, "A": A, "N": N, "launches": launches, "us_per_call": t0.elapsed_time(t1) * 1e3 / launches}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=21)
    ap.add_argument("--launches", type=int, default=2000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/c51_timing.py needs a CUDA device: a time measured anywhere else says nothing")
    out = {"card": card(), "results": [run(w, args.reps) for w in ("cartpole_c51", "atari_c51")],
           "rows_kernel": rows_kernel(args.launches)}
    print(json.dumps(out["card"]))
    for r in out["results"]:
        print(f"{r['workload']:13s} device {r['device_ms']:8.3f} ms ({min(r['device_all_ms']):.3f} - {max(r['device_all_ms']):.3f})"
              f"   eager {r['eager_ms']:8.3f} ms ({min(r['eager_all_ms']):.3f} - {max(r['eager_all_ms']):.3f})   x{r['speedup']:.2f}")
    r = out["rows_kernel"]
    print(f"ts_c51_rows B {r['B']} A {r['A']} N {r['N']}: {r['us_per_call']:.2f} us per call (mean of {r['launches']} launches)")
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
