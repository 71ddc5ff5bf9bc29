"""Time ``FQF.update()`` on one GPU next to the same update in eager PyTorch (oracle/oracle_fqf.py ``fqf_update_torch``: the
reference's fraction proposal, network and loss expressions, autograd, torch's Adam and RMSprop) on the same GPU, the same
buffer and the same initial weights, in the same call; and the parts of one device update's step forward.

    python tools/fqf_timing.py [--reps 21] [--launches 200] [--out timing.json]

Workloads:
  cartpole_fqf : the test_fqf.py shape -- obs 4, 2 actions, trunk ``Net`` [64, 64] to 64, ``last`` [64, 64, 64], 64 cosines,
                 N 32, ent_coef 10, RMSprop on the fractions, batch 64, 3-step returns, target_update_freq 320, a uniform
                 20000-slot buffer of 10 environments with stored obs_next.
  atari_fqf    : the atari_fqf.py shape -- ``DQNet(features_only=True)`` (D = 3136), ``last`` [512], 64 cosines, N 32,
                 ent_coef 10, RMSprop on the fractions, 4 x 84 x 84 uint8 stacks, 6 actions, batch 32, 3-step returns,
                 target_update_freq 500, a 100k-slot buffer of single frames (stack_num 4) with the device mirror on.
Device and eager updates alternate; each number is the median wall time of ``--reps`` updates of each (with min and max) after
three warm-up updates of each, with a device synchronise inside the timed region.  The eager update includes what the
reference's update does on the host: the index draw, the frame-stack gather, the upload and the host n-step return.
The parts (trunk on B rows; fraction net + ``ts_fqf_fractions``; the quantiles at tau_hats on B * N rows; at the inner fractions
on B * (N - 1) rows; ``ts_fqf_fraction_rows``) are timed with CUDA events around ``--launches`` back-to-back runs of each.
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


class _Discrete:
    def __init__(self, n: int) -> None:
        self.n = n
        self.shape = ()


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return {"name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip()}


def _setup(workload: str):
    from oracle import oracle_discrete_bcq as odb
    from oracle import oracle_discrete_sac as ods
    from oracle import oracle_fqf as of
    from oracle import oracle_iqn as oi
    from tianshou_b200.algorithm import FQF, AdamOptimizerFactory, FQFPolicy, RMSpropOptimizerFactory
    from tianshou_b200.data import Batch, VectorReplayBuffer
    from tianshou_b200.env.atari import DQNet
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.discrete import FractionProposalNetwork, FullQuantileFunction
    torch.manual_seed(0)
    rng = np.random.default_rng(0)
    C, N, ent_coef, frac_lr = 64, 32, 10.0, 2.5e-9
    if workload == "cartpole_fqf":
        A, E, size, B, n_step, freq, lr, gamma = 2, 10, 20000, 64, 3, 320, 3e-3, 0.9
        pre, last = Net(state_shape=(4,), action_shape=64, hidden_sizes=(64, 64)), (64, 64, 64)
        trunk, feat = odb.mlp_trunk(4, (64, 64), 64)
        buf = VectorReplayBuffer(size, E, device=DEV)
        for _ in range(size // E):
            buf.add(Batch(obs=rng.standard_normal((E, 4)).astype(np.float32), act=rng.integers(0, A, E), rew=rng.standard_normal(E),
                          terminated=rng.random(E) < 0.02, truncated=np.zeros(E, bool),
                          obs_next=rng.standard_normal((E, 4)).astype(np.float32)), buffer_ids=np.arange(E))
    else:
        A, E, size, B, n_step, freq, lr, gamma = 6, 10, 100_000, 32, 3, 500, 5e-5, 0.99
        pre, last = DQNet(c=4, h=84, w=84, action_shape=A, features_only=True), (512,)
        trunk, feat = odb.cnn_trunk(4, 84, 84)
        buf = VectorReplayBuffer(size, E, stack_num=4, ignore_obs_next=True, save_only_last_obs=True, device=DEV, device_mirror=True)
        for _ in range(size // E):
            st = np.repeat(rng.integers(0, 256, (E, 1, 84, 84), dtype=np.uint8), 4, axis=1)
            buf.add(Batch(obs=st, act=rng.integers(0, A, E), rew=rng.standard_normal(E), terminated=rng.random(E) < 0.01,
                          truncated=np.zeros(E, bool), obs_next=st), buffer_ids=np.arange(E))
    model = FullQuantileFunction(preprocess_net=pre, action_shape=A, hidden_sizes=last, num_cosines=C).to(DEV)
    fm = FractionProposalNetwork(N, model.input_dim).to(DEV)
    ref = oi.IqnNet(trunk(), feat, last, A, C).to(DEV)
    ref_frac = torch.nn.Linear(feat, N).to(DEV)
    with torch.no_grad():
        for p, q in zip(list(model.parameters()) + list(fm.parameters()), list(ref.parameters()) + list(ref_frac.parameters()),
                        strict=True):
            q.copy_(p)
    policy = FQFPolicy(model=model, fraction_model=fm, action_space=_Discrete(A))
    algo = FQF(policy=policy, optim=AdamOptimizerFactory(lr=lr), fraction_optim=RMSpropOptimizerFactory(lr=frac_lr), gamma=gamma,
               num_fractions=N, ent_coef=ent_coef, n_step_return_horizon=n_step, target_update_freq=freq)
    view = dict(obs=np.asarray(buf.obs), act=np.asarray(buf.act), rew=np.asarray(buf.rew), done=np.asarray(buf.done),
                terminated=np.asarray(buf.terminated), offset=np.asarray(buf._extend_offset), last_index=buf.last_index,
                lengths=buf._sizes)
    if workload == "cartpole_fqf":
        view["obs_next"] = np.asarray(buf.obs_next)
        obs_of = ods.flat_obs(view["obs"], DEV)
    else:
        obs_of = ods.frame_obs(view, 4, 1.0, DEV)
    state = of.FqfState(ref, ref_frac, lr, "rmsprop", frac_lr, freq)
    eager = lambda idx: of.fqf_update_torch(state, obs_of, view, idx, gamma, n_step, ent_coef)
    return algo, buf, eager, B


def run(workload: str, reps: int, launches: int, warmup: int = 3) -> dict:
    from tianshou_b200._cabi import call, ptr, stream_ptr
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
    # the parts of the step's forward and loss on one batch, each alone over CUDA events
    idx = buf.sample_indices(B)
    src = algo._obs_source(buf, idx, "obs")
    N, A = algo._n_fractions, algo.n_actions
    st = stream_ptr(torch.device(DEV))
    trunk = algo._trunk.forward(src.x, B, "timing", frames=src.frames)
    fr = algo._propose(trunk[-1], "timing")
    head = algo._quantiles_at(trunk[-1], fr["tau_hats"], N, "timing")[2]
    q_tau = algo._quantiles_at(trunk[-1], fr["inner"], N - 1, "timing_tau")[2][-1]
    act = torch.as_tensor(np.asarray(buf.act)[idx].astype(np.int64), device=DEV)
    dz, rows, losses = algo._buf("timing_dz", (B, N)), algo._buf("timing_rows", (3, B)), algo._buf("timing_losses", 4)

    def fraction_rows():
        call("ts_fqf_fraction_rows", ptr(head[-1]), ptr(q_tau), ptr(act), ptr(fr["taus"]), ptr(fr["p"]), ptr(fr["logp"]),
             ptr(fr["H"]), B, A, N, float(algo.ent_coef), ptr(dz), ptr(rows), ptr(losses), st)

    parts = {}
    for name, fn in (("trunk", lambda: algo._trunk.forward(src.x, B, "timing", frames=src.frames)),
                     ("proposal", lambda: algo._propose(trunk[-1], "timing")),
                     ("quantiles_tau_hats", lambda: algo._quantiles_at(trunk[-1], fr["tau_hats"], N, "timing")),
                     ("quantiles_inner", lambda: algo._quantiles_at(trunk[-1], fr["inner"], N - 1, "timing_tau")),
                     ("fraction_rows", fraction_rows)):
        for _ in range(10):
            fn()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(launches):
            fn()
        t1.record()
        torch.cuda.synchronize()
        parts[name] = t0.elapsed_time(t1) * 1e3 / launches
    return {"workload": workload, "batch": B, "reps": reps, "device_ms": d, "eager_ms": e, "speedup": e / d,
            "device_all_ms": times["device"], "eager_all_ms": times["eager"], "parts_us": parts}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=21)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/fqf_timing.py needs a CUDA device: a time measured anywhere else says nothing")
    out = {"card": card(), "results": [run(w, args.reps, args.launches) for w in ("cartpole_fqf", "atari_fqf")]}
    print(json.dumps(out["card"]))
    for r in out["results"]:
        print(f"{r['workload']:13s} device {r['device_ms']:8.3f} ms ({min(r['device_all_ms']):.3f} - {max(r['device_all_ms']):.3f})"
              f"   eager {r['eager_ms']:8.3f} ms ({min(r['eager_all_ms']):.3f} - {max(r['eager_all_ms']):.3f})   x{r['speedup']:.2f}"
              f"   parts (us): " + ", ".join(f"{k} {v:.1f}" for k, v in r["parts_us"].items()))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
