"""Time ``REDQ.update()`` on one GPU next to the eager-PyTorch restatement of the reference's update (oracle/oracle_redq.py) on
the same GPU, the same buffer and the same initial weights, alternating update by update; and one ensemble layer alone, as one
``ts_net_gemm_batched`` launch against E separate ``ts_net_gemm`` launches.

    python tools/redq_timing.py [--reps 41] [--out timing.json]

Workloads (fixed alpha 0.2, n = 1, a 100k-transition ``from_data`` buffer with the device mirror on):
  ``test_redq``   : test/continuous/test_redq.py -- obs 3, 1 action, hidden [64, 64], E 4, subset 2, batch 64, actor_delay 3
  ``mujoco_redq`` : examples/mujoco/mujoco_redq.py on Ant-v4 -- obs 27, 8 actions, hidden [256, 256], E 10, subset 2, batch 256,
                    actor_delay 20
Each update number is the median wall time of ``--reps`` updates (critic-only and actor-step updates mixed as the schedule
has them) after four warm-up updates, with a device synchronise inside the timed region, and its 10th-90th percentile range.
The eager update includes the index draw, the host n-step return (as the reference computes it) and the upload of the sampled
rows.  The layer timing is the median of CUDA-event times of 200 repetitions of each of the layer's three GEMMs (forward,
input gradient, weight gradient) at the mujoco_redq.py shape.  Prints the card name, power limit and max SM clock with the
numbers.  Needs a CUDA device.
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
WORKLOADS = {"test_redq": dict(O=3, A=1, H=(64, 64), E=4, M=2, B=64, delay=3),
             "mujoco_redq": dict(O=27, A=8, H=(256, 256), E=10, M=2, B=256, delay=20)}


class _Box:
    def __init__(self, dim: int) -> None:
        self.shape = (dim,)
        self.low = -np.ones(dim, np.float32)
        self.high = np.ones(dim, np.float32)


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return {"name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip()}


def run(name: str, reps: int) -> dict:
    from oracle.oracle_redq import FixedAlpha, RedqNets, redq_update
    from tianshou_b200.algorithm import REDQ, AdamOptimizerFactory, REDQPolicy
    from tianshou_b200.data import ReplayBuffer
    from tianshou_b200.utils import policy_within_training_step
    from tianshou_b200.utils.net.common import EnsembleLinear, Net
    from tianshou_b200.utils.net.continuous import ContinuousActorProbabilistic, ContinuousCritic
    w = WORKLOADS[name]
    O, A, H, E, M, B, delay, N = w["O"], w["A"], w["H"], w["E"], w["M"], w["B"], w["delay"], 100_000
    rng = np.random.default_rng(0)
    term = rng.random(N) < 1e-3
    trunc = np.zeros(N, bool)
    trunc[999::1000] = True
    trunc &= ~term
    data = (rng.standard_normal((N, O)).astype(np.float32), np.tanh(rng.standard_normal((N, A))).astype(np.float32),
            rng.standard_normal(N), term, trunc, term | trunc, rng.standard_normal((N, O)).astype(np.float32))
    torch.manual_seed(0)
    actor = ContinuousActorProbabilistic(preprocess_net=Net(state_shape=(O,), hidden_sizes=H), action_shape=(A,), unbounded=True,
                                         conditioned_sigma=True).to(DEV)
    lin = lambda x, y: EnsembleLinear(E, x, y)
    critic = ContinuousCritic(preprocess_net=Net(state_shape=(O,), action_shape=(A,), hidden_sizes=H, concat=True, linear_layer=lin),
                              linear_layer=lin, flatten_input=False).to(DEV)
    nets = RedqNets(O, A, H, E)
    with torch.no_grad():
        for dst, src in ((nets.actor, actor), (nets.critic, critic), (nets.critic_old, critic)):
            for p, q in zip(dst.parameters(), src.parameters(), strict=True):
                p.copy_(q.detach().cpu())
    algo = REDQ(policy=REDQPolicy(actor=actor, action_space=_Box(A)), policy_optim=AdamOptimizerFactory(lr=3e-4), critic=critic,
                critic_optim=AdamOptimizerFactory(lr=3e-4), ensemble_size=E, subset_size=M, actor_delay=delay)
    buf = ReplayBuffer.from_data(*data)
    buf.enable_device_mirror()
    buf.sync_device_mirror()
    for m in nets.modules():
        m.to(DEV)
    opts = [torch.optim.Adam(nets.actor.parameters(), lr=3e-4), torch.optim.Adam(nets.critic.parameters(), lr=3e-4)]
    host = {k: np.asarray(v) for k, v in zip(("obs", "act", "rew", "terminated", "truncated", "done", "obs_next"), data, strict=True)}
    host.update(offset=np.array([0, N]), last_index=np.asarray(buf.last_index), lengths=np.array([N]),
                unfinished=[] if host["done"][N - 1] else [N - 1])
    eager_rs = np.random.RandomState(1)
    eager_cnt = [0]
    alpha = FixedAlpha(0.2)

    def device_update():
        with policy_within_training_step(algo.policy):
            algo.update(buf, B)

    def eager_update():
        idx = eager_rs.choice(N, B)
        subset = eager_rs.choice(E, M, replace=False)
        eager_cnt[0] += 1
        r = redq_update(nets, opts, alpha, host, idx, lambda shape: torch.randn(shape, device=DEV), subset, gamma=0.99, n_step=1,
                        tau=0.005, target_mode="min", actor_step=eager_cnt[0] % delay == 0)
        float(r["critic_loss"])

    for _ in range(4):
        device_update()
        eager_update()
    torch.cuda.synchronize()
    times = {"device": [], "eager": []}
    for _ in range(reps):
        for kind, fn in (("device", device_update), ("eager", eager_update)):
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            times[kind].append((time.perf_counter() - t0) * 1e3)
    pct = lambda x: [float(np.percentile(x, 10)), float(np.percentile(x, 90))]
    out = {"workload": name, **{k: (list(v) if isinstance(v, tuple) else v) for k, v in w.items()}}
    out.update(device_ms=float(np.median(times["device"])), device_p10_p90=pct(times["device"]),
               eager_ms=float(np.median(times["eager"])), eager_p10_p90=pct(times["eager"]),
               speedup=float(np.median(times["eager"]) / np.median(times["device"])))
    return out


def layer_timing(E: int = 10, rows: int = 256, d_in: int = 256, d_out: int = 256, reps: int = 200) -> dict:
    """One hidden ensemble layer of mujoco_redq.py: the batched launch against E ts_net_gemm launches, per GEMM kind."""
    from tianshou_b200._cabi import call, load_library, ptr, stream_ptr
    lib = load_library()
    st = stream_ptr(torch.device(DEV))
    x, w = torch.randn(E, rows, d_in, device=DEV), torch.randn(E, d_in, d_out, device=DEV)
    dz, y = torch.randn(E, rows, d_out, device=DEV), torch.empty(E, rows, max(d_in, d_out), device=DEV)
    gw = torch.empty(E, d_in, d_out, device=DEV)
    # (A, lda, a_mn, stride_a, B, ldb, b_mn, C, ldc, stride_c, M, N, K): forward, input gradient, weight gradient
    kinds = {"forward": (x, d_in, 0, rows * d_in, w, d_out, 1, y, d_out, rows * d_out, rows, d_out, d_in),
             "input_grad": (dz, d_out, 0, rows * d_out, w, d_out, 0, y, d_in, rows * d_in, rows, d_in, d_out),
             "weight_grad": (x, d_in, 1, rows * d_in, dz, d_out, 1, gw, d_out, d_in * d_out, d_in, d_out, rows)}
    ws = torch.empty(int(lib.ts_net_gemm_batched_workspace_floats(E, 512, 512, 512)) + E * 512 * 512, device=DEV)
    out = {}
    for kind, (a, lda, amn, sa, b, ldb, bmn, c, ldc, sc, M_, N_, K_) in kinds.items():
        sb = d_in * d_out
        nb = int(lib.ts_net_gemm_batched_workspace_floats(E, M_, N_, K_))
        n1 = int(lib.ts_net_gemm_workspace_floats(M_, N_, K_))

        def batched():
            call("ts_net_gemm_batched", E, ptr(a), lda, amn, sa, ptr(b), ldb, bmn, sb, ptr(c), ldc, sc, M_, N_, K_, None, 0, 0, None, 0,
                 0, 1, 0, ptr(ws) if nb else None, nb, st)

        def separate():
            for e in range(E):
                call("ts_net_gemm", a.data_ptr() + 4 * e * sa, lda, amn, b.data_ptr() + 4 * e * sb, ldb, bmn,
                     c.data_ptr() + 4 * e * sc, ldc, M_, N_, K_, None, 0, None, 0, 1, 0, ptr(ws) if n1 else None, n1, st)

        res = {}
        for label, fn in (("batched_us", batched), ("separate_us", separate)):
            for _ in range(10):
                fn()
            ts = []
            for _ in range(reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                fn()
                e1.record()
                e1.synchronize()
                ts.append(e0.elapsed_time(e1) * 1e3)
            res[label] = float(np.median(ts))
        res["speedup"] = res["separate_us"] / res["batched_us"]
        out[kind] = res
    return {"E": E, "rows": rows, "in": d_in, "out": d_out, **out}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=41)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    out = {"card": card(), "results": [run(w, args.reps) for w in WORKLOADS], "layer": layer_timing()}
    print(json.dumps(out["card"]))
    for r in out["results"]:
        print(f"{r['workload']:12s} device {r['device_ms']:8.3f} ms (p10-p90 {r['device_p10_p90'][0]:.3f}-{r['device_p10_p90'][1]:.3f})"
              f"   eager {r['eager_ms']:8.3f} ms (p10-p90 {r['eager_p10_p90'][0]:.3f}-{r['eager_p10_p90'][1]:.3f})   x{r['speedup']:.2f}")
    for kind in ("forward", "input_grad", "weight_grad"):
        x = out["layer"][kind]
        print(f"layer E10 256x256 rows 256 {kind:11s} batched {x['batched_us']:7.1f} us   10 x ts_net_gemm {x['separate_us']:7.1f} us"
              f"   x{x['speedup']:.2f}")
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
