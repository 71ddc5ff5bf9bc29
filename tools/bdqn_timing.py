"""Time ``BDQN.update()`` on one GPU next to the eager-PyTorch restatement of the reference's update (oracle/oracle_bdqn.py) on the
same GPU, the same buffer and the same initial weights, alternating update by update; and one branch layer alone, as one
``ts_net_gemm_batched`` launch against num_branches separate ``ts_net_gemm`` launches.

    python tools/bdqn_timing.py [--reps 41] [--out timing.json]

Workloads (double Q with a lagged network, a 100k-transition ``from_data`` buffer with the device mirror on):
  ``test_bdqn``   : test/discrete/test_bdqn.py on Pendulum-v1 -- obs 3, 1 branch of 40 actions, common [64, 64], value [64],
                    action [64], batch 128, target_update_freq 200
  ``bipedal_bdq`` : examples/box2d/bipedal_bdq.py on BipedalWalker-v3 -- obs 24, 4 branches of 25 actions, common [512, 256],
                    value [128], action [128], batch 512, target_update_freq 1000
Each update number is the median wall time of ``--reps`` updates after four warm-up updates, with a device synchronise inside the
timed region, and its 10th-90th percentile range.  The eager update includes the index draw, the numpy target (as the reference
computes it) and the upload of the sampled rows.  The layer timing is the median of CUDA-event times of 200 repetitions of each of
the layer's three GEMMs (forward, input gradient, weight gradient) at bipedal_bdq.py's first branch layer (4 branches, 512 rows,
256 -> 128, the trunk output shared).  Prints the card name, power limit and max SM clock with the numbers.  Needs a CUDA device.
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
WORKLOADS = {"test_bdqn": dict(O=3, nb=1, A=40, common=(64, 64), value=(64,), action=(64,), B=128, freq=200),
             "bipedal_bdq": dict(O=24, nb=4, A=25, common=(512, 256), value=(128,), action=(128,), B=512, freq=1000)}


class _MultiDiscrete:
    def __init__(self, nvec) -> None:
        self.nvec = np.asarray(nvec)
        self.shape = self.nvec.shape


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return {"name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip()}


def run(name: str, reps: int) -> dict:
    from oracle.oracle_bdqn import bdqn_update
    from tianshou_b200.algorithm import BDQN, AdamOptimizerFactory, BDQNPolicy
    from tianshou_b200.data import ReplayBuffer
    from tianshou_b200.utils import policy_within_training_step
    from tianshou_b200.utils.net.common import BranchingNet
    w = WORKLOADS[name]
    O, nb, A, B, freq, N = w["O"], w["nb"], w["A"], w["B"], w["freq"], 100_000
    rng = np.random.default_rng(0)
    term = rng.random(N) < 1e-3
    trunc = np.zeros(N, bool)
    trunc[999::1000] = True
    trunc &= ~term
    data = (rng.standard_normal((N, O)).astype(np.float32), rng.integers(0, A, (N, nb)), rng.standard_normal(N), term, trunc,
            term | trunc, rng.standard_normal((N, O)).astype(np.float32))
    torch.manual_seed(0)
    net = BranchingNet(state_shape=(O,), num_branches=nb, action_per_branch=A, common_hidden_sizes=list(w["common"]),
                       value_hidden_sizes=list(w["value"]), action_hidden_sizes=list(w["action"])).to(DEV)
    eager_net = copy.deepcopy(net)
    eager_old = copy.deepcopy(net)
    algo = BDQN(policy=BDQNPolicy(model=net, action_space=_MultiDiscrete([A] * nb)), optim=AdamOptimizerFactory(lr=1e-4),
                target_update_freq=freq)
    buf = ReplayBuffer.from_data(*data)
    buf.enable_device_mirror()
    buf.sync_device_mirror()
    opt = torch.optim.Adam(eager_net.parameters(), lr=1e-4)
    host = {k: np.asarray(v) for k, v in zip(("obs", "act", "rew", "terminated", "truncated", "done", "obs_next"), data, strict=True)}
    end = host["done"].copy()
    end[N - 1] = True                   # done, or the buffer's one unfinished episode
    eager_rs = np.random.RandomState(1)
    eager_cnt = [0]

    def device_update():
        with policy_within_training_step(algo.policy):
            algo.update(buf, B)

    def eager_update():
        idx = eager_rs.choice(N, B)
        r = bdqn_update(eager_net, opt, eager_old, host, end, idx, is_double=True, refresh=eager_cnt[0] % freq == 0)
        eager_cnt[0] += 1
        float(r["loss"])

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


def layer_timing(nb: int = 4, rows: int = 512, d_in: int = 256, d_out: int = 128, reps: int = 200) -> dict:
    """bipedal_bdq.py's first branch layer: the batched launch (the trunk output shared at stride 0, nn.Linear [out, in] weights)
    against nb ts_net_gemm launches, per GEMM kind."""
    from tianshou_b200._cabi import call, load_library, ptr, stream_ptr
    lib = load_library()
    st = stream_ptr(torch.device(DEV))
    x, w = torch.randn(rows, d_in, device=DEV), torch.randn(nb, d_out, d_in, device=DEV)
    dz, y = torch.randn(nb, rows, d_out, device=DEV), torch.empty(nb, rows, max(d_in, d_out), device=DEV)
    gw = torch.empty(nb, d_out, d_in, device=DEV)
    sw = d_in * d_out
    # (A, lda, a_mn, stride_a, B, ldb, b_mn, stride_b, C, ldc, stride_c, M, N, K): forward, input gradient, weight gradient
    kinds = {"forward": (x, d_in, 0, 0, w, d_in, 0, sw, y, d_out, rows * d_out, rows, d_out, d_in),
             "input_grad": (dz, d_out, 0, rows * d_out, w, d_in, 1, sw, y, d_in, rows * d_in, rows, d_in, d_out),
             "weight_grad": (dz, d_out, 1, rows * d_out, x, d_in, 1, 0, gw, d_in, sw, d_out, d_in, rows)}
    ws = torch.empty(int(lib.ts_net_gemm_batched_workspace_floats(nb, 512, 512, 512)) + nb * 512 * 512, device=DEV)
    out = {}
    for kind, (a, lda, amn, sa, b, ldb, bmn, sb, c, ldc, sc, M_, N_, K_) in kinds.items():
        n_b = int(lib.ts_net_gemm_batched_workspace_floats(nb, M_, N_, K_))
        n1 = int(lib.ts_net_gemm_workspace_floats(M_, N_, K_))

        def batched():
            call("ts_net_gemm_batched", nb, ptr(a), lda, amn, sa, ptr(b), ldb, bmn, sb, ptr(c), ldc, sc, M_, N_, K_, None, 0, 0, None, 0,
                 0, 1, 0, ptr(ws) if n_b else None, n_b, st)

        def separate():
            for e in range(nb):
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
    return {"branches": nb, "rows": rows, "in": d_in, "out": d_out, **out}


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
        print(f"branch layer nb4 256->128 rows 512 {kind:11s} batched {x['batched_us']:7.1f} us   4 x ts_net_gemm "
              f"{x['separate_us']:7.1f} us   x{x['speedup']:.2f}")
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
