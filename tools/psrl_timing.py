"""PSRL on the GPU: ``PSRL.update()`` on a full 50,000-transition buffer and ``solve_policy()`` across model sizes, against the
reference's host loops (oracle/oracle_psrl.py restates them) and an eager-PyTorch value iteration on the same GPU.

    python tools/psrl_timing.py [--reps 21] [--out FILE]

Prints the card, its power limit and max SM clock, then medians with min-max of ``--reps`` synchronised calls.  ``solve_policy``
is the two draws + the kernel + the policy readback; the kernel alone is timed with CUDA events.  ``P GB/s`` is the bytes of P
read (n_s^2 n_a 8 per sweep, times the sweeps) over the kernel time, against the H100's 3.35 TB/s of HBM3; P of up to ~50 MB
(the L2's size) stays L2-resident across sweeps.
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

from oracle import oracle_psrl as op  # noqa: E402
from tianshou_b200 import ops  # noqa: E402
from tianshou_b200.algorithm import PSRL  # noqa: E402
from tianshou_b200.algorithm.modelbased.psrl import PSRLPolicy, _solve  # noqa: E402
from tianshou_b200.data import Batch, VectorReplayBuffer  # noqa: E402
from tianshou_b200.utils import policy_within_training_step  # noqa: E402

DEV = "cuda:0"
HBM_TBPS = 3.35


class _Discrete:
    def __init__(self, n):
        self.n, self.shape = n, ()


def stat(ts):
    a = np.asarray(ts) * 1e3
    return {"median_ms": float(np.median(a)), "min_ms": float(a.min()), "max_ms": float(a.max()), "n": len(a)}


def timed(fn, reps):
    out = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        out.append(time.perf_counter() - t0)
    return out


def make(n_s, n_a, gamma=0.99, eps=0.01):
    pol = PSRLPolicy(trans_count_prior=np.ones((n_s, n_a, n_s)), rew_mean_prior=np.zeros((n_s, n_a)),
                     rew_std_prior=np.ones((n_s, n_a)), action_space=_Discrete(n_a), discount_factor=gamma, epsilon=eps, device=DEV)
    return PSRL(policy=pol)


def update_rows(n_s, n_a, reps):
    rng = np.random.default_rng(0)
    E, N = 100, 50_000
    res = {}
    for mirror in (False, True):
        buf = VectorReplayBuffer(N, E, device=DEV, device_mirror=mirror)
        for _ in range(N // E):
            buf.add(Batch(obs=rng.integers(0, n_s, E), act=rng.integers(0, n_a, E), rew=rng.standard_normal(E),
                          terminated=rng.random(E) < 0.01, truncated=np.zeros(E, bool), obs_next=rng.integers(0, n_s, E),
                          info=Batch()), buffer_ids=np.arange(E))
        algo = make(n_s, n_a)
        with policy_within_training_step(algo.policy):
            algo.update(buffer=buf, batch_size=0, repeat=1)                       # warm-up
            res["mirror" if mirror else "upload"] = stat(timed(lambda: algo.update(buffer=buf, batch_size=0, repeat=1), reps))
    b, _ = buf.sample(0)
    perm = np.random.permutation(N)
    host = []
    for _ in range(3):
        t0 = time.perf_counter()
        op.update_rows(n_s, n_a, b.obs, b.act, b.obs_next, b.rew, b.done, perm, False)
        host.append(time.perf_counter() - t0)
    res["host_loop"] = stat(host)
    return res


def solve(n_s, n_a, reps):
    algo = make(n_s, n_a)
    model = algo.policy.model
    rng = np.random.default_rng(n_s)
    b = Batch(obs=rng.integers(0, n_s, 20 * n_s * n_a), act=rng.integers(0, n_a, 20 * n_s * n_a),
              obs_next=rng.integers(0, n_s, 20 * n_s * n_a), rew=rng.standard_normal(20 * n_s * n_a),
              done=np.zeros(20 * n_s * n_a, bool))
    algo._update_with_batch(b, None, 1)
    res = {}
    for warm in (False, True):
        def call():
            if not warm:
                model._value.zero_()
            model.updated = False
            model.solve_policy()
        call()
        times = timed(call, reps)
        sweeps = model.last_sweeps
        # the kernel alone, on one fixed draw
        P, R, noise = model.sample_trans_prob(), model.sample_reward(), model._tie_noise((n_s, n_a))
        V0 = model._value.clone() if warm else torch.zeros(n_s, dtype=torch.float64, device=DEV)
        ev, ks = [torch.cuda.Event(enable_timing=True) for _ in range(2)], []
        for _ in range(reps):
            V = V0.clone()
            ev[0].record()
            ops.psrl_value_iteration(P, R, noise, model.gamma, model.eps, 100_000, V, model._vi_scratch, model._vi_out)
            ev[1].record()
            torch.cuda.synchronize()
            ks.append(ev[0].elapsed_time(ev[1]) / 1e3)
        k_sweeps = int(model._vi_out[n_s].item())
        kt = float(np.median(ks))
        pbytes = n_s * n_s * n_a * 8
        res["warm" if warm else "cold"] = {
            "solve_policy": stat(times), "sweeps_last_solve": sweeps, "kernel": stat(ks), "kernel_sweeps": k_sweeps,
            "us_per_sweep": kt / k_sweeps * 1e6, "P_bytes": pbytes, "P_GBps": pbytes * k_sweeps / kt / 1e9,
            "share_of_hbm": pbytes * k_sweeps / kt / (HBM_TBPS * 1e12), "P_fits_L2": pbytes <= 50 * 2**20}
        # numpy on the host and eager torch on the GPU, same draw and start
        Pn, Rn, Nn, V0n = (x.cpu().numpy() for x in (P, R, noise, V0))
        host = []
        for _ in range(1 if n_s >= 1024 else 3):
            t0 = time.perf_counter()
            op.value_iteration(Pn, Rn, model.gamma, model.eps, V0n, Nn)
            host.append(time.perf_counter() - t0)
        res["warm" if warm else "cold"]["numpy_host"] = stat(host)

        def eager():
            v = V0.clone()
            Q = R + model.gamma * (P @ v)
            nv = Q.max(dim=1).values
            while not torch.allclose(nv, v, rtol=model.eps):
                v = nv
                Q = R + model.gamma * (P @ v)
                nv = Q.max(dim=1).values
            return (Q + model.eps * noise).argmax(dim=1).cpu()
        eager()
        res["warm" if warm else "cold"]["eager_torch"] = stat(timed(eager, max(3, reps // 3)))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=21)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print("card:", torch.cuda.get_device_name(0), "|", smi)
    out = {"card": torch.cuda.get_device_name(0), "nvidia_smi": smi, "update": {}, "solve": {}}
    for n_s, n_a in ((5, 2), (64, 4)):
        r = update_rows(n_s, n_a, a.reps)
        out["update"][f"{n_s}x{n_a}"] = r
        print(f"update {n_s}x{n_a} (50,000 rows): upload {r['upload']['median_ms']:.3f} ms "
              f"[{r['upload']['min_ms']:.3f}-{r['upload']['max_ms']:.3f}], mirror {r['mirror']['median_ms']:.3f} ms "
              f"[{r['mirror']['min_ms']:.3f}-{r['mirror']['max_ms']:.3f}], host per-row loop {r['host_loop']['median_ms']:.1f} ms")
    for n_s in (5, 64, 256, 1024, 2048):
        r = solve(n_s, 4, a.reps)
        out["solve"][f"{n_s}x4"] = r
        for kind in ("cold", "warm"):
            x = r[kind]
            print(f"solve {n_s}x4 {kind}: solve_policy {x['solve_policy']['median_ms']:.3f} ms "
                  f"[{x['solve_policy']['min_ms']:.3f}-{x['solve_policy']['max_ms']:.3f}], kernel {x['kernel']['median_ms']:.3f} ms "
                  f"over {x['kernel_sweeps']} sweeps ({x['us_per_sweep']:.2f} us/sweep, P {x['P_GBps']:.0f} GB/s, "
                  f"L2-resident {x['P_fits_L2']}), numpy {x['numpy_host']['median_ms']:.1f} ms, "
                  f"eager torch {x['eager_torch']['median_ms']:.2f} ms")
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
