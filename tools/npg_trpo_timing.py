"""Time NPG.update() and TRPO.update() on one GPU (CUDA events, after warm-up), one Fisher-vector product in isolation with
its algorithmic flop count, and the eager-PyTorch restatement (oracle/oracle_npg.py) on the same GPU in the same call.

    python tools/npg_trpo_timing.py [--reps 5] [--out timing.json]

Workloads: the reference's MuJoCo example (16 envs x 64 steps, obs 17 / act 6, [64, 64] tanh, full batch, repeat 1,
optim_critic_iters 20), the BASELINE rollout shape 4096 x 128 at obs 17 / act 6, and obs 376 / act 17 with [256, 256].
NPG steps with trust_region_size 0.01 (random advantages would drive the default 0.5 out of range).  Prints the card name
and power limit with the numbers.  Needs a CUDA device; there is no CPU fallback.
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

WORKLOADS = [  # name, envs, steps, obs, act, hidden
    ("mujoco_example_16x64", 16, 64, 17, 6, (64, 64)),
    ("baseline_4096x128", 4096, 128, 17, 6, (64, 64)),
    ("humanoid_376_256x256", 16, 64, 376, 17, (256, 256)),
]


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return {"name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip()}


def fvp_flops(B: int, dims: list[int]) -> int:
    """Tangent pass (2 GEMMs per layer after the first) + backward (weight and input gradient GEMMs): 2 flops per MAC."""
    macs = 0
    for i in range(len(dims) - 1):
        mk = B * dims[i] * dims[i + 1]
        macs += mk * (1 if i == 0 else 2)           # x W'^T (+ x' W^T)
        macs += mk * (1 if i == 0 else 2)           # dW (+ dX)
    return 2 * macs


def events_ms(fn, reps: int) -> list[float]:
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        out.append(a.elapsed_time(b))
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the results as JSON here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("npg_trpo_timing: needs a CUDA device")
    from test_npg_gpu import _algo, _nets
    from ts_testutil import synth_rollout

    from oracle import oracle_npg as on
    from tianshou_b200.algorithm import NPG, TRPO
    from tianshou_b200.data import Batch, VectorReplayBuffer
    from tianshou_b200.utils import policy_within_training_step
    res = {"card": card(), "workloads": []}
    for name, E, T, O, A, H in WORKLOADS:
        buf = VectorReplayBuffer(E * T, E, device="cuda:0")
        for s in synth_rollout(np.random.default_rng(0), E, T, O, A, p_term=0.01, trunc_len=200):
            buf.add(Batch(**s), buffer_ids=np.arange(E))
        row = {"workload": name, "rows": E * T, "obs": O, "act": A, "hidden": list(H)}
        for cls in (NPG, TRPO):
            torch.manual_seed(0)
            actor, critic = _nets(False, O, A, H)
            algo = _algo(cls, actor, critic, False, A, optim_critic_iters=20, trust_region_size=0.01)

            def run():
                with policy_within_training_step(algo.policy):
                    algo.update(buffer=buf, batch_size=None, repeat=1)

            run()
            row[f"{cls.__name__}_update_ms"] = events_ms(run, args.reps)
            if cls is NPG:
                L = algo._layered
                B = E * T
                obs = torch.randn(B, O, device="cuda:0")
                at = L.a_trunk.forward(obs, B, "up")
                ah = L.a_head.forward(at[-1], B, "up")
                v = torch.randn(L.group.n, device="cuda:0")
                algo._fvp(at, ah, v, B)
                ms = events_ms(lambda: [algo._fvp(at, ah, v, B) for _ in range(20)], args.reps)
                per = float(np.median(ms)) / 20
                fl = fvp_flops(B, [O, *H, A])
                row["fvp_ms"] = per
                row["fvp_algorithmic_tflops"] = fl / (per * 1e-3) / 1e12
        # eager PyTorch restatement on the same GPU, same shapes (full batch, repeat 1)
        N = E * T
        actor_o = on.Actor(O, A, H, torch.nn.Tanh, False).cuda()
        critic_o = on.critic_net(O, H, torch.nn.Tanh).cuda()
        opt = torch.optim.Adam(critic_o.parameters(), lr=1e-3)
        data = {"obs": torch.randn(N, O, device="cuda:0"), "act": torch.randn(N, A, device="cuda:0"),
                "adv": torch.randn(N, device="cuda:0"), "returns": torch.randn(N, device="cuda:0")}
        with torch.no_grad():
            data["logp_old"] = actor_o.dist(data["obs"]).log_prob(data["act"])
        perm = [np.random.permutation(N)]
        for trpo in (False, True):
            key = "eager_TRPO_update_ms" if trpo else "eager_NPG_update_ms"
            fn = lambda: on.update(actor_o, critic_o, opt, data, perm, None, trpo=trpo, optim_critic_iters=20,  # noqa: E731
                                   trust_region_size=0.01)
            fn()
            row[key] = events_ms(fn, args.reps)
        res["workloads"].append(row)
        print(json.dumps(row), flush=True)
    print(json.dumps(res["card"]))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
