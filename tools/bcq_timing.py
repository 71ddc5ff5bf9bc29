"""Time ``BCQ.update()`` on one GPU next to the eager-PyTorch restatement of the reference's update (oracle/oracle_bcq.py) on the
same GPU, the same buffer and the same initial weights, and ``BCQPolicy.forward`` on 10 observations next to the reference's loop
over them, in the same call.

    python tools/bcq_timing.py [--reps 21] [--out timing.json]

Workload: examples/offline/d4rl_bcq.py -- obs 17, act 6, an MLP perturbation and Net critics of [256, 256], a VAE of [512, 512]
with latent 12, batch 256, N = 10, on a 100k-transition ``from_data`` buffer with the device mirror on; the policy samples 100
actions per observation.  Each number is the median wall time of ``--reps`` calls after four warm-up calls, with a device
synchronise inside the timed region, and its 10th-90th percentile range.  The eager update includes the index draw and the upload
of the sampled rows; the reference loop is ``BCQPolicy.forward`` with grad enabled on the same modules.  Prints the card name and
power limit with the numbers.  Needs a CUDA device.
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


class _Box:
    def __init__(self, dim: int) -> None:
        self.shape = (dim,)
        self.low = -np.ones(dim, np.float32)
        self.high = np.ones(dim, np.float32)


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return {"name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip()}


def _time_ms(fn, reps: int, warmup: int = 4) -> list[float]:
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        out.append((time.perf_counter() - t0) * 1e3)
    return out


def run(reps: int) -> dict:
    from oracle.oracle_bcq import BcqNets, bcq_update
    from tianshou_b200.algorithm import BCQ, AdamOptimizerFactory, BCQPolicy
    from tianshou_b200.data import Batch, ReplayBuffer
    from tianshou_b200.utils import policy_within_training_step
    from tianshou_b200.utils.net.common import MLP, Net
    from tianshou_b200.utils.net.continuous import VAE, ContinuousCritic, Perturbation
    O, A, H, VH, L, B, N, S, size = 17, 6, (256, 256), (512, 512), 12, 256, 10, 100, 100_000
    rng = np.random.default_rng(0)
    term = rng.random(size) < 1e-3
    term[[0, -1]] = True
    trunc = np.zeros(size, bool)
    data = (rng.standard_normal((size, O)).astype(np.float32), np.tanh(rng.standard_normal((size, A))).astype(np.float32),
            rng.standard_normal(size), term, trunc, term | trunc, rng.standard_normal((size, O)).astype(np.float32))
    torch.manual_seed(0)
    pert = Perturbation(preprocess_net=MLP(input_dim=O + A, output_dim=A, hidden_sizes=H), max_action=1.0).to(DEV)
    crit = ContinuousCritic(preprocess_net=Net(state_shape=(O,), action_shape=(A,), hidden_sizes=H, concat=True)).to(DEV)
    vae = VAE(encoder=MLP(input_dim=O + A, hidden_sizes=VH), decoder=MLP(input_dim=O + L, output_dim=A, hidden_sizes=VH), hidden_dim=VH[-1],
              latent_dim=L, max_action=1.0).to(DEV)
    nets = BcqNets(O, A, H, VH, L)
    with torch.no_grad():
        for dst, src in ((nets.p, pert), (nets.c[0], crit), (nets.c[1], crit), (torch.nn.ModuleList(nets.vae_modules()), vae)):
            for p, q in zip(dst.parameters(), src.parameters(), strict=True):
                p.copy_(q.detach().cpu())
        nets.p_old.load_state_dict(nets.p.state_dict())
        for k in range(2):
            nets.c_old[k].load_state_dict(nets.c[k].state_dict())
    policy = BCQPolicy(actor_perturbation=pert, critic=crit, vae=vae, action_space=_Box(A), forward_sampled_times=S)
    algo = BCQ(policy=policy, actor_perturbation_optim=AdamOptimizerFactory(lr=1e-3), critic_optim=AdamOptimizerFactory(lr=1e-3),
               vae_optim=AdamOptimizerFactory(lr=1e-3), num_sampled_action=N)
    buf = ReplayBuffer.from_data(*data)
    buf.enable_device_mirror()
    buf.sync_device_mirror()

    def device_update():
        with policy_within_training_step(algo.policy):
            algo.update(buf, B)

    for m in nets.modules():
        m.to(DEV)
    opts = [torch.optim.Adam(nets.p.parameters(), lr=1e-3), torch.optim.Adam(nets.c[0].parameters(), lr=1e-3),
            torch.optim.Adam(nets.c[1].parameters(), lr=1e-3), torch.optim.Adam(nets.vae_parameters(), lr=1e-3)]
    host = dict(zip(("obs", "act", "rew", "terminated", "truncated", "done", "obs_next"), data, strict=True))
    eager_rs = np.random.RandomState(1)

    def eager_update():
        idx = eager_rs.choice(size, B)
        batch = {k: torch.as_tensor(host[k][idx], device=DEV) for k in ("obs", "act", "obs_next", "done")}
        batch["rew"] = torch.as_tensor(host["rew"][idx], device=DEV).float()
        r = bcq_update(nets, opts, batch, lambda shape: torch.randn(shape, device=DEV), gamma=0.99, tau=0.005, lmbda=0.75, N=N)
        float(r["critic1_loss"])

    obs = rng.standard_normal((10, O)).astype(np.float32)

    def device_policy():
        with torch.no_grad():
            algo.policy(Batch(obs=obs, info={}))

    def reference_policy():
        algo.policy(Batch(obs=obs, info={}))          # grad enabled: the reference's loop on the same modules

    du, eu = _time_ms(device_update, reps), _time_ms(eager_update, reps)
    dp, rp = _time_ms(device_policy, reps), _time_ms(reference_policy, reps)
    pct = lambda x: [float(np.percentile(x, 10)), float(np.percentile(x, 90))]
    out = {"workload": "d4rl_bcq", "obs": O, "act": A, "batch": B, "num_sampled_action": N, "forward_sampled_times": S}
    for kind, d, e in (("update", du, eu), ("policy_10_obs", dp, rp)):
        out[kind] = {"device_ms": float(np.median(d)), "device_p10_p90": pct(d), "eager_ms": float(np.median(e)),
                     "eager_p10_p90": pct(e), "speedup": float(np.median(e) / np.median(d))}
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=21)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    out = {"card": card(), "results": [run(args.reps)]}
    print(json.dumps(out["card"]))
    for r in out["results"]:
        for kind in ("update", "policy_10_obs"):
            x = r[kind]
            print(f"{r['workload']:10s} {kind:14s} device {x['device_ms']:8.3f} ms (p10-p90 {x['device_p10_p90'][0]:.3f}-"
                  f"{x['device_p10_p90'][1]:.3f})   eager {x['eager_ms']:8.3f} ms (p10-p90 {x['eager_p10_p90'][0]:.3f}-"
                  f"{x['eager_p10_p90'][1]:.3f})   x{x['speedup']:.2f}")
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
