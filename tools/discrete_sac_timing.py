"""Time ``DiscreteSAC.update()`` on one GPU next to the eager-PyTorch restatement of the reference's update
(oracle/oracle_discrete_sac.py) on the same GPU, the same buffer and the same initial weights, in the same call.

    python tools/discrete_sac_timing.py [--reps 21] [--out timing.json]

Workloads:
  cartpole_mlp  : the test_discrete_sac.py shape -- obs 4, 2 actions, Net (64, 64) trunks, batch 64, n_step 3, a uniform
                  20000-slot buffer of 10 environments with stored obs_next.
  atari_cnn     : the atari_sac.py shape with separate trunks -- three DQNet(4, 84, 84, features_only=True,
                  output_dim_added_layer=512) behind ScaledObsInputActionReprNet, 6 actions, batch 64, n_step 3, a 100k-slot
                  prioritised buffer of uint8 single frames (stack_num 4) with the device mirror on.
Each number is the median wall time of ``--reps`` updates after three warm-up updates, with a device synchronise inside the
timed region.  The eager update includes what the reference's update does on the host: the index draw, the frame-stack
gather and upload, and the priority update.  Prints the card name and power limit with the numbers.  Needs a CUDA device.
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


class _Discrete:
    def __init__(self, n: int) -> None:
        self.n = n
        self.shape = ()


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return {"name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip()}


def _median_ms(fn, reps: int, warmup: int = 3) -> tuple[float, list[float]]:
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        out.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(out)), out


def _setup(name: str):
    """(tianshou_b200 algorithm, buffer, eager modules, eager buffer view, obs reader, per, cfg)."""
    from oracle import oracle_discrete_sac as ods
    from tianshou_b200.algorithm import AdamOptimizerFactory, DiscreteSAC
    from tianshou_b200.algorithm.modelfree.discrete_sac import DiscreteSACPolicy
    from tianshou_b200.data import Batch, PrioritizedVectorReplayBuffer, VectorReplayBuffer
    from tianshou_b200.env.atari import DQNet, ScaledObsInputActionReprNet
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.discrete import DiscreteActor, DiscreteCritic
    torch.manual_seed(0)
    rng = np.random.default_rng(0)
    if name == "cartpole_mlp":
        A, E, size = 2, 10, 20000
        trunk = lambda: Net(state_shape=(4,), hidden_sizes=(64, 64))
        eager = lambda: ods.mlp_head_net(4, (64, 64), A)
        buf = VectorReplayBuffer(size, E, device=DEV)
        for _ in range(size // E):
            buf.add(Batch(obs=rng.standard_normal((E, 4)).astype(np.float32), act=rng.integers(0, A, E), rew=rng.standard_normal(E),
                          terminated=rng.random(E) < 0.02, truncated=np.zeros(E, bool),
                          obs_next=rng.standard_normal((E, 4)).astype(np.float32)), buffer_ids=np.arange(E))
        per, cfg = False, dict(actor_lr=1e-4, critic_lr=1e-3, gamma=0.95, alpha=0.05)
    else:
        A, E, size = 6, 10, 100_000
        trunk = lambda: ScaledObsInputActionReprNet(DQNet(4, 84, 84, A, features_only=True, output_dim_added_layer=512))
        eager = lambda: ods.cnn_head_net(4, 84, 84, 512, A)
        buf = PrioritizedVectorReplayBuffer(size, E, alpha=0.6, beta=0.4, stack_num=4, ignore_obs_next=True, save_only_last_obs=True,
                                            device=DEV, device_mirror=True)
        for _ in range(size // E):
            st = np.repeat(rng.integers(0, 256, (E, 1, 84, 84), dtype=np.uint8), 4, axis=1)
            buf.add(Batch(obs=st, act=rng.integers(0, A, E), rew=rng.standard_normal(E), terminated=rng.random(E) < 0.01,
                          truncated=np.zeros(E, bool), obs_next=st), buffer_ids=np.arange(E))
        per, cfg = True, dict(actor_lr=1e-5, critic_lr=1e-5, gamma=0.99, alpha=0.05)
    actor = DiscreteActor(preprocess_net=trunk(), action_shape=A, softmax_output=False).to(DEV)
    c1 = DiscreteCritic(preprocess_net=trunk(), last_size=A).to(DEV)
    c2 = DiscreteCritic(preprocess_net=trunk(), last_size=A).to(DEV)
    mods = [eager().to(DEV) for _ in range(3)]
    with torch.no_grad():
        for src, dst in zip((actor, c1, c2), mods, strict=True):
            for p, q in zip(src.parameters(), dst.parameters(), strict=True):
                q.copy_(p)
    algo = DiscreteSAC(policy=DiscreteSACPolicy(actor=actor, action_space=_Discrete(A)),
                       policy_optim=AdamOptimizerFactory(lr=cfg["actor_lr"]), critic=c1, critic_optim=AdamOptimizerFactory(lr=cfg["critic_lr"]),
                       critic2=c2, critic2_optim=AdamOptimizerFactory(lr=cfg["critic_lr"]), gamma=cfg["gamma"], alpha=cfg["alpha"],
                       n_step_return_horizon=3)
    view = dict(obs=np.asarray(buf.obs), act=np.asarray(buf.act), rew=np.asarray(buf.rew), done=np.asarray(buf.done),
                terminated=np.asarray(buf.terminated), offset=np.asarray(buf._extend_offset), last_index=buf.last_index,
                lengths=buf._sizes)
    if name == "cartpole_mlp":
        view["obs_next"] = np.asarray(buf.obs_next)
        obs_of = ods.flat_obs(view["obs"], DEV)
    else:
        obs_of = ods.frame_obs(view, 4, 255.0, DEV)
    return algo, buf, mods, view, obs_of, per, cfg


def run(name: str, reps: int) -> dict:
    from oracle import oracle_discrete_sac as ods
    from tianshou_b200.utils import policy_within_training_step
    algo, buf, (actor, c1, c2), view, obs_of, per, cfg = _setup(name)
    olds = [copy.deepcopy(c1), copy.deepcopy(c2)]
    opts = [torch.optim.Adam(actor.parameters(), lr=cfg["actor_lr"]), torch.optim.Adam(c1.parameters(), lr=cfg["critic_lr"]),
            torch.optim.Adam(c2.parameters(), lr=cfg["critic_lr"])]
    B = 64

    def device_update():
        with policy_within_training_step(algo.policy):
            algo.update(buffer=buf, sample_size=B)

    def eager_update():
        idx = buf.sample_indices(B)
        w = None
        if per:
            w = buf.get_weight(idx)
            w = (w / np.max(w)).astype(np.float32)
        res = ods.discrete_sac_update(actor, [c1, c2], olds, opts, obs_of, view, idx, w, cfg["gamma"], 3, cfg["alpha"], 0.005,
                                      "obs_next" in view)
        if per:
            buf.update_weight(idx, res["weight"])

    np.random.seed(0)
    dev_ms, dev_all = _median_ms(device_update, reps)
    np.random.seed(0)
    eager_ms, eager_all = _median_ms(eager_update, reps)
    return {"workload": name, "batch": B, "reps": reps, "device_ms": dev_ms, "eager_ms": eager_ms, "speedup": eager_ms / dev_ms,
            "device_all_ms": dev_all, "eager_all_ms": eager_all}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=21)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    out = {"card": card(), "results": [run(n, args.reps) for n in ("cartpole_mlp", "atari_cnn")]}
    print(json.dumps(out["card"]))
    for r in out["results"]:
        print(f"{r['workload']:14s} device {r['device_ms']:8.3f} ms   eager {r['eager_ms']:8.3f} ms   x{r['speedup']:.2f}")
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
