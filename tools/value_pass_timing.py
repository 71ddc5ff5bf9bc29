"""Time the passes of PPO's value recompute on the benchmark shapes, the value pass with and without the
next-observation alias map alternating launch by launch on the same inputs.

    python tools/value_pass_timing.py [--envs 4096] [--steps 128] [--reps 20] [--out timing.json]

Rollout: a seeded ``fill_vector_buffer`` rollout of envs x steps transitions (obs 17 / act 6), weights from
``build_mujoco_ppo``.  Timed with CUDA events, 3 warm-ups and ``--reps`` launches each, a 256 MB write before every launch so
that nothing is served from L2:
  * ``critic_forward``: ``ops.critic_forward(obs, obs_next)``, the critic on all 2 N rows;
  * ``critic_forward_dedup``: ``ops.critic_forward_dedup`` with the map of ``ops.next_alias_map`` (one evaluation per
    distinct row), alternated with the former; ``max_abs_diff`` of v_s / v_next between the two (must be 0);
  * ``next_alias_map`` (once per update), ``actor_logp``, ``gae``;
  * ``add_returns_and_advantages``: one full recompute call of the algorithm (value pass + GAE), with the map and with
    it disabled, alternated.
``rows_not_aliased`` is the number of rows whose obs_next is not bit-equal to the following obs row (env segment ends and
episode ends).  Prints the card name and power limit with the numbers.  Needs a CUDA device.
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

O, A = 17, 6


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return {"name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip()}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=128)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("value_pass_timing.py needs a CUDA device")
    from tianshou_b200 import ops
    from tianshou_b200.data import VectorReplayBuffer
    from tianshou_b200.synthetic import build_mujoco_ppo, fill_vector_buffer
    from tianshou_b200.utils import policy_within_training_step
    dev = torch.device("cuda:0")
    E, T = args.envs, args.steps
    N = E * T
    buf = VectorReplayBuffer(N, E, device=dev)
    fill_vector_buffer(buf, np.random.default_rng(0), E, T, O, A)
    algo, _, _ = build_mujoco_ppo(O, A, dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def timed(fns: dict) -> dict:
        """median / p10 / p90 of ``--reps`` event-timed launches per entry, the entries alternating launch by launch"""
        for _ in range(3):
            for fn in fns.values():
                fn()
        spans = {k: [] for k in fns}
        for _ in range(max(args.reps, 1)):
            for k, fn in fns.items():
                flush.zero_()
                t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0.record()
                fn()
                t1.record()
                spans[k].append((t0, t1))
        torch.cuda.synchronize()
        out = {}
        for k, evs in spans.items():
            ms = [a.elapsed_time(b) for a, b in evs]
            out[k] = {"ms_median": float(np.median(ms)), "ms_p10_p90": [float(np.percentile(ms, 10)), float(np.percentile(ms, 90))]}
        return out

    with policy_within_training_step(algo.policy):
        batch, idx = algo._sample(buf, 0)
        batch = algo._preprocess_batch(batch, buf, idx)
        f, desc = algo._flat.flat, algo._desc
        obs, obs_next = batch.obs, batch.obs_next
        amap = ops.next_alias_map(obs, obs_next)
        full = [torch.empty(N, device=dev) for _ in range(2)]
        dedup = [torch.empty(N, device=dev) for _ in range(2)]
        logp = torch.empty(N, device=dev)
        adv, ret = torch.empty(N, device=dev), torch.empty(N, device=dev)
        ws = algo._gae_workspace(N)
        passes = timed({
            "critic_forward": lambda: ops.critic_forward(f, desc, obs, obs_next, out=full[0], out2=full[1]),
            "critic_forward_dedup": lambda: ops.critic_forward_dedup(f, desc, obs, obs_next, amap, out=dedup[0], out2=dedup[1]),
        })
        passes.update(timed({
            "next_alias_map": lambda: ops.next_alias_map(obs, obs_next, out=amap),
            "actor_logp": lambda: ops.actor_logp(f, desc, obs, batch.act, out=logp),
            "gae": lambda: ops.gae(full[0], full[1], batch.rew, batch.terminated, batch.truncated, batch.get("_unfinished"),
                                   gamma=0.99, gae_lambda=0.95, out=(adv, ret), workspace=ws),
        }))
        kept = algo._next_alias

        def recompute(with_map: bool):
            algo._next_alias = kept if with_map else None
            algo._add_returns_and_advantages(batch, None, None)
        calls = timed({"add_returns_and_advantages": lambda: recompute(False),
                       "add_returns_and_advantages_dedup": lambda: recompute(True)})
        algo._rms_end()
    result = {
        "card": card(), "rows": N, "obs_dim": O, "reps": args.reps,
        "rows_not_aliased": int(amap.count.item()),
        "max_abs_diff": {"v_s": float((full[0] - dedup[0]).abs().max()), "v_next": float((full[1] - dedup[1]).abs().max())},
        "bit_equal": bool(torch.equal(full[0], dedup[0]) and torch.equal(full[1], dedup[1])),
        "passes": passes, "calls": calls,
    }
    print(json.dumps(result, indent=1))
    if args.out:
        with open(args.out, "w") as fo:
            json.dump(result, fo, indent=1)


if __name__ == "__main__":
    main()
