"""Host-side timeline of the PASS-BY-PASS driver of PPO's default minibatch order (the loop the multi-GPU path and the
layer-wise path use: ``order.ready(r)``, then the pass): how long each host statement of a pass takes, and whether the stream had already drained when the pass was enqueued (then the
GPU idled while Python worked).  Diagnostics only; needs a GPU."""
import os
import sys
import time

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import numpy as np
import torch

import bench
from tianshou_b200.data.batch import minibatch_bounds
from tianshou_b200.synthetic import build_mujoco_ppo
from tianshou_b200.utils import policy_within_training_step


def main() -> None:
    dev = torch.device("cuda:0")
    c = bench.CONFIGS["c2"]
    E, T, BS, REPEAT = c["E"], c["T"], c["bs"], bench.REPEAT
    buf = bench.build_host_buffer(E, T, seed=0, device=dev)
    np.random.seed(1000)
    algo, _, _ = build_mujoco_ppo(bench.OBS, bench.ACT, dev, minibatch_shuffle="numpy")
    now = time.perf_counter
    with policy_within_training_step(algo.policy):
        batch, idx = algo._sample(buf, 0)
        for it in range(3):
            b = algo._preprocess_batch(batch, buf, idx)
            N = b.obs.shape[0]
            bounds = minibatch_bounds(N, BS, merge_last=True)
            n_mb = len(bounds)
            hp = algo._loss_hparams()
            stats = algo._alloc_stats(REPEAT * n_mb)
            torch.cuda.synchronize()
            rows = []
            t_start = now()
            with algo._minibatch_order(REPEAT, N) as order:
                for r in range(REPEAT):
                    idle = torch.cuda.current_stream().query()          # True: nothing pending -> the GPU is waiting for the host
                    t0 = now(); order.ready(r)
                    t1 = now()
                    if algo.recompute_adv and r > 0:
                        algo._add_returns_and_advantages(b, None, None)
                    t2 = now(); algo._device_passes(b, order.rows[r], bounds, hp, stats[r * n_mb:], 1, False)
                    t3 = now()
                    rows.append((r, idle, 1e3 * (t0 - t_start), 1e6 * (t1 - t0), 1e6 * (t2 - t1), 1e6 * (t3 - t2)))
                torch.cuda.synchronize()
                total = 1e3 * (now() - t_start)
            if it == 2:
                print("pass stream_idle_at_entry t_entry_ms ready_us recompute_enqueue_us pass_enqueue_us")
                for row in rows:
                    print("%4d %5s %10.3f %10.1f %10.1f %10.1f" % row)
                print(f"total {total:.3f} ms for {REPEAT} passes")


if __name__ == "__main__":
    main()
