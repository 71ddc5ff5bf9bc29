"""Where the default (numpy-order) update loses time against the device-order update on ONE GPU: CUDA-event time of
`_preprocess_batch + _update_with_batch` on a device-resident rollout (bench.py's `value` region) in five variants.
Diagnostics only; needs a GPU."""
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
    algo_dv, _, _ = build_mujoco_ppo(bench.OBS, bench.ACT, dev, minibatch_shuffle="device")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def timed(fn, iters=5, warm=3):
        for _ in range(warm):
            fn()
        ms, wall = [], []
        for _ in range(iters):
            flush.zero_()
            torch.cuda.synchronize()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0 = time.perf_counter()
            s.record(); fn(); e.record()
            torch.cuda.synchronize()
            wall.append(1e3 * (time.perf_counter() - t0)); ms.append(s.elapsed_time(e))
        return sum(ms) / len(ms), sum(wall) / len(wall)

    with policy_within_training_step(algo.policy), policy_within_training_step(algo_dv.policy):
        batch, idx = algo._sample(buf, 0)

        def a_device_order():
            b = algo_dv._preprocess_batch(batch, buf, idx)
            algo_dv._update_with_batch(b, BS, REPEAT)

        def b_default():
            with algo._minibatch_order_job(buf, REPEAT):
                b = algo._preprocess_batch(batch, buf, idx)
                algo._update_with_batch(b, BS, REPEAT)

        def c_default_rows_ready_first():
            with algo._minibatch_order_job(buf, REPEAT) as order:
                for r in range(REPEAT):
                    order.ready(r)
                torch.cuda.current_stream().synchronize()       # every row is on the device
                b = algo._preprocess_batch(batch, buf, idx)
                algo._update_with_batch(b, BS, REPEAT)

        def d_preprocess_only():
            algo._preprocess_batch(batch, buf, idx)

        def e_job_only():
            with algo._minibatch_order_job(buf, REPEAT) as order:
                for r in range(REPEAT):
                    order.ready(r)
                torch.cuda.current_stream().synchronize()

        def f_default_no_early_start():
            b = algo._preprocess_batch(batch, buf, idx)
            algo._update_with_batch(b, BS, REPEAT)

        for name, fn in (("a device order", a_device_order), ("b default (job started first, as update() does)", b_default),
                         ("c default, every row complete before the update is enqueued", c_default_rows_ready_first),
                         ("d _preprocess_batch only", d_preprocess_only), ("e minibatch orders only (host job + feed)", e_job_only),
                         ("f default, order opened inside _update_with_batch", f_default_no_early_start)):
            ev, wall = timed(fn)
            print(f"{name:70s} events {ev:8.3f} ms   wall {wall:8.3f} ms")


if __name__ == "__main__":
    main()
