"""Host timeline of ONE default-order `PPO.update()`-equivalent (device-resident rollout): when each C entry point is called
and how long the call blocks the host, plus the order's open / close.  Diagnostics only; needs a GPU."""
import os
import sys
import time

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import numpy as np
import torch

import bench
import tianshou_b200._cabi as cabi
import tianshou_b200.algorithm.modelfree.ppo as ppo_mod
import tianshou_b200.algorithm.modelfree.a2c as a2c_mod
import tianshou_b200.algorithm.minibatch_order as order_mod
import tianshou_b200.data.batch as batch_mod
import tianshou_b200.ops as ops_mod
from tianshou_b200.synthetic import build_mujoco_ppo
from tianshou_b200.utils import policy_within_training_step

LOG: list = []
T0 = [0.0]
_real_call = cabi.call


def traced_call(name, *args):
    t = time.perf_counter()
    r = _real_call(name, *args)
    LOG.append((name, 1e3 * (t - T0[0]), 1e6 * (time.perf_counter() - t)))
    return r


def main() -> None:
    dev = torch.device("cuda:0")
    c = bench.CONFIGS["c2"]
    E, T, BS, REPEAT = c["E"], c["T"], c["bs"], bench.REPEAT
    buf = bench.build_host_buffer(E, T, seed=0, device=dev)
    np.random.seed(1000)
    algo, _, _ = build_mujoco_ppo(bench.OBS, bench.ACT, dev, minibatch_shuffle="numpy")
    for mod in (ppo_mod, a2c_mod, order_mod, batch_mod, ops_mod):
        if hasattr(mod, "call"):
            mod.call = traced_call
    batch_mod_call_patch = batch_mod.__dict__.get("call")
    cabi.call = traced_call          # `from .._cabi import call` inside functions picks this up
    sync = torch.cuda.synchronize
    with policy_within_training_step(algo.policy):
        batch, idx = algo._sample(buf, 0)
        for it in range(4):
            sync()
            LOG.clear()
            T0[0] = time.perf_counter()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            with algo._minibatch_order_job(buf, REPEAT):
                LOG.append(("<order opened>", 1e3 * (time.perf_counter() - T0[0]), 0.0))
                b = algo._preprocess_batch(batch, buf, idx)
                LOG.append(("<preprocess enqueued>", 1e3 * (time.perf_counter() - T0[0]), 0.0))
                algo._update_with_batch(b, BS, REPEAT)
                LOG.append(("<_update_with_batch returned>", 1e3 * (time.perf_counter() - T0[0]), 0.0))
            LOG.append(("<order closed>", 1e3 * (time.perf_counter() - T0[0]), 0.0))
            e.record()
            sync()
            if it == 3:
                print(f"events {s.elapsed_time(e):.3f} ms")
                print("   at_ms  blocks_us  entry")
                for name, at, dur in LOG:
                    print(f"{at:8.3f} {dur:10.1f}  {name}")


if __name__ == "__main__":
    main()
