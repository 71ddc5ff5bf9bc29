"""Time GAIL.update() on one GPU next to PPO.update() alone on the same inputs (what the discriminator adds) and next to the
eager-PyTorch GAIL on the same GPU in the same call.

    python tools/gail_timing.py [--reps 7] [--out timing.json]

Workloads: the reference's irl_gail example (obs 17 / act 6, tanh [64, 64] actor, critic and discriminator, 64 envs x 32 steps
= 2048 rows, minibatch 64, repeat 10, disc_update_num 2, advantage recompute and return scaling on) and the same networks on a
64 x 256 rollout.  Times are CUDA-event medians of ``--reps`` updates after two warm-up updates.  The eager GAIL is the stock
PyTorch PPO update of tools/torch_eager_context.py plus the eager discriminator half of oracle/oracle_gail.py (reward pass and
the disc_update_num Adam steps), each timed here.  Prints the card name and power limit with the numbers.  Needs a CUDA device.
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
sys.path.insert(0, os.path.join(ROOT, "tools"))

WORKLOADS = [("irl_gail_64x32", 64, 32), ("rollout_64x256", 64, 256)]     # name, envs, steps
O, A, HIDDEN, BS, REPEAT, DUN = 17, 6, (64, 64), 64, 10, 2


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return {"name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip()}


def _events_ms(fn, reps: int, warmup: int = 2) -> list[float]:
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b))
    return out


def _buffer(E: int, T: int, seed: int):
    from tianshou_b200.data import Batch, VectorReplayBuffer
    rng = np.random.default_rng(seed)
    buf = VectorReplayBuffer(E * T, E, device="cuda:0")
    for _ in range(T):
        buf.add(Batch(obs=rng.standard_normal((E, O)).astype(np.float32), act=rng.standard_normal((E, A)).astype(np.float32),
                      rew=np.zeros(E), terminated=rng.random(E) < 0.01, truncated=np.zeros(E, bool),
                      obs_next=rng.standard_normal((E, O)).astype(np.float32), info=Batch()))
    return buf


def _algos(expert):
    from test_gail_gpu import _gail, _nets
    from tianshou_b200.algorithm import PPO, AdamOptimizerFactory, ProbabilisticActorPolicy
    from ts_testutil import Box
    torch.manual_seed(0)
    actor, critic, disc = _nets(O, A, HIDDEN)
    kw = dict(max_grad_norm=0.5, vf_coef=0.25, ent_coef=0.001, return_scaling=True, recompute_advantage=True,
              advantage_normalization=False)
    gail = _gail(actor, critic, disc, expert, A, disc_update_num=DUN, **kw)
    torch.manual_seed(0)
    actor2, critic2, _ = _nets(O, A, HIDDEN)
    policy = ProbabilisticActorPolicy(actor=actor2, dist_fn=gail.policy.dist_fn, action_scaling=True, action_bound_method="clip",
                                      action_space=Box(A))
    ppo = PPO(policy=policy, critic=critic2, optim=AdamOptimizerFactory(lr=3e-4), **kw)
    return gail, ppo


def _eager_disc_ms(E: int, T: int, reps: int) -> list[float]:
    from oracle import oracle_gail as og
    dev = torch.device("cuda:0")
    N = E * T
    disc = og.disc_net(O, A, HIDDEN, torch.nn.Tanh).to(dev)
    opt = torch.optim.Adam(disc.parameters(), lr=2.5e-5)
    g = torch.Generator().manual_seed(0)
    obs, act = torch.randn(N, O, generator=g).to(dev), torch.randn(N, A, generator=g).to(dev)
    e_obs, e_act = torch.randn(N, O, generator=g).to(dev), torch.randn(N, A, generator=g).to(dev)

    def step():
        og.rewards(disc, obs, act).cpu()            # the reference's to_numpy of the rewards
        order = np.random.permutation(N)
        og.disc_update(disc, opt, obs, act, order, e_obs, e_act, DUN)
    return _events_ms(step, reps)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gail_timing.py needs a CUDA device")
    from tianshou_b200.data import ReplayBuffer
    from tianshou_b200.utils import policy_within_training_step
    from torch_eager_context import run as eager_ppo
    rng = np.random.default_rng(7)
    n_exp = 20000
    expert = ReplayBuffer.from_data(rng.standard_normal((n_exp, O)).astype(np.float32),
                                    (rng.standard_normal((n_exp, A)) + 0.5).astype(np.float32), np.zeros(n_exp),
                                    np.zeros(n_exp, bool), np.zeros(n_exp, bool), np.zeros(n_exp, bool),
                                    rng.standard_normal((n_exp, O)).astype(np.float32))
    res = {"card": card(), "workloads": {}}
    for name, E, T in WORKLOADS:
        buf = _buffer(E, T, 1)
        gail, ppo = _algos(expert)
        np.random.seed(0)
        with policy_within_training_step(gail.policy), policy_within_training_step(ppo.policy):
            t_gail = _events_ms(lambda: gail.update(buffer=buf, batch_size=BS, repeat=REPEAT), a.reps)
            t_ppo = _events_ms(lambda: ppo.update(buffer=buf, batch_size=BS, repeat=REPEAT), a.reps)
            t_gail2 = _events_ms(lambda: gail.update(buffer=buf, batch_size=BS, repeat=REPEAT), a.reps, warmup=0)
        t_disc = _eager_disc_ms(E, T, a.reps)
        eager = eager_ppo(E=E, T=T, bs=BS, repeat=REPEAT, steps=a.reps)
        med = lambda v: float(np.median(v))  # noqa: E731
        res["workloads"][name] = {
            "rows": E * T, "minibatch": BS, "repeat": REPEAT, "disc_update_num": DUN,
            "gail_update_ms": med(t_gail + t_gail2), "gail_update_ms_runs": [med(t_gail), med(t_gail2)],
            "ppo_update_ms": med(t_ppo), "disc_overhead_ms": med(t_gail + t_gail2) - med(t_ppo),
            "eager_ppo_update_ms": float(eager["ms_per_update"]), "eager_disc_half_ms": med(t_disc),
            "eager_gail_ms": float(eager["ms_per_update"]) + med(t_disc),
        }
        print(name, json.dumps(res["workloads"][name]), flush=True)
    print(json.dumps(res["card"]))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
