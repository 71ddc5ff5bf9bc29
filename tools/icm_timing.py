"""Time ``ICMOffPolicyWrapper.update()`` / ``ICMOnPolicyWrapper.update()`` on one GPU against the same wrapped algorithm's update
without the wrapper (the difference is the ICM's share), and the ICM's part against an eager-PyTorch restatement of the reference
(icm.py:77-109: the batch read through the buffer's ``__getitem__``, ``IntrinsicCuriosityModule.forward``, the reference's loss,
autograd and torch's Adam), on the same GPU, the same buffer and the same initial weights, in the same call.

    python tools/icm_timing.py [--reps 21] [--out timing.json]

Workloads:
  dqn_icm    test/modelbased/test_dqn_icm.py: obs 4, 2 actions, batch 64, ``Net([128, 128, 128])`` Q-network, feature
             ``MLP([128, 128]) -> 128``, ICM hidden ``[128]``, n-step 3;
  atari_icm  examples/atari/atari_dqn.py with ``icm_lr_scale > 0``: ``DQNet`` Q-network behind ``ScaledObsInputActionReprNet``,
             ``DQNet(features_only=True).net`` features, 4 x 84 x 84 uint8 stacks, 6 actions, batch 32, a 100k-slot mirrored
             buffer, ICM hidden ``[512]``;
  ppo_icm    test/modelbased/test_ppo_icm.py: one ``Net([64, 64])`` shared by actor and critic, a 2000-row rollout, repeat 10,
             minibatch 64, feature ``MLP([64]) -> 64``, ICM hidden ``[64]``.
The wrapped, unwrapped and eager updates alternate update by update; each number is the median wall time of ``--reps`` updates
(with min and max) after three warm-up updates of each, with a device synchronise inside the timed region.  ``launches`` counts
the kernel launches of one wrapped and one unwrapped update through the project's library.  Prints the card's name, power limit
and max SM clock, read in the same run (query only).  Fails without a CUDA device.
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
import torch.nn.functional as F

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


def _fill(buf, rng, E, T, obs_shape, A, frames=False):
    from tianshou_b200.data import Batch
    for _ in range(T):
        if frames:
            obs = np.repeat(rng.integers(0, 256, (E, 1, *obs_shape[1:]), dtype=np.uint8), obs_shape[0], axis=1)
        else:
            obs = rng.standard_normal((E, *obs_shape)).astype(np.float32)
        buf.add(Batch(obs=obs, act=rng.integers(0, A, E), rew=rng.standard_normal(E), terminated=rng.random(E) < 0.01,
                      truncated=np.zeros(E, bool), obs_next=obs), buffer_ids=np.arange(E))


def _setup(workload: str):
    from tianshou_b200.algorithm import DQN, PPO, AdamOptimizerFactory, DiscreteActorPolicy, ICMOffPolicyWrapper, ICMOnPolicyWrapper
    from tianshou_b200.algorithm.modelfree.dqn import DiscreteQLearningPolicy
    from tianshou_b200.data import VectorReplayBuffer
    from tianshou_b200.env.atari.atari_network import DQNet, ScaledObsInputActionReprNet
    from tianshou_b200.utils.net.common import MLP, Net
    from tianshou_b200.utils.net.discrete import DiscreteActor, DiscreteCritic, IntrinsicCuriosityModule
    rng = np.random.default_rng(0)

    def algo_pair(make):
        torch.manual_seed(0)
        a = make()
        torch.manual_seed(0)
        return a, make()

    if workload == "ppo_icm":
        def make():
            net = Net(state_shape=(4,), hidden_sizes=[64, 64])
            actor = DiscreteActor(preprocess_net=net, action_shape=(2,)).to(DEV)
            critic = DiscreteCritic(preprocess_net=net).to(DEV)
            policy = DiscreteActorPolicy(actor=actor, dist_fn=torch.distributions.Categorical, action_space=_Discrete(2))
            return PPO(policy=policy, critic=critic, optim=AdamOptimizerFactory(lr=3e-4), max_grad_norm=0.5, vf_coef=0.5,
                       ent_coef=0.0, gae_lambda=0.95, advantage_normalization=False)
        wrapped, plain = algo_pair(make)
        torch.manual_seed(1)
        icm = IntrinsicCuriosityModule(feature_net=MLP(input_dim=4, output_dim=64, hidden_sizes=[64]), feature_dim=64, action_dim=2,
                                       hidden_sizes=[64]).to(DEV)
        ref = copy.deepcopy(icm)
        algo = ICMOnPolicyWrapper(wrapped_algorithm=wrapped, model=icm, optim=AdamOptimizerFactory(lr=3e-4), lr_scale=1.0,
                                  reward_scale=0.01, forward_loss_weight=0.2)
        buf = VectorReplayBuffer(2000, 10, device=DEV, device_mirror=True)
        _fill(buf, rng, 10, 200, (4,), 2)
        kw, batch_of = dict(batch_size=64, repeat=10), (lambda: buf.sample(0)[0])
    else:
        atari = workload == "atari_icm"
        A = 6 if atari else 2

        def make():
            if atari:
                net = ScaledObsInputActionReprNet(DQNet(c=4, h=84, w=84, action_shape=A)).to(DEV)
            else:
                net = Net(state_shape=(4,), action_shape=A, hidden_sizes=[128, 128, 128]).to(DEV)
            policy = DiscreteQLearningPolicy(model=net, action_space=_Discrete(A))
            return DQN(policy=policy, optim=AdamOptimizerFactory(lr=1e-4 if atari else 1e-3), gamma=0.99, n_step_return_horizon=3,
                       target_update_freq=500 if atari else 320)
        wrapped, plain = algo_pair(make)
        torch.manual_seed(1)
        if atari:
            feat = DQNet(c=4, h=84, w=84, action_shape=A, features_only=True)
            icm = IntrinsicCuriosityModule(feature_net=feat.net, feature_dim=feat.output_dim, action_dim=A, hidden_sizes=[512]).to(DEV)
        else:
            icm = IntrinsicCuriosityModule(feature_net=MLP(input_dim=4, output_dim=128, hidden_sizes=[128, 128]), feature_dim=128,
                                           action_dim=A, hidden_sizes=[128]).to(DEV)
        ref = copy.deepcopy(icm)
        lr = 1e-4 if atari else 1e-3
        algo = ICMOffPolicyWrapper(wrapped_algorithm=wrapped, model=icm, optim=AdamOptimizerFactory(lr=lr),
                                   lr_scale=0.01 if atari else 1.0, reward_scale=0.01, forward_loss_weight=0.2)
        if atari:
            buf = VectorReplayBuffer(100_000, 10, stack_num=4, ignore_obs_next=True, save_only_last_obs=True, device=DEV,
                                     device_mirror=True)
            _fill(buf, rng, 10, 10_000, (4, 84, 84), A, frames=True)
        else:
            buf = VectorReplayBuffer(20_000, 10, device=DEV)
            _fill(buf, rng, 10, 2_000, (4,), A)
        B = 32 if atari else 64
        kw, batch_of = dict(sample_size=B), (lambda: buf[buf.sample_indices(B)])
    opt = torch.optim.Adam(ref.parameters(), lr=algo.optim._optim.param_groups[0]["lr"])
    lr_scale, w = algo.lr_scale, algo.forward_loss_weight

    def eager() -> None:
        batch = batch_of()
        mse, act_hat = ref(batch.obs, batch.act, batch.obs_next)
        act = torch.as_tensor(batch.act, dtype=torch.long, device=DEV)
        loss = ((1 - w) * F.cross_entropy(act_hat, act).mean() + w * mse.mean()) * lr_scale
        _ = batch.rew + (mse * algo.reward_scale).detach().cpu().numpy()
        opt.zero_grad()
        loss.backward()
        opt.step()
        float(loss.item())

    return algo, plain, buf, eager, kw


def run(workload: str, reps: int, warmup: int = 3) -> dict:
    from tianshou_b200 import _cabi
    from tianshou_b200.utils import policy_within_training_step
    algo, plain, buf, eager, kw = _setup(workload)
    launches = {"wrapped": [], "unwrapped": []}

    def device(a, name):
        def fn():
            _cabi.reset_launch_count()
            with policy_within_training_step(a.policy):
                a.update(buffer=buf, **kw)
            launches[name].append(_cabi.launch_count())
        return fn

    np.random.seed(0)
    fns = (("wrapped", device(algo, "wrapped")), ("unwrapped", device(plain, "unwrapped")), ("eager_icm", eager))
    times: dict[str, list[float]] = {k: [] for k, _ in fns}
    for i in range(warmup + reps):
        for name, fn in fns:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            if i >= warmup:
                times[name].append((time.perf_counter() - t0) * 1e3)
    med = {k: float(np.median(v)) for k, v in times.items()}
    return {"workload": workload, "reps": reps, "median_ms": med, "min_ms": {k: min(v) for k, v in times.items()},
            "max_ms": {k: max(v) for k, v in times.items()}, "icm_share_ms": med["wrapped"] - med["unwrapped"],
            "launches": {k: int(np.median(v)) for k, v in launches.items()}}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=21)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/icm_timing.py needs a CUDA device: a time measured anywhere else says nothing")
    out = {"card": card(), "results": [run(w, args.reps) for w in ("dqn_icm", "atari_icm", "ppo_icm")]}
    print(json.dumps(out["card"]))
    for r in out["results"]:
        m, lo, hi = r["median_ms"], r["min_ms"], r["max_ms"]
        print(f"{r['workload']:10s} " + "   ".join(f"{k} {m[k]:8.3f} ms ({lo[k]:.3f} - {hi[k]:.3f})" for k in m)
              + f"   ICM share {r['icm_share_ms']:.3f} ms   launches wrapped {r['launches']['wrapped']}, unwrapped "
              f"{r['launches']['unwrapped']}")
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
