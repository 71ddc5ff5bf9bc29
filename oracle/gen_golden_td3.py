"""TEST INFRASTRUCTURE -- golden vectors for TD3 and TD3+BC from the UNMODIFIED reference (thu-ml/tianshou 2.0.1 imported through
oracle/ref_shim.py), run on the CPU.

    python -m oracle.gen_golden_td3       # writes tests/golden/td3_ref_{mujoco,per_nstep,bc,bc_freq1}.npz

Cases (each runs enough updates for both actor steps and critic-only steps):
  mujoco    : TD3 with its defaults, n = 1, a ReplayBuffer filled by add()
  per_nstep : TD3 on a PrioritizedReplayBuffer filled by add() past its capacity, n = 3, episodes ending by termination and by
              truncation, an explicit critic2 with its own learning rate, update_actor_freq=3, noise_clip=0 (no clamp),
              max_action=2 with action_scaling=False; the noisy target actions leave the action bounds
  bc        : TD3BC with the d4rl_td3_bc.py defaults, n = 3, on a ``ReplayBuffer.from_data`` buffer
  bc_freq1  : TD3BC with update_actor_freq=1 and alpha=1.0
Captured: the initial weights, the buffer (and the add() sequence that built it), the reference's state_dict() keys, and per
``update()`` the sampled indices, the three losses, every parameter of the actor, both critics and the three lagged networks,
the importance weights of the sample and the priorities after the update (PER), and the torch CPU generator state.  Before
update u the recipe seeds numpy with 500 + u (the PER draw) and torch with 100 + u.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "tests", "golden")

from oracle.ref_shim import import_reference  # noqa: E402

ts = import_reference()
from gymnasium.spaces import Box  # noqa: E402  (shim stand-in)
from tianshou.algorithm import TD3  # noqa: E402
from tianshou.algorithm.imitation.td3_bc import TD3BC  # noqa: E402
from tianshou.algorithm.modelfree.ddpg import ContinuousDeterministicPolicy  # noqa: E402
from tianshou.algorithm.optim import AdamOptimizerFactory  # noqa: E402
from tianshou.data import Batch, PrioritizedReplayBuffer, ReplayBuffer  # noqa: E402
from tianshou.utils.net.common import Net  # noqa: E402
from tianshou.utils.net.continuous import ContinuousActorDeterministic, ContinuousCritic  # noqa: E402
from tianshou.utils.torch_utils import policy_within_training_step  # noqa: E402

_BASE = dict(tau=0.005, gamma=0.99, policy_noise=0.2, noise_clip=0.5, freq=2, max_action=1.0, action_scaling=True, critic2=False,
             per=False, adds=0, alpha=2.5)
VARIANTS = {
    "mujoco": dict(_BASE, algo="td3", obs=11, act=3, hidden=(32, 32), size=200, adds=150, bs=32, updates=5, n_step=1,
                   actor_lr=3e-4, critic_lr=3e-4),
    "per_nstep": dict(_BASE, algo="td3", obs=7, act=4, hidden=(24, 24), size=80, adds=110, bs=24, updates=7, n_step=3,
                      actor_lr=1e-3, critic_lr=1e-3, critic2=True, critic2_lr=5e-4, freq=3, noise_clip=0.0, policy_noise=0.6,
                      max_action=2.0, action_scaling=False, per=True, per_alpha=0.6, per_beta=0.4, tau=0.01, gamma=0.95),
    "bc": dict(_BASE, algo="bc", obs=11, act=3, hidden=(32, 32), size=150, bs=32, updates=5, n_step=3, actor_lr=3e-4,
               critic_lr=3e-4),
    "bc_freq1": dict(_BASE, algo="bc", obs=6, act=2, hidden=(16, 16), size=100, bs=16, updates=5, n_step=3, actor_lr=1e-3,
                     critic_lr=1e-3, freq=1, alpha=1.0, gamma=0.9),
}
KEYS = ("obs", "act", "rew", "terminated", "truncated", "obs_next")


def named(mod: torch.nn.Module, prefix: str) -> dict[str, np.ndarray]:
    return {f"{prefix}{i}": p.detach().numpy().copy() for i, p in enumerate(mod.parameters())}


def transitions(rng, n, O, A, max_action):
    """Episodes that end by termination and by truncation."""
    term = rng.random(n) < 0.06
    trunc = (rng.random(n) < 0.05) & ~term
    return dict(obs=rng.standard_normal((n, O)).astype(np.float32),
                act=(max_action * np.tanh(rng.standard_normal((n, A)))).astype(np.float32), rew=rng.standard_normal(n),
                terminated=term, truncated=trunc, obs_next=rng.standard_normal((n, O)).astype(np.float32))


def build(cfg, seed=0):
    torch.manual_seed(seed)
    O, A, H, m = cfg["obs"], cfg["act"], cfg["hidden"], cfg["max_action"]
    actor = ContinuousActorDeterministic(preprocess_net=Net(state_shape=(O,), hidden_sizes=H), action_shape=(A,), max_action=m)
    crit = lambda: ContinuousCritic(preprocess_net=Net(state_shape=(O,), action_shape=(A,), hidden_sizes=H, concat=True))
    c1 = crit()
    c2 = crit() if cfg["critic2"] else None
    policy = ContinuousDeterministicPolicy(actor=actor, action_space=Box(-m, m, (A,)), action_scaling=cfg["action_scaling"])
    kw = dict(policy=policy, policy_optim=AdamOptimizerFactory(lr=cfg["actor_lr"]), critic=c1,
              critic_optim=AdamOptimizerFactory(lr=cfg["critic_lr"]), critic2=c2,
              critic2_optim=AdamOptimizerFactory(lr=cfg["critic2_lr"]) if c2 is not None else None, tau=cfg["tau"],
              gamma=cfg["gamma"], policy_noise=cfg["policy_noise"], update_actor_freq=cfg["freq"], noise_clip=cfg["noise_clip"],
              n_step_return_horizon=cfg["n_step"])
    if cfg["algo"] == "bc":
        return TD3BC(alpha=cfg["alpha"], **kw)
    return TD3(**kw)


def gen(tag: str, cfg: dict) -> None:
    algo = build(cfg)
    out = {"cfg_" + k: np.asarray(v) for k, v in cfg.items()}
    out.update(named(algo.policy.actor, "p0_actor_")); out.update(named(algo.critic, "p0_c1_")); out.update(named(algo.critic2, "p0_c2_"))
    out["state_dict_keys"] = np.asarray(sorted(algo.state_dict().keys()))
    rng = np.random.default_rng(17)
    O, A = cfg["obs"], cfg["act"]
    if cfg["adds"] == 0:
        d = transitions(rng, cfg["size"], O, A, cfg["max_action"])
        # the first and the last slot end episodes: a from_data buffer keeps last_index = [0] while its unfinished slot is the
        # last one, and tianshou_b200's n-step end flags take the unfinished slot from last_index (not reproduced here)
        d["terminated"][[0, -1]], d["truncated"][[0, -1]] = True, False
        buf = ReplayBuffer.from_data(d["obs"], d["act"], d["rew"], d["terminated"], d["truncated"],
                                     np.logical_or(d["terminated"], d["truncated"]), d["obs_next"])
    else:
        buf = (PrioritizedReplayBuffer(cfg["size"], alpha=cfg["per_alpha"], beta=cfg["per_beta"]) if cfg["per"]
               else ReplayBuffer(cfg["size"]))
        d = transitions(rng, cfg["adds"], O, A, cfg["max_action"])
        for i in range(cfg["adds"]):
            buf.add(Batch(**{k: d[k][i] for k in KEYS}, info={}))
        for k in KEYS:
            out["add_" + k] = d[k]
    for k in (*KEYS, "done"):
        out["buf_" + k] = np.asarray(buf._meta[k]).copy()
    out["buf_last_index"] = np.asarray(buf.last_index, dtype=np.int64)
    out["buf_len"] = np.int64(len(buf))
    out["buf_insertion_idx"] = np.int64(buf._insertion_idx)
    captured = {}
    orig_pre = algo._preprocess_batch

    def pre(batch, buffer, indices):
        captured["indices"] = np.asarray(indices).copy()
        if cfg["per"]:
            captured["is_weight"] = np.asarray(batch.weight, dtype=np.float64).copy()
        return orig_pre(batch, buffer, indices)

    algo._preprocess_batch = pre
    for u in range(cfg["updates"]):
        np.random.seed(500 + u)
        torch.manual_seed(100 + u)
        with policy_within_training_step(algo.policy):
            stats = algo.update(buf, cfg["bs"])
        o = f"u{u}_"
        out[o + "indices"] = captured["indices"]
        out[o + "losses"] = np.array([stats.actor_loss, stats.critic1_loss, stats.critic2_loss], dtype=np.float64)
        out[o + "torch_rng"] = torch.get_rng_state().numpy().copy()
        if cfg["per"]:
            out[o + "is_weight"] = captured["is_weight"]
            out[o + "priorities"] = np.asarray(buf.weight[np.arange(len(buf))], dtype=np.float64).copy()
        out.update(named(algo.policy.actor, o + "actor_")); out.update(named(algo.critic, o + "c1_"))
        out.update(named(algo.critic2, o + "c2_")); out.update(named(algo.critic_old, o + "c1old_"))
        out.update(named(algo.critic2_old, o + "c2old_")); out.update(named(algo.actor_old, o + "aold_"))
    np.savez_compressed(os.path.join(OUT, f"td3_ref_{tag}.npz"), **out)
    print(f"td3_ref_{tag}.npz", len(out), "arrays; losses", [out[f"u{u}_losses"].tolist() for u in range(cfg["updates"])])


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    for tag in sys.argv[1:] or list(VARIANTS):
        gen(tag, VARIANTS[tag])
