"""TEST INFRASTRUCTURE -- golden vectors for REDQ from the UNMODIFIED reference (thu-ml/tianshou 2.0.1 imported through
oracle/ref_shim.py), run on the CPU.

    python -m oracle.gen_golden_redq       # writes tests/golden/redq_ref_{mujoco,per_mean,full}.npz

Cases (each runs enough updates for both actor steps and critic-only steps):
  mujoco   : the mujoco_redq.py choices at a small width: E 10, subset 2, ``min``, fixed alpha, n = 1, a ReplayBuffer filled by
             add(), actor_delay 3
  per_mean : a PrioritizedReplayBuffer filled by add() past its capacity, n = 3, episodes ending by termination and by truncation,
             ``mean`` target, E 5 / subset 3, AutoAlpha, actor_delay 2, gamma 0.95, tau 0.01
  full     : the subset is the whole ensemble (4 of 4), actor_delay 1
Captured: the initial weights, the buffer (and the add() sequence that built it), the reference's state_dict() keys, and per
``update()`` the sampled indices, the ensemble subset the update drew, the losses, alpha, every parameter of the actor, the
ensemble and the lagged ensemble, the importance weights of the sample and the priorities after the update (PER).  Before update
u the recipe seeds numpy with 500 + u and torch with 100 + u.
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
from tianshou.algorithm import REDQ  # noqa: E402
from tianshou.algorithm.modelfree.redq import REDQPolicy  # noqa: E402
from tianshou.algorithm.modelfree.sac import AutoAlpha  # noqa: E402
from tianshou.algorithm.optim import AdamOptimizerFactory  # noqa: E402
from tianshou.data import Batch, PrioritizedReplayBuffer, ReplayBuffer  # noqa: E402
from tianshou.utils.net.common import EnsembleLinear, Net  # noqa: E402
from tianshou.utils.net.continuous import ContinuousActorProbabilistic, ContinuousCritic  # noqa: E402
from tianshou.utils.torch_utils import policy_within_training_step  # noqa: E402

_BASE = dict(tau=0.005, gamma=0.99, alpha=0.2, auto_alpha=False, alpha_lr=3e-4, per=False, target_mode="min")
VARIANTS = {
    "mujoco": dict(_BASE, obs=11, act=3, hidden=(32, 32), E=10, M=2, delay=3, size=200, adds=150, bs=32, updates=7, n_step=1,
                   actor_lr=1e-3, critic_lr=1e-3),
    "per_mean": dict(_BASE, obs=7, act=2, hidden=(24, 24), E=5, M=3, delay=2, size=80, adds=110, bs=24, updates=6, n_step=3,
                     actor_lr=1e-3, critic_lr=1e-3, per=True, per_alpha=0.6, per_beta=0.4, target_mode="mean", auto_alpha=True,
                     alpha_lr=3e-3, tau=0.01, gamma=0.95),
    "full": dict(_BASE, obs=5, act=2, hidden=(16, 16), E=4, M=4, delay=1, size=100, adds=90, bs=16, updates=4, n_step=1,
                 actor_lr=1e-3, critic_lr=1e-3, alpha=0.05),
}
KEYS = ("obs", "act", "rew", "terminated", "truncated", "obs_next")


def named(mod: torch.nn.Module, prefix: str) -> dict[str, np.ndarray]:
    return {f"{prefix}{i}": p.detach().numpy().copy() for i, p in enumerate(mod.parameters())}


def transitions(rng, n, O, A):
    """Episodes that end by termination and by truncation."""
    term = rng.random(n) < 0.06
    trunc = (rng.random(n) < 0.05) & ~term
    return dict(obs=rng.standard_normal((n, O)).astype(np.float32), act=np.tanh(rng.standard_normal((n, A))).astype(np.float32),
                rew=rng.standard_normal(n), terminated=term, truncated=trunc, obs_next=rng.standard_normal((n, O)).astype(np.float32))


def build(cfg, seed=0):
    """test/continuous/test_redq.py:85-137 at the variant's sizes."""
    torch.manual_seed(seed)
    O, A, H, E = cfg["obs"], cfg["act"], cfg["hidden"], cfg["E"]
    actor = ContinuousActorProbabilistic(preprocess_net=Net(state_shape=(O,), hidden_sizes=H), action_shape=(A,), unbounded=True,
                                         conditioned_sigma=True)

    def linear(x: int, y: int) -> torch.nn.Module:
        return EnsembleLinear(E, x, y)

    net_c = Net(state_shape=(O,), action_shape=(A,), hidden_sizes=H, concat=True, linear_layer=linear)
    critic = ContinuousCritic(preprocess_net=net_c, linear_layer=linear, flatten_input=False)
    alpha = AutoAlpha(-A, 0.0, AdamOptimizerFactory(lr=cfg["alpha_lr"])) if cfg["auto_alpha"] else cfg["alpha"]
    policy = REDQPolicy(actor=actor, action_space=Box(-1.0, 1.0, (A,)))
    return REDQ(policy=policy, policy_optim=AdamOptimizerFactory(lr=cfg["actor_lr"]), critic=critic,
                critic_optim=AdamOptimizerFactory(lr=cfg["critic_lr"]), ensemble_size=E, subset_size=cfg["M"], tau=cfg["tau"],
                gamma=cfg["gamma"], alpha=alpha, n_step_return_horizon=cfg["n_step"], actor_delay=cfg["delay"],
                target_mode=cfg["target_mode"])


def gen(tag: str, cfg: dict) -> None:
    algo = build(cfg)
    out = {"cfg_" + k: np.asarray(v) for k, v in cfg.items()}
    out.update(named(algo.policy.actor, "p0_actor_")); out.update(named(algo.critic, "p0_critic_"))
    out["state_dict_keys"] = np.asarray(sorted(algo.state_dict().keys()))
    rng = np.random.default_rng(23)
    O, A = cfg["obs"], cfg["act"]
    buf = (PrioritizedReplayBuffer(cfg["size"], alpha=cfg["per_alpha"], beta=cfg["per_beta"]) if cfg["per"]
           else ReplayBuffer(cfg["size"]))
    d = transitions(rng, cfg["adds"], O, A)
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
    orig_choice = np.random.choice

    def choice(*args, **kwargs):         # records the subset draw; the draw itself is numpy's own
        r = orig_choice(*args, **kwargs)
        if kwargs.get("replace", True) is False:
            captured["subset"] = np.asarray(r).copy()
        return r

    np.random.choice = choice
    try:
        for u in range(cfg["updates"]):
            np.random.seed(500 + u)
            torch.manual_seed(100 + u)
            with policy_within_training_step(algo.policy):
                stats = algo.update(buf, cfg["bs"])
            o = f"u{u}_"
            out[o + "indices"] = captured["indices"]
            out[o + "subset"] = captured["subset"]
            out[o + "losses"] = np.array([stats.actor_loss, stats.critic_loss], dtype=np.float64)
            out[o + "alpha"] = np.float64(stats.alpha)
            out[o + "alpha_loss"] = np.float64(np.nan if stats.alpha_loss is None else stats.alpha_loss)
            if cfg["per"]:
                out[o + "is_weight"] = captured["is_weight"]
                out[o + "priorities"] = np.asarray(buf.weight[np.arange(len(buf))], dtype=np.float64).copy()
            out.update(named(algo.policy.actor, o + "actor_")); out.update(named(algo.critic, o + "critic_"))
            out.update(named(algo.critic_old, o + "cold_"))
    finally:
        np.random.choice = orig_choice
    np.savez_compressed(os.path.join(OUT, f"redq_ref_{tag}.npz"), **out)
    print(f"redq_ref_{tag}.npz", len(out), "arrays; losses", [out[f"u{u}_losses"].tolist() for u in range(cfg["updates"])])


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    for tag in sys.argv[1:] or list(VARIANTS):
        gen(tag, VARIANTS[tag])
