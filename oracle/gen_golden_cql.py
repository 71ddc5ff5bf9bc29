"""TEST INFRASTRUCTURE -- golden vectors for CQL from the UNMODIFIED reference (thu-ml/tianshou 2.0.1 imported through
oracle/ref_shim.py), run on the CPU.

    python -m oracle.gen_golden_cql       # writes tests/golden/cql_ref_{d4rl,nolag,wrap}.npz

Cases:
  d4rl  : the d4rl_cql.py defaults (Lagrange, calibrated, fixed alpha, R = 10) on a ``ReplayBuffer.from_data`` buffer
  nolag : with_lagrange=False, calibrated=False, AutoAlpha, temperature 2, cql_weight 3, an explicit critic2 with its own
          optimiser, min_action=-0.5 (the random actions are uniform in [0.5, 1) instead of all 1.0)
  wrap  : a full buffer that has wrapped around (the positional calibration store), num_repeat_actions=1, alpha_max=0.5 (the
          multiplier is clamped and its gradient is zero)
Captured: the buffer, its calibration returns, the reference's state_dict() keys, and per ``update()`` the sampled indices, the
three losses, alpha / alpha_loss, cql_alpha / cql_alpha_loss / cql_log_alpha, every parameter of the actor, both critics and
both lagged critics, and the torch CPU generator state after the update.
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
from tianshou.algorithm.imitation.cql import CQL  # noqa: E402
from tianshou.algorithm.modelfree.sac import AutoAlpha, SACPolicy  # noqa: E402
from tianshou.algorithm.optim import AdamOptimizerFactory  # noqa: E402
from tianshou.data import Batch, ReplayBuffer  # noqa: E402
from tianshou.utils.net.common import Net  # noqa: E402
from tianshou.utils.net.continuous import ContinuousActorProbabilistic, ContinuousCritic  # noqa: E402
from tianshou.utils.torch_utils import policy_within_training_step  # noqa: E402

VARIANTS = {
    "d4rl": dict(obs=11, act=3, hidden=(32, 32), size=120, adds=0, bs=32, updates=3, actor_lr=1e-4, critic_lr=3e-4, tau=0.005,
                 gamma=0.99, alpha=0.2, auto=False, critic2=False, cql_alpha_lr=3e-4, cql_weight=1.0, temperature=1.0,
                 with_lagrange=True, lagrange_threshold=10.0, min_action=-1.0, max_action=1.0, R=10, alpha_min=0.0,
                 alpha_max=1e6, max_grad_norm=1.0, calibrated=True),
    "nolag": dict(obs=6, act=4, hidden=(24, 24), size=100, adds=0, bs=24, updates=3, actor_lr=1e-3, critic_lr=1e-3, tau=0.01,
                  gamma=0.95, alpha=0.0, auto=True, alpha_lr=3e-3, critic2=True, critic2_lr=5e-4, cql_alpha_lr=1e-4,
                  cql_weight=3.0, temperature=2.0, with_lagrange=False, lagrange_threshold=10.0, min_action=-0.5, max_action=1.0,
                  R=4, alpha_min=0.0, alpha_max=1e6, max_grad_norm=0.5, calibrated=False),
    "wrap": dict(obs=5, act=2, hidden=(16, 16), size=60, adds=97, bs=16, updates=3, actor_lr=1e-3, critic_lr=1e-3, tau=0.005,
                 gamma=0.9, alpha=0.1, auto=False, critic2=False, cql_alpha_lr=1e-3, cql_weight=1.0, temperature=1.0,
                 with_lagrange=True, lagrange_threshold=2.0, min_action=-1.0, max_action=1.0, R=1, alpha_min=0.0,
                 alpha_max=0.5, max_grad_norm=1.0, calibrated=True),
}


def named(mod: torch.nn.Module, prefix: str) -> dict[str, np.ndarray]:
    return {f"{prefix}{i}": p.detach().numpy().copy() for i, p in enumerate(mod.parameters())}


def transitions(rng, n, O, A):
    obs = rng.standard_normal((n, O)).astype(np.float32)
    term = rng.random(n) < 0.05
    trunc = (rng.random(n) < 0.03) & ~term
    return dict(obs=obs, act=np.tanh(rng.standard_normal((n, A))).astype(np.float32), rew=rng.standard_normal(n),
                terminated=term, truncated=trunc, obs_next=rng.standard_normal((n, O)).astype(np.float32))


def build(cfg, seed=0):
    torch.manual_seed(seed)
    O, A, H = cfg["obs"], cfg["act"], cfg["hidden"]
    actor = ContinuousActorProbabilistic(preprocess_net=Net(state_shape=(O,), hidden_sizes=H), action_shape=(A,), unbounded=True,
                                         conditioned_sigma=True)
    crit = lambda: ContinuousCritic(preprocess_net=Net(state_shape=(O,), action_shape=(A,), hidden_sizes=H, concat=True))
    c1 = crit()
    c2 = crit() if cfg["critic2"] else None
    alpha = AutoAlpha(-float(A), 0.0, AdamOptimizerFactory(lr=cfg["alpha_lr"])) if cfg["auto"] else cfg["alpha"]
    policy = SACPolicy(actor=actor, action_space=Box(-1.0, 1.0, (A,)))
    algo = CQL(policy=policy, policy_optim=AdamOptimizerFactory(lr=cfg["actor_lr"]), critic=c1,
               critic_optim=AdamOptimizerFactory(lr=cfg["critic_lr"]), critic2=c2,
               critic2_optim=AdamOptimizerFactory(lr=cfg["critic2_lr"]) if c2 is not None else None, cql_alpha_lr=cfg["cql_alpha_lr"],
               cql_weight=cfg["cql_weight"], tau=cfg["tau"], gamma=cfg["gamma"], alpha=alpha, temperature=cfg["temperature"],
               with_lagrange=cfg["with_lagrange"], lagrange_threshold=cfg["lagrange_threshold"], min_action=cfg["min_action"],
               max_action=cfg["max_action"], num_repeat_actions=cfg["R"], alpha_min=cfg["alpha_min"], alpha_max=cfg["alpha_max"],
               max_grad_norm=cfg["max_grad_norm"], calibrated=cfg["calibrated"])
    return algo


def gen(tag: str, cfg: dict) -> None:
    algo = build(cfg)
    out = {"cfg_" + k: np.asarray(v) for k, v in cfg.items()}
    out.update(named(algo.policy.actor, "p0_actor_")); out.update(named(algo.critic, "p0_c1_")); out.update(named(algo.critic2, "p0_c2_"))
    out["state_dict_keys"] = np.asarray(sorted(algo.state_dict().keys()))
    rng = np.random.default_rng(11)
    O, A = cfg["obs"], cfg["act"]
    if cfg["adds"] == 0:
        d = transitions(rng, cfg["size"], O, A)
        buf = ReplayBuffer.from_data(d["obs"], d["act"], d["rew"], d["terminated"], d["truncated"],
                                     np.logical_or(d["terminated"], d["truncated"]), d["obs_next"])
    else:
        buf = ReplayBuffer(cfg["size"])
        d = transitions(rng, cfg["adds"], O, A)
        for i in range(cfg["adds"]):
            buf.add(Batch(obs=d["obs"][i], act=d["act"][i], rew=d["rew"][i], terminated=d["terminated"][i],
                          truncated=d["truncated"][i], obs_next=d["obs_next"][i], info={}))
    for k in ("obs", "act", "rew", "terminated", "truncated", "done", "obs_next"):
        out["buf_" + k] = np.asarray(buf._meta[k]).copy()
    out["buf_insertion_idx"] = np.int64(buf._insertion_idx)
    out["buf_size"] = np.int64(len(buf))
    buf = algo.process_buffer(buf)
    if cfg["calibrated"]:
        out["calibration_returns"] = np.asarray(buf._meta.calibration_returns).copy()
    captured = {}
    orig_pre = algo._preprocess_batch

    def pre(batch, buffer, indices):
        captured["indices"] = np.asarray(indices).copy()
        return orig_pre(batch, buffer, indices)

    algo._preprocess_batch = pre
    for u in range(cfg["updates"]):
        torch.manual_seed(100 + u)
        with policy_within_training_step(algo.policy):
            stats = algo.update(buf, cfg["bs"])
        o = f"u{u}_"
        out[o + "indices"] = captured["indices"]
        out[o + "losses"] = np.array([stats.actor_loss, stats.critic1_loss, stats.critic2_loss], dtype=np.float64)
        nan = lambda v: np.float64(np.nan if v is None else v)
        out[o + "alpha"], out[o + "alpha_loss"] = nan(stats.alpha), nan(stats.alpha_loss)
        out[o + "cql_alpha"], out[o + "cql_alpha_loss"] = nan(stats.cql_alpha), nan(stats.cql_alpha_loss)
        out[o + "cql_log_alpha"] = np.float64(algo.cql_log_alpha.item())
        if cfg["auto"]:
            out[o + "log_alpha"] = np.float64(algo.alpha._log_alpha.item())
        out[o + "torch_rng"] = torch.get_rng_state().numpy().copy()
        out.update(named(algo.policy.actor, o + "actor_")); out.update(named(algo.critic, o + "c1_"))
        out.update(named(algo.critic2, o + "c2_"))
        out.update(named(algo.critic_old, o + "c1old_")); out.update(named(algo.critic2_old, o + "c2old_"))
    np.savez_compressed(os.path.join(OUT, f"cql_ref_{tag}.npz"), **out)
    print(f"cql_ref_{tag}.npz", len(out), "arrays; losses", [out[f"u{u}_losses"].tolist() for u in range(cfg["updates"])])


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    for tag in sys.argv[1:] or list(VARIANTS):
        gen(tag, VARIANTS[tag])
