"""TEST INFRASTRUCTURE -- golden vectors for BDQN from the UNMODIFIED reference (thu-ml/tianshou 2.0.1 imported through
oracle/ref_shim.py), run on the CPU.

    python -m oracle.gen_golden_bdqn       # writes tests/golden/bdqn_ref_{pendulum,bipedal,per_trunc,b1}.npz

Cases:
  pendulum  : test_bdqn.py's network (obs 3, 1 branch of 40 actions, common [64, 64], value [64], action [64]), gamma 0.9, a
              lagged network refreshed inside the recorded updates
  bipedal   : bipedal_bdq.py's branching (obs 24, 4 branches of 25 actions) at a reduced width, a VectorReplayBuffer of 3
              sub-buffers filled by add() (episodes left running, so unfinished_index matters), target_update_freq 2
  per_trunc : a PrioritizedReplayBuffer filled past its capacity, episodes ending by termination and by truncation, no lagged
              network, is_double=False, 9 branches (the branch mean runs over more than 8 values), single-Linear heads, Tanh
  b1        : B = 1, 3 branches, a uniform buffer (the reference's broadcast loss)
Captured: the initial weights, the buffer (and the add() sequence that built it), its end flags' unfinished slots, the
reference's state_dict() keys, and per ``update()`` the sampled indices, the loss, every parameter of the network and of the
lagged network, the importance weights of the sample and the priorities after the update (PER).  Before update u the recipe
seeds numpy with 500 + u and torch with 100 + u.
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
from gymnasium.spaces import MultiDiscrete  # noqa: E402  (shim stand-in)
from tianshou.algorithm import BDQN  # noqa: E402
from tianshou.algorithm.modelfree.bdqn import BDQNPolicy  # noqa: E402
from tianshou.algorithm.optim import AdamOptimizerFactory  # noqa: E402
from tianshou.data import Batch, PrioritizedReplayBuffer, ReplayBuffer, VectorReplayBuffer  # noqa: E402
from tianshou.utils.net.common import BranchingNet  # noqa: E402
from tianshou.utils.torch_utils import policy_within_training_step  # noqa: E402

_BASE = dict(act_fn="relu", per=False, envs=1, target_update_freq=0, is_double=True, gamma=0.99, lr=1e-3)
VARIANTS = {
    "pendulum": dict(_BASE, obs=3, nb=1, A=40, common=(64, 64), value=(64,), action=(64,), gamma=0.9, target_update_freq=3,
                     size=300, adds=200, bs=32, updates=7),
    "bipedal": dict(_BASE, obs=24, nb=4, A=25, common=(48, 32), value=(16,), action=(16,), envs=3, target_update_freq=2,
                    size=240, adds=60, bs=24, updates=5),
    "per_trunc": dict(_BASE, obs=6, nb=9, A=5, common=(24,), value=(), action=(), act_fn="tanh", per=True, per_alpha=0.6,
                      per_beta=0.4, is_double=False, size=80, adds=110, bs=20, updates=5, gamma=0.95, lr=3e-3),
    "b1": dict(_BASE, obs=5, nb=3, A=4, common=(16, 16), value=(8,), action=(8,), target_update_freq=2, size=60, adds=40, bs=1,
               updates=4),
}
KEYS = ("obs", "act", "rew", "terminated", "truncated", "obs_next")


def named(mod: torch.nn.Module, prefix: str) -> dict[str, np.ndarray]:
    return {f"{prefix}{i}": p.detach().numpy().copy() for i, p in enumerate(mod.parameters())}


def transitions(rng, n, O, nb, A):
    """Episodes that end by termination and by truncation."""
    term = rng.random(n) < 0.07
    trunc = (rng.random(n) < 0.06) & ~term
    return dict(obs=rng.standard_normal((n, O)).astype(np.float32), act=rng.integers(0, A, (n, nb)), rew=rng.standard_normal(n),
                terminated=term, truncated=trunc, obs_next=rng.standard_normal((n, O)).astype(np.float32))


def build(cfg, seed=0):
    """test/discrete/test_bdqn.py:84-106 at the variant's sizes."""
    torch.manual_seed(seed)
    act = torch.nn.Tanh if cfg["act_fn"] == "tanh" else torch.nn.ReLU
    net = BranchingNet(state_shape=(cfg["obs"],), num_branches=cfg["nb"], action_per_branch=cfg["A"],
                       common_hidden_sizes=list(cfg["common"]), value_hidden_sizes=list(cfg["value"]),
                       action_hidden_sizes=list(cfg["action"]), activation=act)
    policy = BDQNPolicy(model=net, action_space=MultiDiscrete([cfg["A"]] * cfg["nb"]))
    return BDQN(policy=policy, optim=AdamOptimizerFactory(lr=cfg["lr"]), gamma=cfg["gamma"],
                target_update_freq=cfg["target_update_freq"], is_double=cfg["is_double"])


def make_buffer(cfg):
    if cfg["per"]:
        return PrioritizedReplayBuffer(cfg["size"], alpha=cfg["per_alpha"], beta=cfg["per_beta"])
    if cfg["envs"] > 1:
        return VectorReplayBuffer(cfg["size"], cfg["envs"])
    return ReplayBuffer(cfg["size"])


def fill(buf, d, cfg):
    """``adds`` rows through add(): one transition at a time, or one per sub-buffer of a VectorReplayBuffer."""
    E = cfg["envs"]
    for i in range(0, cfg["adds"], E):
        if E > 1:
            buf.add(Batch(**{k: d[k][i:i + E] for k in KEYS}, info=[{}] * E), buffer_ids=np.arange(E))
        else:
            buf.add(Batch(**{k: d[k][i] for k in KEYS}, info={}))


def gen(tag: str, cfg: dict) -> None:
    algo = build(cfg)
    out = {"cfg_" + k: np.asarray(v) for k, v in cfg.items()}
    out.update(named(algo.policy.model, "p0_net_"))
    out["state_dict_keys"] = np.asarray(sorted(algo.state_dict().keys()))
    rng = np.random.default_rng(29)
    d = transitions(rng, cfg["adds"], cfg["obs"], cfg["nb"], cfg["A"])
    buf = make_buffer(cfg)
    fill(buf, d, cfg)
    for k in KEYS:
        out["add_" + k] = d[k]
    for k in (*KEYS, "done"):
        out["buf_" + k] = np.asarray(buf._meta[k]).copy()
    out["buf_unfinished"] = np.asarray(buf.unfinished_index(), dtype=np.int64)
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
        out[o + "loss"] = np.float64(stats.loss)
        if cfg["per"]:
            out[o + "is_weight"] = captured["is_weight"]
            out[o + "priorities"] = np.asarray(buf.weight[np.arange(len(buf))], dtype=np.float64).copy()
        out.update(named(algo.policy.model, o + "net_"))
        if algo.use_target_network:
            out.update(named(algo.model_old, o + "old_"))
    np.savez_compressed(os.path.join(OUT, f"bdqn_ref_{tag}.npz"), **out)
    print(f"bdqn_ref_{tag}.npz", len(out), "arrays; losses", [float(out[f"u{u}_loss"]) for u in range(cfg["updates"])])


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    for tag in sys.argv[1:] or list(VARIANTS):
        gen(tag, VARIANTS[tag])
