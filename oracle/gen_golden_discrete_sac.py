"""TEST INFRASTRUCTURE -- golden vectors for discrete SAC from the UNMODIFIED reference (thu-ml/tianshou 2.0.1 imported
through oracle/ref_shim.py).

    python -m oracle.gen_golden_discrete_sac       # writes tests/golden/dsac_ref_{mlp,auto,cnn}.npz

Captured per ``update()``: sampled indices, n-step returns, IS weights, the priority-update TD errors (``batch.weight``), the
three losses, alpha / alpha_loss / log_alpha, every parameter of the actor, both critics and both lagged critics, the PER
tree leaves, and the torch CPU generator state after the update (the reference draws two discarded Categorical samples).
The NatureCNN variant is ``compact``: its ~82 k parameters per network would make the file several MB, so its initial
weights come from ``oracle_discrete_sac.seeded_params`` (the seed is stored, not the tensors) and its parameters are stored
after the last update only, each tensor as ``oracle_discrete_sac.golden_view`` (a fixed-stride sample of at most 2048
elements; the full tensors' gradients are checked against float64 autograd in tests/test_discrete_sac_gpu.py).
The rollout is stored step by step so the tests can replay it into a tianshou_b200 buffer with ``add``.
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

from oracle.oracle_discrete_sac import golden_view, seeded_params  # noqa: E402
from oracle.ref_shim import import_reference  # noqa: E402

ts = import_reference()
from gymnasium.spaces import Discrete  # noqa: E402  (shim stand-in)
from tianshou.algorithm import DiscreteSAC  # noqa: E402
from tianshou.algorithm.modelfree.discrete_sac import DiscreteSACPolicy  # noqa: E402
from tianshou.algorithm.modelfree.sac import AutoAlpha  # noqa: E402
from tianshou.algorithm.optim import AdamOptimizerFactory  # noqa: E402
from tianshou.data import Batch, PrioritizedVectorReplayBuffer, VectorReplayBuffer  # noqa: E402
from tianshou.env.atari.atari_network import DQNet, ScaledObsInputActionReprNet  # noqa: E402
from tianshou.utils.net.common import Net  # noqa: E402
from tianshou.utils.net.discrete import DiscreteActor, DiscreteCritic  # noqa: E402
from tianshou.utils.torch_utils import policy_within_training_step  # noqa: E402

VARIANTS = {
    "mlp": dict(kind="mlp", obs=11, A=5, hidden=(48, 40), E=4, cap=40, steps=36, bs=64, n_step=3, updates=3, actor_lr=3e-4,
                critic_lr=1e-3, tau=0.005, gamma=0.95, alpha=0.05, auto=False, per=True, per_alpha=0.6, per_beta=0.4,
                critic2=True, compact=False),
    "auto": dict(kind="mlp", obs=4, A=2, hidden=(64, 64), E=4, cap=40, steps=36, bs=64, n_step=1, updates=4, actor_lr=1e-4,
                 critic_lr=1e-3, tau=0.005, gamma=0.95, alpha=0.0, auto=True, alpha_lr=3e-4, per=False, critic2=False,
                 compact=False),
    "cnn": dict(kind="cnn", H=36, W=36, feat=64, A=6, E=4, cap=32, steps=28, bs=16, n_step=3, updates=3, actor_lr=3e-4,
                critic_lr=1e-3, tau=0.005, gamma=0.99, alpha=0.05, auto=False, per=True, per_alpha=0.6, per_beta=0.4,
                critic2=True, compact=True, init_seed=21),
}


def named(mod: torch.nn.Module, prefix: str, compact: bool = False) -> dict[str, np.ndarray]:
    return {f"{prefix}{i}": golden_view(p) if compact else p.detach().numpy().copy() for i, p in enumerate(mod.parameters())}


def mlp_rollout(rng, E, steps, obs_dim, A):
    out = []
    obs = rng.standard_normal((E, obs_dim)).astype(np.float32)
    for _ in range(steps):
        act = rng.integers(0, A, E)
        rew = rng.standard_normal(E)
        obs_next = rng.standard_normal((E, obs_dim)).astype(np.float32)
        term = rng.random(E) < 0.06
        trunc = (rng.random(E) < 0.04) & ~term
        out.append(dict(obs=obs, act=act, rew=rew, terminated=term, truncated=trunc, obs_next=obs_next))
        done = term | trunc
        obs = np.where(done[:, None], rng.standard_normal((E, obs_dim)).astype(np.float32), obs_next)
    return out


def frame_rollout(rng, E, steps, H, W, A):
    """uint8 single frames: the stored obs is the last frame of the stack (save_only_last_obs)."""
    out = []
    for _ in range(steps):
        frame = rng.integers(0, 256, (E, H, W), dtype=np.uint8)
        act = rng.integers(0, A, E)
        rew = rng.standard_normal(E)
        term = rng.random(E) < 0.08
        trunc = (rng.random(E) < 0.03) & ~term
        out.append(dict(obs=frame, act=act, rew=rew, terminated=term, truncated=trunc))
    return out


def build(cfg, seed=0):
    torch.manual_seed(seed)
    A = cfg["A"]
    if cfg["kind"] == "mlp":
        trunk = lambda: Net(state_shape=(cfg["obs"],), hidden_sizes=cfg["hidden"])
    else:
        trunk = lambda: ScaledObsInputActionReprNet(DQNet(4, cfg["H"], cfg["W"], A, features_only=True,
                                                          output_dim_added_layer=cfg["feat"]))
    actor = DiscreteActor(preprocess_net=trunk(), action_shape=A, softmax_output=False)
    c1 = DiscreteCritic(preprocess_net=trunk(), last_size=A)
    c2 = DiscreteCritic(preprocess_net=trunk(), last_size=A) if cfg["critic2"] else None
    if cfg["compact"]:
        for k, m in enumerate((actor, c1, c2)):
            if m is not None:
                seeded_params(m, cfg["init_seed"] + k)
    if cfg["auto"]:
        alpha = AutoAlpha(0.98 * np.log(A), 0.0, AdamOptimizerFactory(lr=cfg["alpha_lr"]))
    else:
        alpha = cfg["alpha"]
    policy = DiscreteSACPolicy(actor=actor, action_space=Discrete(A))
    algo = DiscreteSAC(policy=policy, policy_optim=AdamOptimizerFactory(lr=cfg["actor_lr"]), critic=c1,
                       critic_optim=AdamOptimizerFactory(lr=cfg["critic_lr"]), critic2=c2,
                       critic2_optim=AdamOptimizerFactory(lr=cfg["critic_lr"]) if c2 is not None else None, tau=cfg["tau"],
                       gamma=cfg["gamma"], alpha=alpha, n_step_return_horizon=cfg["n_step"])
    return algo


def gen(tag: str, cfg: dict) -> None:
    algo = build(cfg)
    out = {"cfg_" + k: np.asarray(v) for k, v in cfg.items() if k != "kind"}
    out["cfg_kind"] = np.asarray(cfg["kind"])
    if not cfg["compact"]:
        out.update(named(algo.policy.actor, "p0_actor_")); out.update(named(algo.critic, "p0_c1_")); out.update(named(algo.critic2, "p0_c2_"))
    E, cap = cfg["E"], cfg["cap"]
    kw = dict(stack_num=4, ignore_obs_next=True, save_only_last_obs=True) if cfg["kind"] == "cnn" else {}
    if cfg["per"]:
        buf = PrioritizedVectorReplayBuffer(E * cap, E, alpha=cfg["per_alpha"], beta=cfg["per_beta"], **kw)
    else:
        buf = VectorReplayBuffer(E * cap, E, **kw)
    rng = np.random.default_rng(5)
    if cfg["kind"] == "mlp":
        roll = mlp_rollout(rng, E, cfg["steps"], cfg["obs"], cfg["A"])
    else:
        roll = frame_rollout(rng, E, cfg["steps"], cfg["H"], cfg["W"], cfg["A"])
    for i, s in enumerate(roll):
        for k, v in s.items():
            out[f"roll{i}_{k}"] = v
        if cfg["kind"] == "cnn":        # the buffer stores the last frame of each stack; obs_next is never stored
            st = np.repeat(s["obs"][:, None], 4, axis=1)
            s = dict(s, obs=st, obs_next=st)
        buf.add(Batch(**s), buffer_ids=np.arange(E))
    for k in ("obs", "act", "rew", "terminated", "done") + (("obs_next",) if cfg["kind"] == "mlp" else ()):
        out["buf_" + k] = np.asarray(buf._meta[k]).copy()
    out["meta_last_index"] = np.asarray(buf.last_index, dtype=np.int64)
    out["meta_lengths"] = np.asarray(buf._lengths, dtype=np.int64)
    captured = {}
    orig_pre, orig_post = algo._preprocess_batch, algo._postprocess_batch

    def pre(batch, buffer, indices):
        if cfg["per"]:
            captured["is_weight"] = np.asarray(batch.weight).copy()
        b = orig_pre(batch, buffer, indices)
        captured["indices"] = np.asarray(indices).copy()
        captured["returns"] = b.returns.detach().numpy().copy()
        return b

    def post(batch, buffer, indices):
        captured["weight"] = batch.weight.detach().numpy().copy()
        return orig_post(batch, buffer, indices)

    algo._preprocess_batch, algo._postprocess_batch = pre, post
    for u in range(cfg["updates"]):
        np.random.seed(500 + u)
        torch.manual_seed(100 + u)
        with policy_within_training_step(algo.policy):
            stats = algo.update(buffer=buf, sample_size=cfg["bs"])
        o = f"u{u}_"
        out[o + "indices"], out[o + "returns"], out[o + "weight"] = captured["indices"], captured["returns"], captured["weight"]
        if cfg["per"]:
            out[o + "is_weight"] = captured["is_weight"]
            out[o + "tree_leaves"] = np.asarray(buf.weight[np.arange(len(buf))]).copy()
        out[o + "losses"] = np.array([stats.actor_loss, stats.critic1_loss, stats.critic2_loss], dtype=np.float64)
        out[o + "alpha"] = np.float64(stats.alpha)
        out[o + "alpha_loss"] = np.float64(np.nan if stats.alpha_loss is None else stats.alpha_loss)
        if cfg["auto"]:
            out[o + "log_alpha"] = np.float64(algo.alpha._log_alpha.item())
        out[o + "torch_rng"] = torch.get_rng_state().numpy().copy()
        c = cfg["compact"]
        if c and u < cfg["updates"] - 1:
            continue        # compact: parameters after the LAST update only (every earlier step feeds into them)
        out.update(named(algo.policy.actor, o + "actor_", c)); out.update(named(algo.critic, o + "c1_", c))
        out.update(named(algo.critic2, o + "c2_", c))
        out.update(named(algo.critic_old, o + "c1old_", c)); out.update(named(algo.critic2_old, o + "c2old_", c))
    np.savez_compressed(os.path.join(OUT, f"dsac_ref_{tag}.npz"), **out)
    print(f"dsac_ref_{tag}.npz", len(out), "arrays; losses", [out[f"u{u}_losses"].tolist() for u in range(cfg["updates"])])


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    for tag in sys.argv[1:] or list(VARIANTS):
        gen(tag, VARIANTS[tag])
