"""TEST INFRASTRUCTURE -- golden vectors for imitation learning from the UNMODIFIED reference (thu-ml/tianshou 2.0.1 imported
through oracle/ref_shim.py).

    python -m oracle.gen_golden_imitation       # writes tests/golden/il_ref_{cont,d4rl,disc_sm,disc_logits,cnn,per}.npz

``cont`` is the imitation half of test/continuous/test_sac_with_il.py (``ContinuousActorDeterministic`` over ``Net([128, 128])``,
obs 3, one action dimension, ``max_action`` 2, ``OffPolicyImitationLearning``) on stored actions of which part lies outside +-2, as
SAC's unbounded actor stores them; ``d4rl`` the layout of examples/offline/d4rl_il.py with a smaller hidden width (``Net(action_shape
=6)`` under the actor, so the chain ends ``Linear(h, 6)``, then ``last = Linear(6, 6)``); ``disc_sm`` the imitation half of
test/discrete/test_a2c_with_il.py (``DiscreteActor(Net([64, 64]))`` with its default ``softmax_output=True``, obs 4, 2 actions,
batch 64); ``disc_logits`` a ``DiscreteActor(softmax_output=False)`` over 40 actions, so a row spans two warp passes; ``cnn`` the
layout of examples/offline/atari_il.py on small frames (``DQNet`` over a ``stack_num=4`` uint8 buffer, 6 actions, seeded compact
weights as in gen_golden_discrete_sac.py); ``per`` a ``Net(action_shape=5)`` on a ``PrioritizedVectorReplayBuffer``.

Captured: the rollout step by step, per ``update()`` the sampled indices, the batch's observations and actions as the reference's
buffer delivered them, the loss, and (``per``) the priorities written back; after the last update every parameter in the
optimiser's order with its Adam moments, the optimiser's parameter ids, the keys of ``state_dict()`` and (``per``) the tree's
leaves.
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
from oracle.oracle_imitation import make_actor  # noqa: E402
from oracle.ref_shim import import_reference  # noqa: E402

ts = import_reference()
from gymnasium.spaces import Box, Discrete  # noqa: E402  (shim stand-ins)
from tianshou.algorithm import OffPolicyImitationLearning  # noqa: E402
from tianshou.algorithm.imitation.imitation_base import ImitationPolicy, OfflineImitationLearning  # noqa: E402
from tianshou.algorithm.optim import AdamOptimizerFactory  # noqa: E402
from tianshou.data import Batch, PrioritizedVectorReplayBuffer, VectorReplayBuffer  # noqa: E402
from tianshou.env.atari.atari_network import DQNet  # noqa: E402
from tianshou.utils.net.common import Net  # noqa: E402
from tianshou.utils.net.continuous import ContinuousActorDeterministic  # noqa: E402
from tianshou.utils.net.discrete import DiscreteActor  # noqa: E402
from tianshou.utils.torch_utils import policy_within_training_step  # noqa: E402

VARIANTS = {
    "cont": dict(kind="cont", obs=3, A=1, hidden=(128, 128), net_action=False, max_action=2.0, act_scale=2.5, algo="offpolicy",
                 E=4, cap=40, steps=36, bs=64, lr=1e-3, updates=5, compact=False),
    "d4rl": dict(kind="cont", obs=17, A=6, hidden=(64, 64), net_action=True, max_action=1.0, act_scale=0.6, algo="offline",
                 E=4, cap=40, steps=36, bs=64, lr=1e-3, updates=4, compact=False),
    "disc_sm": dict(kind="mlp", obs=4, A=2, hidden=(64, 64), actor="discrete", softmax=True, algo="offpolicy", E=4, cap=40,
                    steps=36, bs=64, lr=1e-3, updates=5, compact=False),
    "disc_logits": dict(kind="mlp", obs=9, A=40, hidden=(48,), actor="discrete", softmax=False, algo="offpolicy", E=4, cap=40,
                        steps=36, bs=64, lr=1e-3, updates=4, compact=False),
    "cnn": dict(kind="cnn", H=44, W=44, A=6, actor="dqnet", softmax=False, algo="offline", E=4, cap=32, steps=28, bs=16,
                lr=1e-4, updates=3, compact=True, init_seed=51),
    "per": dict(kind="mlp", obs=6, A=5, hidden=(32,), actor="net", softmax=False, algo="offpolicy", per=True, alpha=0.6,
                beta=0.4, E=4, cap=40, steps=36, bs=32, lr=1e-3, updates=4, compact=False),
}


def rollout(rng, cfg):
    E, A = cfg["E"], cfg["A"]
    out = []
    for _ in range(cfg["steps"]):
        if cfg["kind"] == "cnn":
            obs = rng.integers(0, 256, (E, cfg["H"], cfg["W"]), dtype=np.uint8)
        else:
            obs = rng.standard_normal((E, cfg["obs"])).astype(np.float32)
        if cfg["kind"] == "cont":
            act = (rng.standard_normal((E, A)) * cfg["act_scale"]).astype(np.float32)
        else:
            act = rng.integers(0, A, E)
        term = rng.random(E) < 0.06
        trunc = (rng.random(E) < 0.04) & ~term
        s = dict(obs=obs, act=act, rew=rng.standard_normal(E), terminated=term, truncated=trunc)
        if cfg["kind"] != "cnn":
            s["obs_next"] = rng.standard_normal((E, cfg["obs"])).astype(np.float32)
        out.append(s)
    return out


def fill_buffer(cfg, out):
    """The rollout into the reference's buffer as tests/offpolicy_testutil.vector_buffer_from_golden replays it."""
    E, cap = cfg["E"], cfg["cap"]
    cnn = cfg["kind"] == "cnn"
    kw = dict(stack_num=4, ignore_obs_next=True, save_only_last_obs=True) if cnn else {}
    if cfg.get("per"):
        buf = PrioritizedVectorReplayBuffer(E * cap, E, alpha=cfg["alpha"], beta=cfg["beta"], **kw)
    else:
        buf = VectorReplayBuffer(E * cap, E, **kw)
    for i, s in enumerate(rollout(np.random.default_rng(5), cfg)):
        for k, v in s.items():
            out[f"roll{i}_{k}"] = v
        if cnn:        # the buffer stores the last frame of each stack
            st = np.repeat(s["obs"][:, None], 4, axis=1)
            s = dict(s, obs=st, obs_next=st)
        buf.add(Batch(info=Batch(), **s), buffer_ids=np.arange(E))
    return buf


def gen(tag: str, cfg: dict) -> None:
    actor = make_actor(cfg, (Net, ContinuousActorDeterministic, DiscreteActor, DQNet))
    if cfg["compact"]:
        seeded_params(actor, cfg["init_seed"])
    if cfg["kind"] == "cont":
        space = Box(-cfg["max_action"], cfg["max_action"], shape=(cfg["A"],))
        policy = ImitationPolicy(actor=actor, action_space=space, action_scaling=True, action_bound_method="clip")
    else:
        policy = ImitationPolicy(actor=actor, action_space=Discrete(cfg["A"]))
    Algo = OffPolicyImitationLearning if cfg["algo"] == "offpolicy" else OfflineImitationLearning
    algo = Algo(policy=policy, optim=AdamOptimizerFactory(lr=cfg["lr"]))
    params = list(policy.parameters())
    out = {"cfg_" + k: np.asarray(v) for k, v in cfg.items()}
    if not cfg["compact"]:
        for i, p in enumerate(params):
            out[f"p0_{i}"] = p.detach().numpy().copy()
    buf = fill_buffer(cfg, out)
    captured = {}
    orig_pre, orig_post = algo._preprocess_batch, algo._postprocess_batch

    def pre(batch, buffer, indices):
        captured.update(indices=np.asarray(indices).copy(), obs=np.asarray(batch.obs).copy(), act=np.asarray(batch.act).copy())
        return orig_pre(batch, buffer, indices)

    def post(batch, buffer, indices):
        if cfg.get("per"):
            captured["prio"] = np.asarray(batch.weight).copy()
        return orig_post(batch, buffer, indices)

    algo._preprocess_batch, algo._postprocess_batch = pre, post
    for u in range(cfg["updates"]):
        np.random.seed(500 + u)
        with policy_within_training_step(algo.policy):
            stats = algo.update(buffer=buf, sample_size=cfg["bs"])
        for k in ("indices", "obs", "act") + (("prio",) if cfg.get("per") else ()):
            out[f"u{u}_{k}"] = captured[k]
        out[f"u{u}_loss"] = np.float64(stats.loss)
    view = golden_view if cfg["compact"] else (lambda t: t.detach().numpy().copy())
    opt = algo.optim._optim
    assert [id(p) for p in opt.param_groups[0]["params"]] == [id(p) for p in params]
    for i, p in enumerate(params):
        st = opt.state[p]
        out[f"pf_{i}"], out[f"m_{i}"], out[f"v_{i}"] = view(p), view(st["exp_avg"]), view(st["exp_avg_sq"])
        out["adam_step"] = np.int64(int(st["step"]))
    sd = algo.state_dict()
    out["state_dict_keys"] = np.asarray(list(sd.keys()))
    out["optim_param_ids"] = np.asarray(sd["_optimizers"][0]["param_groups"][0]["params"], dtype=np.int64)
    if cfg.get("per"):
        out["prio_leaves"] = np.asarray(buf.weight[np.arange(buf.maxsize)], dtype=np.float64)
    np.savez_compressed(os.path.join(OUT, f"il_ref_{tag}.npz"), **out)
    print(f"il_ref_{tag}.npz", len(out), "arrays; losses", [round(float(out[f"u{u}_loss"]), 6) for u in range(cfg["updates"])])


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    for tag in sys.argv[1:] or list(VARIANTS):
        gen(tag, VARIANTS[tag])
