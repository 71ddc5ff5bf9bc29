"""TEST INFRASTRUCTURE -- golden vectors for discrete BCQ from the UNMODIFIED reference (thu-ml/tianshou 2.0.1 imported
through oracle/ref_shim.py).

    python -m oracle.gen_golden_discrete_bcq       # writes tests/golden/dbcq_ref_{mlp,cnn,sep}.npz

``mlp`` is the shape of test/offline/test_discrete_bcq.py (obs 4, one ``Net`` to 64 under both heads, heads [64, 64], 2 actions,
batch 64, 3-step returns, threshold 0.6); ``cnn`` is the layout of examples/offline/atari_bcq.py on small frames (one
``DQNet(features_only=True)`` ending in Flatten under both heads, stacked uint8 frames); ``sep`` gives each head its own trunk.
Captured: the rollout step by step, per ``update()`` the sampled indices, n-step returns and the four losses, after the last
update every parameter in the optimiser's order with its Adam moments, the lagged model and ``_iter``, and the keys of
``state_dict()``.  The ``cnn`` variant is ``compact`` as in gen_golden_discrete_sac.py: seeded initial weights, tensors stored
as ``golden_view`` samples.
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

from oracle.gen_golden_discrete_sac import frame_rollout, mlp_rollout  # noqa: E402  (imports the reference)
from oracle.oracle_discrete_sac import golden_view, seeded_params  # noqa: E402
from gymnasium.spaces import Discrete  # noqa: E402  (shim stand-in)
from tianshou.algorithm.imitation.discrete_bcq import DiscreteBCQ, DiscreteBCQPolicy  # noqa: E402
from tianshou.algorithm.optim import AdamOptimizerFactory  # noqa: E402
from tianshou.data import Batch, VectorReplayBuffer  # noqa: E402
from tianshou.env.atari.atari_network import DQNet, ScaledObsInputActionReprNet  # noqa: E402
from tianshou.utils.net.common import Net  # noqa: E402
from tianshou.utils.net.discrete import DiscreteActor, DiscreteCritic  # noqa: E402
from tianshou.utils.torch_utils import policy_within_training_step  # noqa: E402

VARIANTS = {
    "mlp": dict(kind="mlp", obs=4, hidden=(), trunk_out=64, last_hidden=(64, 64), A=2, shared=True, E=4, cap=40, steps=36, bs=64,
                n_step=3, tau=0.6, freq=2, penalty=1e-2, gamma=0.99, lr=3e-4, updates=5, compact=False),
    "cnn": dict(kind="cnn", H=44, W=44, hidden=(), trunk_out=0, last_hidden=(32,), A=6, shared=True, E=4, cap=32, steps=28, bs=16,
                n_step=3, tau=0.3, freq=2, penalty=1e-2, gamma=0.99, lr=1e-4, updates=4, compact=True, init_seed=31),
    "sep": dict(kind="mlp", obs=11, hidden=(48,), trunk_out=0, last_hidden=(), A=5, shared=False, E=4, cap=40, steps=36, bs=64,
                n_step=1, tau=0.0, freq=3, penalty=0.5, gamma=0.95, lr=1e-3, updates=4, compact=False),
}


def make_trunk(cfg):
    if cfg["kind"] == "cnn":
        return ScaledObsInputActionReprNet(DQNet(4, cfg["H"], cfg["W"], cfg["A"], features_only=True))
    return Net(state_shape=(cfg["obs"],), action_shape=cfg["trunk_out"], hidden_sizes=cfg["hidden"])


def make_heads(cfg, seed=0):
    """(actor-shaped head, critic-shaped head) on one trunk or one each, as the reference's examples build them."""
    torch.manual_seed(seed)
    t1 = make_trunk(cfg)
    t2 = t1 if cfg["shared"] else make_trunk(cfg)
    a = DiscreteActor(preprocess_net=t1, action_shape=cfg["A"], hidden_sizes=cfg["last_hidden"], softmax_output=False)
    b = DiscreteActor(preprocess_net=t2, action_shape=cfg["A"], hidden_sizes=cfg["last_hidden"], softmax_output=False)
    return a, b


def fill_buffer(cfg, out):
    E, cap = cfg["E"], cfg["cap"]
    cnn = cfg["kind"] == "cnn"
    kw = dict(stack_num=4, ignore_obs_next=True, save_only_last_obs=True) if cnn else {}
    buf = VectorReplayBuffer(E * cap, E, **kw)
    rng = np.random.default_rng(5)
    roll = frame_rollout(rng, E, cfg["steps"], cfg["H"], cfg["W"], cfg["A"]) if cnn else mlp_rollout(rng, E, cfg["steps"], cfg["obs"], cfg["A"])
    for i, s in enumerate(roll):
        for k, v in s.items():
            out[f"roll{i}_{k}"] = v
        if cnn:        # the buffer stores the last frame of each stack; obs_next is never stored
            st = np.repeat(s["obs"][:, None], 4, axis=1)
            s = dict(s, obs=st, obs_next=st)
        buf.add(Batch(info=Batch(), **s), buffer_ids=np.arange(E))
    for k in ("obs", "act", "rew", "terminated", "done") + (() if cnn else ("obs_next",)):
        out["buf_" + k] = np.asarray(buf._meta[k]).copy()
    out["meta_last_index"] = np.asarray(buf.last_index, dtype=np.int64)
    out["meta_lengths"] = np.asarray(buf._lengths, dtype=np.int64)
    return buf


def store_final(out, cfg, algo, params, lagged):
    """Parameters in the optimiser's order with their Adam moments, the lagged parameters, the state_dict keys."""
    view = golden_view if cfg["compact"] else (lambda t: t.detach().numpy().copy())
    opt = algo.optim._optim
    assert [id(p) for p in opt.param_groups[0]["params"]] == [id(p) for p in params]
    for i, p in enumerate(params):
        st = opt.state[p]
        out[f"pf_{i}"], out[f"m_{i}"], out[f"v_{i}"] = view(p), view(st["exp_avg"]), view(st["exp_avg_sq"])
        out["adam_step"] = np.int64(int(st["step"]))
    for i, p in enumerate(lagged):
        out[f"old_{i}"] = view(p)
    out["iter"] = np.int64(algo._iter)
    out["state_dict_keys"] = np.asarray(list(algo.state_dict().keys()))


def gen(tag: str, cfg: dict) -> None:
    model, imitator = make_heads(cfg)
    if cfg["compact"]:
        seeded_params(torch.nn.ModuleList([model, imitator]), cfg["init_seed"])
    policy = DiscreteBCQPolicy(model=model, imitator=imitator, action_space=Discrete(cfg["A"]), target_update_freq=cfg["freq"],
                               unlikely_action_threshold=cfg["tau"])
    algo = DiscreteBCQ(policy=policy, optim=AdamOptimizerFactory(lr=cfg["lr"]), gamma=cfg["gamma"],
                       n_step_return_horizon=cfg["n_step"], target_update_freq=cfg["freq"], imitation_logits_penalty=cfg["penalty"])
    params = list(policy.parameters())
    out = {"cfg_" + k: np.asarray(v) for k, v in cfg.items()}
    if not cfg["compact"]:
        for i, p in enumerate(params):
            out[f"p0_{i}"] = p.detach().numpy().copy()
    buf = fill_buffer(cfg, out)
    captured = {}
    orig_pre = algo._preprocess_batch

    def pre(batch, buffer, indices):
        b = orig_pre(batch, buffer, indices)
        captured["indices"], captured["returns"] = np.asarray(indices).copy(), b.returns.detach().numpy().copy()
        return b

    algo._preprocess_batch = pre
    for u in range(cfg["updates"]):
        np.random.seed(500 + u)
        with policy_within_training_step(algo.policy):
            stats = algo.update(buffer=buf, sample_size=cfg["bs"])
        out[f"u{u}_indices"], out[f"u{u}_returns"] = captured["indices"], captured["returns"]
        out[f"u{u}_losses"] = np.array([stats.loss, stats.q_loss, stats.i_loss, stats.reg_loss], dtype=np.float64)
    store_final(out, cfg, algo, params, list(algo.model_old.parameters()))
    np.savez_compressed(os.path.join(OUT, f"dbcq_ref_{tag}.npz"), **out)
    print(f"dbcq_ref_{tag}.npz", len(out), "arrays; losses", [out[f"u{u}_losses"].round(5).tolist() for u in range(cfg["updates"])])


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    for tag in sys.argv[1:] or list(VARIANTS):
        gen(tag, VARIANTS[tag])
