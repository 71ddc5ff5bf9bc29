"""TEST INFRASTRUCTURE -- golden vectors for discrete CRR from the UNMODIFIED reference (thu-ml/tianshou 2.0.1 imported
through oracle/ref_shim.py).

    python -m oracle.gen_golden_discrete_crr       # writes tests/golden/dcrr_ref_{mlp,cnn,sep}.npz

``mlp`` is the shape of test/offline/test_discrete_crr.py (obs 4, one ``Net`` to 64 under actor and critic, heads [64, 64],
2 actions, batch 64) in ``"exp"`` mode with an upper bound low enough that the clamp saturates on some rows; ``cnn`` is the
layout of examples/offline/atari_crr.py on small frames (one ``DQNet(features_only=True)`` ending in Flatten under both heads),
``"binary"`` mode, ``target_update_freq = 0``; ``sep`` gives actor and critic a trunk each, ``"all"`` mode, return
standardisation on.  Captured as in gen_golden_discrete_bcq.py; the lagged parameters are ``actor_old``'s then ``critic_old``'s.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

from oracle.gen_golden_discrete_bcq import OUT, fill_buffer, make_trunk, store_final  # noqa: E402  (imports the reference)
from oracle.oracle_discrete_sac import seeded_params  # noqa: E402
from gymnasium.spaces import Discrete  # noqa: E402  (shim stand-in)
from tianshou.algorithm.imitation.discrete_crr import DiscreteCRR  # noqa: E402
from tianshou.algorithm.modelfree.reinforce import DiscreteActorPolicy  # noqa: E402
from tianshou.algorithm.optim import AdamOptimizerFactory  # noqa: E402
from tianshou.utils.net.discrete import DiscreteActor, DiscreteCritic  # noqa: E402
from tianshou.utils.torch_utils import policy_within_training_step  # noqa: E402

VARIANTS = {
    "mlp": dict(kind="mlp", obs=4, hidden=(64,), trunk_out=0, last_hidden=(64, 64), A=2, shared=True, E=4, cap=40, steps=36, bs=64,
                mode="exp", bound=1.05, beta=0.5, min_q_weight=10.0, freq=2, gamma=0.99, lr=3e-4, updates=5, ret_std=False,
                compact=False),
    "cnn": dict(kind="cnn", H=44, W=44, hidden=(), trunk_out=0, last_hidden=(32,), A=6, shared=True, E=4, cap=32, steps=28, bs=16,
                mode="binary", bound=20.0, beta=1.0, min_q_weight=10.0, freq=0, gamma=0.99, lr=1e-4, updates=3, ret_std=False,
                compact=True, init_seed=41),
    "sep": dict(kind="mlp", obs=11, hidden=(48,), trunk_out=0, last_hidden=(), A=5, shared=False, E=4, cap=40, steps=36, bs=64,
                mode="all", bound=20.0, beta=1.0, min_q_weight=2.0, freq=3, gamma=0.95, lr=1e-3, updates=4, ret_std=True,
                compact=False),
}


def gen(tag: str, cfg: dict) -> None:
    torch.manual_seed(0)
    t1 = make_trunk(cfg)
    t2 = t1 if cfg["shared"] else make_trunk(cfg)
    actor = DiscreteActor(preprocess_net=t1, action_shape=cfg["A"], hidden_sizes=cfg["last_hidden"], softmax_output=False)
    critic = DiscreteCritic(preprocess_net=t2, hidden_sizes=cfg["last_hidden"], last_size=cfg["A"])
    if cfg["compact"]:
        seeded_params(torch.nn.ModuleList([actor, critic]), cfg["init_seed"])
    policy = DiscreteActorPolicy(actor=actor, action_space=Discrete(cfg["A"]))
    algo = DiscreteCRR(policy=policy, critic=critic, optim=AdamOptimizerFactory(lr=cfg["lr"]), gamma=cfg["gamma"],
                       policy_improvement_mode=cfg["mode"], ratio_upper_bound=cfg["bound"], beta=cfg["beta"],
                       min_q_weight=cfg["min_q_weight"], target_update_freq=cfg["freq"], return_standardization=cfg["ret_std"])
    params = list(torch.nn.ModuleList([policy, critic]).parameters())
    out = {"cfg_" + k: np.asarray(v) for k, v in cfg.items()}
    if not cfg["compact"]:
        for i, p in enumerate(params):
            out[f"p0_{i}"] = p.detach().numpy().copy()
    buf = fill_buffer(cfg, out)
    captured = {}
    orig_pre = algo._preprocess_batch

    def pre(batch, buffer, indices):
        captured["indices"] = np.asarray(indices).copy()
        return orig_pre(batch, buffer, indices)

    algo._preprocess_batch = pre
    for u in range(cfg["updates"]):
        np.random.seed(500 + u)
        torch.manual_seed(100 + u)
        with policy_within_training_step(algo.policy):
            stats = algo.update(buffer=buf, sample_size=cfg["bs"])
        out[f"u{u}_indices"] = captured["indices"]
        out[f"u{u}_losses"] = np.array([stats.loss, stats.actor_loss, stats.critic_loss, stats.cql_loss], dtype=np.float64)
    lagged = [*algo.actor_old.parameters(), *algo.critic_old.parameters()] if cfg["freq"] > 0 else []
    store_final(out, cfg, algo, params, lagged)
    np.savez_compressed(os.path.join(OUT, f"dcrr_ref_{tag}.npz"), **out)
    print(f"dcrr_ref_{tag}.npz", len(out), "arrays; losses", [out[f"u{u}_losses"].round(5).tolist() for u in range(cfg["updates"])])


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    for tag in sys.argv[1:] or list(VARIANTS):
        gen(tag, VARIANTS[tag])
