"""TEST INFRASTRUCTURE -- golden vectors for QR-DQN and discrete CQL from the UNMODIFIED reference (thu-ml/tianshou 2.0.1
imported through oracle/ref_shim.py).

    python -m oracle.gen_golden_qrdqn       # writes tests/golden/qrdqn_ref_{mlp,cnn,per}.npz, dcql_ref_{mlp,cnn}.npz

``qrdqn_mlp`` is the shape of test/discrete/test_qrdqn.py shrunk (obs 4, ``Net`` hidden [128, 128], 2 actions, 200 quantiles,
3-step returns, lagged copies inside the run); ``qrdqn_cnn`` is ``QRDQNet`` behind ``ScaledObsInputActionReprNet`` on small
stacked uint8 frames with ``target_update_freq = 0`` and 1-step returns; ``qrdqn_per`` draws from a prioritised buffer;
``dcql_mlp`` is the shape of test/offline/test_discrete_cql.py (hidden [64]); ``dcql_cnn`` the layout of
examples/offline/atari_cql.py on small frames (an unscaled ``QRDQNet``, 1-step returns, ``min_q_weight`` 10).
Captured as in gen_golden_discrete_bcq.py -- per ``update()`` the sampled indices, n-step returns and losses (PER: the importance
weights, the priorities written back and the tree leaves), after the last update every parameter with its Adam moments, the
lagged model, ``_iter`` and the keys of ``state_dict()``.  Every variant is ``compact`` (seeded initial weights, tensors stored
as ``golden_view`` samples) to keep the 200-quantile heads small.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

from oracle.gen_golden_discrete_bcq import OUT, fill_buffer, store_final  # noqa: E402  (imports the reference)
from oracle.gen_golden_discrete_sac import frame_rollout, mlp_rollout  # noqa: E402
from oracle.oracle_discrete_sac import seeded_params  # noqa: E402
from gymnasium.spaces import Discrete  # noqa: E402  (shim stand-in)
from tianshou.algorithm.imitation.discrete_cql import DiscreteCQL  # noqa: E402
from tianshou.algorithm.modelfree.qrdqn import QRDQN, QRDQNPolicy  # noqa: E402
from tianshou.algorithm.optim import AdamOptimizerFactory  # noqa: E402
from tianshou.data import Batch, PrioritizedVectorReplayBuffer  # noqa: E402
from tianshou.env.atari.atari_network import QRDQNet, ScaledObsInputActionReprNet  # noqa: E402
from tianshou.utils.net.common import Net  # noqa: E402
from tianshou.utils.torch_utils import policy_within_training_step  # noqa: E402

VARIANTS = {
    "qrdqn_mlp": dict(algo="qrdqn", kind="mlp", obs=4, hidden=(128, 128), A=2, N=200, E=4, cap=40, steps=36, bs=64, n_step=3,
                      freq=2, gamma=0.9, lr=1e-3, updates=5, per=False, compact=True, init_seed=51),
    "qrdqn_cnn": dict(algo="qrdqn", kind="cnn", H=44, W=44, scale=True, A=6, N=51, E=4, cap=32, steps=28, bs=16, n_step=1,
                      freq=0, gamma=0.99, lr=1e-4, updates=3, per=False, compact=True, init_seed=52),
    "qrdqn_per": dict(algo="qrdqn", kind="mlp", obs=4, hidden=(64,), A=3, N=201, E=4, cap=40, steps=36, bs=48, n_step=2, freq=3,
                      gamma=0.95, lr=1e-3, updates=4, per=True, alpha=0.6, beta=0.4, compact=True, init_seed=53),
    "dcql_mlp": dict(algo="dcql", kind="mlp", obs=4, hidden=(64,), A=2, N=200, E=4, cap=40, steps=36, bs=32, n_step=3, freq=2,
                     gamma=0.99, lr=3e-3, min_q_weight=10.0, updates=5, per=False, compact=True, init_seed=54),
    "dcql_cnn": dict(algo="dcql", kind="cnn", H=44, W=44, scale=False, A=6, N=51, E=4, cap=32, steps=28, bs=16, n_step=1, freq=2,
                     gamma=0.99, lr=1e-4, min_q_weight=10.0, updates=4, per=False, compact=True, init_seed=55),
}


def make_model(cfg):
    if cfg["kind"] == "cnn":
        net = QRDQNet(c=4, h=cfg["H"], w=cfg["W"], action_shape=cfg["A"], num_quantiles=cfg["N"])
        return ScaledObsInputActionReprNet(net) if cfg["scale"] else net
    return Net(state_shape=(cfg["obs"],), action_shape=cfg["A"], hidden_sizes=cfg["hidden"], num_atoms=cfg["N"])


def fill_per_buffer(cfg, out):
    """``fill_buffer``'s rollout into a ``PrioritizedVectorReplayBuffer`` (flat observations)."""
    E, cap = cfg["E"], cfg["cap"]
    buf = PrioritizedVectorReplayBuffer(E * cap, E, alpha=cfg["alpha"], beta=cfg["beta"])
    for i, s in enumerate(mlp_rollout(np.random.default_rng(5), E, cfg["steps"], cfg["obs"], cfg["A"])):
        for k, v in s.items():
            out[f"roll{i}_{k}"] = v
        buf.add(Batch(info=Batch(), **s), buffer_ids=np.arange(E))
    for k in ("obs", "act", "rew", "terminated", "done", "obs_next"):
        out["buf_" + k] = np.asarray(buf._meta[k]).copy()
    out["meta_last_index"] = np.asarray(buf.last_index, dtype=np.int64)
    out["meta_lengths"] = np.asarray(buf._lengths, dtype=np.int64)
    return buf


def gen(tag: str, cfg: dict) -> None:
    torch.manual_seed(0)
    model = make_model(cfg)
    seeded_params(model, cfg["init_seed"])
    policy = QRDQNPolicy(model=model, action_space=Discrete(cfg["A"]))
    kw = dict(policy=policy, optim=AdamOptimizerFactory(lr=cfg["lr"]), gamma=cfg["gamma"], num_quantiles=cfg["N"],
              n_step_return_horizon=cfg["n_step"], target_update_freq=cfg["freq"])
    algo = DiscreteCQL(min_q_weight=cfg["min_q_weight"], **kw) if cfg["algo"] == "dcql" else QRDQN(**kw)
    params = list(policy.parameters())
    out = {"cfg_" + k: np.asarray(v) for k, v in cfg.items()}
    buf = fill_per_buffer(cfg, out) if cfg["per"] else fill_buffer(cfg, out)
    captured = {}
    orig_pre, orig_post = algo._preprocess_batch, algo._postprocess_batch

    def pre(batch, buffer, indices):
        if cfg["per"]:
            captured["is_weight"] = np.asarray(batch.weight).copy()
        b = orig_pre(batch, buffer, indices)
        captured["indices"], captured["returns"] = np.asarray(indices).copy(), b.returns.detach().numpy().copy()
        return b

    def post(batch, buffer, indices):
        captured["prio"] = batch.weight.detach().numpy().copy()
        return orig_post(batch, buffer, indices)

    algo._preprocess_batch, algo._postprocess_batch = pre, post
    for u in range(cfg["updates"]):
        np.random.seed(500 + u)
        with policy_within_training_step(algo.policy):
            stats = algo.update(buffer=buf, sample_size=cfg["bs"])
        o = f"u{u}_"
        out[o + "indices"], out[o + "returns"], out[o + "prio"] = captured["indices"], captured["returns"], captured["prio"]
        if cfg["per"]:
            out[o + "is_weight"] = captured["is_weight"]
            out[o + "tree_leaves"] = np.asarray(buf.weight[np.arange(len(buf))]).copy()
        if cfg["algo"] == "dcql":
            out[o + "losses"] = np.array([stats.loss, stats.qr_loss, stats.cql_loss], dtype=np.float64)
        else:
            out[o + "losses"] = np.array([stats.loss], dtype=np.float64)
    store_final(out, cfg, algo, params, list(algo.model_old.parameters()) if cfg["freq"] > 0 else [])
    np.savez_compressed(os.path.join(OUT, f"{tag.replace('_', '_ref_', 1)}.npz"), **out)
    print(tag, len(out), "arrays; losses", [out[f"u{u}_losses"].round(5).tolist() for u in range(cfg["updates"])])


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    for tag in sys.argv[1:] or list(VARIANTS):
        gen(tag, VARIANTS[tag])
