"""TEST INFRASTRUCTURE -- golden vectors for IQN from the UNMODIFIED reference (thu-ml/tianshou 2.0.1 imported through
oracle/ref_shim.py).

    python -m oracle.gen_golden_iqn       # writes tests/golden/iqn_ref_{mlp,sizes,cnn,per}.npz

``iqn_mlp`` is the shape of test/discrete/test_iqn.py shrunk (obs 4, trunk ``Net(hidden [64], action_shape=64)`` so the trunk's
output is linear, ``last`` hidden [64], 2 actions, sizes 32 / 8 / 8, 3-step returns, lagged copies inside the run); ``iqn_sizes``
has unequal online / target sizes (8 / 5), 17 cosines, a trunk ending in ReLU (``Net(action_shape=0, hidden [48])``), ``last``
hidden [40] and 5 actions; ``iqn_cnn`` is ``DQNet(features_only=True)`` behind ``ScaledObsInputActionReprNet`` on stacked 44 x 44
uint8 frames with ``target_update_freq = 0`` (the returns have the ``online_sample_size`` of 8 columns, not the
``target_sample_size`` of 5); ``iqn_per`` draws from a prioritised buffer (test_iqn.py's ``test_piqn``: alpha 0.6, beta 0.4).  Per ``update()``: every fraction tensor the online and
the lagged model draw, in call order (``taus_<k>``, ``u<u>_ntaus`` of them per update), the sampled indices, n-step returns,
loss and priorities (PER: the importance weights and the tree leaves); after the last update every parameter with its Adam
moments, the lagged model, ``_iter`` and the keys of ``state_dict()``.  Every variant is ``compact`` (seeded initial weights,
tensors stored as ``golden_view`` samples).
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

from oracle.gen_golden_discrete_bcq import OUT, fill_buffer, store_final  # noqa: E402  (imports the reference)
from oracle.gen_golden_qrdqn import fill_per_buffer  # noqa: E402
from oracle.oracle_discrete_sac import seeded_params  # noqa: E402
from gymnasium.spaces import Discrete  # noqa: E402  (shim stand-in)
from tianshou.algorithm.modelfree.iqn import IQN, IQNPolicy  # noqa: E402
from tianshou.algorithm.optim import AdamOptimizerFactory  # noqa: E402
from tianshou.env.atari.atari_network import DQNet, ScaledObsInputActionReprNet  # noqa: E402
from tianshou.utils.net.common import Net  # noqa: E402
from tianshou.utils.net.discrete import ImplicitQuantileNetwork  # noqa: E402
from tianshou.utils.torch_utils import policy_within_training_step  # noqa: E402

VARIANTS = {
    "iqn_mlp": dict(kind="mlp", obs=4, hidden=(64,), trunk_out=64, last=(64,), A=2, C=64, S=32, S_on=8, S_t=8, E=4, cap=40,
                    steps=36, bs=48, n_step=3, freq=2, gamma=0.9, lr=1e-3, updates=5, per=False, compact=True, init_seed=61),
    "iqn_sizes": dict(kind="mlp", obs=4, hidden=(48,), trunk_out=0, last=(40,), A=5, C=17, S=32, S_on=8, S_t=5, E=4, cap=40,
                      steps=36, bs=40, n_step=2, freq=3, gamma=0.95, lr=1e-3, updates=5, per=False, compact=True, init_seed=62),
    "iqn_cnn": dict(kind="cnn", H=44, W=44, scale=True, last=(64,), A=6, C=64, S=32, S_on=8, S_t=5, E=4, cap=32, steps=28, bs=16,
                    n_step=1, freq=0, gamma=0.99, lr=1e-4, updates=3, per=False, compact=True, init_seed=63),
    "iqn_per": dict(kind="mlp", obs=4, hidden=(64,), trunk_out=64, last=(64,), A=3, C=64, S=32, S_on=8, S_t=8, E=4, cap=40,
                    steps=36, bs=48, n_step=2, freq=3, gamma=0.95, lr=1e-3, updates=4, per=True, alpha=0.6, beta=0.4, compact=True,
                    init_seed=64),
}


def make_model(cfg):
    if cfg["kind"] == "cnn":
        pre = DQNet(c=4, h=cfg["H"], w=cfg["W"], action_shape=cfg["A"], features_only=True)
        pre = ScaledObsInputActionReprNet(pre) if cfg["scale"] else pre
    else:
        pre = Net(state_shape=(cfg["obs"],), action_shape=cfg["trunk_out"], hidden_sizes=cfg["hidden"])
    return ImplicitQuantileNetwork(preprocess_net=pre, action_shape=cfg["A"], hidden_sizes=cfg["last"], num_cosines=cfg["C"])


def record_taus(module, taus_out):
    """Wrap ``module.forward`` so every fraction tensor it draws is appended to ``taus_out``."""
    orig = module.forward

    def forward(*args, **kwargs):
        (out, taus), hidden = orig(*args, **kwargs)
        taus_out.append(taus.detach().numpy().copy())
        return (out, taus), hidden

    module.forward = forward


def gen(tag: str, cfg: dict) -> None:
    torch.manual_seed(0)
    model = make_model(cfg)
    seeded_params(model, cfg["init_seed"])
    policy = IQNPolicy(model=model, action_space=Discrete(cfg["A"]), sample_size=cfg["S"], online_sample_size=cfg["S_on"],
                       target_sample_size=cfg["S_t"])
    algo = IQN(policy=policy, optim=AdamOptimizerFactory(lr=cfg["lr"]), gamma=cfg["gamma"], n_step_return_horizon=cfg["n_step"],
               target_update_freq=cfg["freq"])
    params = list(policy.parameters())
    out = {"cfg_" + k: np.asarray(v) for k, v in cfg.items()}
    buf = fill_per_buffer(cfg, out) if cfg["per"] else fill_buffer(cfg, out)
    taus: list[np.ndarray] = []
    record_taus(model, taus)
    if cfg["freq"] > 0:
        record_taus(algo.model_old.module, taus)
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
        torch.manual_seed(900 + u)
        n0 = len(taus)
        with policy_within_training_step(algo.policy):
            stats = algo.update(buffer=buf, sample_size=cfg["bs"])
        o = f"u{u}_"
        out[o + "indices"], out[o + "returns"], out[o + "prio"] = captured["indices"], captured["returns"], captured["prio"]
        out[o + "ntaus"] = np.int64(len(taus) - n0)
        if cfg["per"]:
            out[o + "is_weight"] = captured["is_weight"]
            out[o + "tree_leaves"] = np.asarray(buf.weight[np.arange(len(buf))]).copy()
        out[o + "losses"] = np.array([stats.loss], dtype=np.float64)
    for k, t in enumerate(taus):
        out[f"taus_{k}"] = t
    store_final(out, cfg, algo, params, list(algo.model_old.parameters()) if cfg["freq"] > 0 else [])
    np.savez_compressed(os.path.join(OUT, f"{tag.replace('_', '_ref_', 1)}.npz"), **out)
    print(tag, len(out), "arrays;", len(taus), "fraction draws; losses",
          [out[f"u{u}_losses"].round(5).tolist() for u in range(cfg["updates"])])


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    for tag in sys.argv[1:] or list(VARIANTS):
        gen(tag, VARIANTS[tag])
