"""TEST INFRASTRUCTURE -- golden vectors for FQF from the UNMODIFIED reference (thu-ml/tianshou 2.0.1 imported through
oracle/ref_shim.py).

    python -m oracle.gen_golden_fqf       # writes tests/golden/fqf_ref_{mlp,relu,cnn,per}.npz

``fqf_mlp`` is the shape of test/discrete/test_fqf.py shrunk (obs 4, trunk ``Net(hidden [64], action_shape=64)`` so the trunk's
output is linear, ``last`` hidden [64], 2 actions, 64 cosines, N 32, 3-step returns, lagged copies inside the run, RMSprop on the
fractions, ``ent_coef`` 10); ``fqf_relu`` has a trunk ending in ReLU (``Net(action_shape=0, hidden [48])``), N 13, 17 cosines,
``last`` hidden [40], 5 actions, Adam on the fractions and ``ent_coef`` 0; ``fqf_cnn`` is ``DQNet(features_only=True)`` behind
``ScaledObsInputActionReprNet`` on stacked 44 x 44 uint8 frames with ``target_update_freq = 0``; ``fqf_per`` draws from a
prioritised buffer (alpha 0.6, beta 0.4).  The update draws no random number besides the buffer's indices, so nothing else is
recorded to replay it.  Per ``update()``: the sampled indices, n-step returns, the four statistics (loss, quantile_loss,
fraction_loss, entropy_loss) and priorities (PER: the importance weights and the tree leaves); after the last update every
parameter of both optimisers with its state (Adam's moments, RMSprop's square_avg), the lagged model, ``_iter`` and the keys
of ``state_dict()``.  Every variant is ``compact``: seeded initial weights (the fraction net's by
``oracle_fqf.seed_fraction_net``, far from the reference's near-uniform gain-0.01 start), tensors stored as ``golden_view``
samples.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

from oracle.gen_golden_discrete_bcq import OUT, fill_buffer, store_final  # noqa: E402  (imports the reference)
from oracle.gen_golden_qrdqn import fill_per_buffer  # noqa: E402
from oracle.oracle_discrete_sac import golden_view, seeded_params  # noqa: E402
from oracle.oracle_fqf import seed_fraction_net  # noqa: E402
from gymnasium.spaces import Discrete  # noqa: E402  (shim stand-in)
from tianshou.algorithm.modelfree.fqf import FQF, FQFPolicy  # noqa: E402
from tianshou.algorithm.optim import AdamOptimizerFactory, RMSpropOptimizerFactory  # noqa: E402
from tianshou.env.atari.atari_network import DQNet, ScaledObsInputActionReprNet  # noqa: E402
from tianshou.utils.net.common import Net  # noqa: E402
from tianshou.utils.net.discrete import FractionProposalNetwork, FullQuantileFunction  # noqa: E402
from tianshou.utils.torch_utils import policy_within_training_step  # noqa: E402

VARIANTS = {
    "fqf_mlp": dict(kind="mlp", obs=4, hidden=(64,), trunk_out=64, last=(64,), A=2, C=64, N=32, E=4, cap=40, steps=36, bs=48,
                    n_step=3, freq=2, gamma=0.9, lr=1e-3, frac_opt="rmsprop", frac_lr=1e-4, ent_coef=10.0, updates=3, per=False,
                    compact=True, init_seed=71),
    "fqf_relu": dict(kind="mlp", obs=4, hidden=(48,), trunk_out=0, last=(40,), A=5, C=17, N=13, E=4, cap=40, steps=36, bs=40,
                     n_step=2, freq=3, gamma=0.95, lr=1e-3, frac_opt="adam", frac_lr=1e-3, ent_coef=0.0, updates=5, per=False,
                     compact=True, init_seed=72),
    "fqf_cnn": dict(kind="cnn", H=44, W=44, scale=True, last=(64,), A=6, C=64, N=32, E=4, cap=32, steps=28, bs=16, n_step=1,
                    freq=0, gamma=0.99, lr=1e-4, frac_opt="rmsprop", frac_lr=1e-4, ent_coef=1.0, updates=3, per=False,
                    compact=True, init_seed=73),
    "fqf_per": dict(kind="mlp", obs=4, hidden=(64,), trunk_out=64, last=(64,), A=3, C=64, N=24, E=4, cap=40, steps=36, bs=48,
                    n_step=2, freq=3, gamma=0.95, lr=1e-3, frac_opt="rmsprop", frac_lr=1e-4, ent_coef=10.0, updates=4, per=True,
                    alpha=0.6, beta=0.4, compact=True, init_seed=74),
}


def make_model(cfg):
    if cfg["kind"] == "cnn":
        pre = DQNet(c=4, h=cfg["H"], w=cfg["W"], action_shape=cfg["A"], features_only=True)
        pre = ScaledObsInputActionReprNet(pre) if cfg["scale"] else pre
    else:
        pre = Net(state_shape=(cfg["obs"],), action_shape=cfg["trunk_out"], hidden_sizes=cfg["hidden"])
    model = FullQuantileFunction(preprocess_net=pre, action_shape=cfg["A"], hidden_sizes=cfg["last"], num_cosines=cfg["C"])
    return model, FractionProposalNetwork(cfg["N"], model.input_dim)


def store_fraction_final(out, algo, fm):
    """The fraction net's parameters and its optimiser's state: ``fpf_<i>``, RMSprop's ``fsq_<i>`` or Adam's ``fm_<i>`` /
    ``fv_<i>``, and ``fstep``."""
    opt = algo.fraction_optim._optim
    assert [id(p) for p in opt.param_groups[0]["params"]] == [id(p) for p in fm.parameters()]
    for i, p in enumerate(fm.parameters()):
        st = opt.state[p]
        out[f"fpf_{i}"] = golden_view(p)
        if "square_avg" in st:
            out[f"fsq_{i}"] = golden_view(st["square_avg"])
        else:
            out[f"fm_{i}"], out[f"fv_{i}"] = golden_view(st["exp_avg"]), golden_view(st["exp_avg_sq"])
        out["fstep"] = np.int64(int(st["step"]))


def gen(tag: str, cfg: dict) -> None:
    torch.manual_seed(0)
    model, fm = make_model(cfg)
    seeded_params(model, cfg["init_seed"])
    seed_fraction_net(fm.net, cfg["init_seed"] + 100)
    policy = FQFPolicy(model=model, fraction_model=fm, action_space=Discrete(cfg["A"]))
    frac_factory = (RMSpropOptimizerFactory if cfg["frac_opt"] == "rmsprop" else AdamOptimizerFactory)(lr=cfg["frac_lr"])
    algo = FQF(policy=policy, optim=AdamOptimizerFactory(lr=cfg["lr"]), fraction_optim=frac_factory, gamma=cfg["gamma"],
               num_fractions=cfg["N"], ent_coef=cfg["ent_coef"], n_step_return_horizon=cfg["n_step"],
               target_update_freq=cfg["freq"])
    out = {"cfg_" + k: np.asarray(v) for k, v in cfg.items()}
    buf = fill_per_buffer(cfg, out) if cfg["per"] else fill_buffer(cfg, out)
    with torch.no_grad():        # the first proposal's widths, to show they are far from uniform
        x = torch.as_tensor(np.asarray(buf[np.arange(8)].obs), dtype=torch.float32)
        feat, _ = model.preprocess(x)
        out["init_widths"] = torch.diff(fm(feat)[0], dim=1).numpy()
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
        out[o + "losses"] = np.array([stats.loss, stats.quantile_loss, stats.fraction_loss, stats.entropy_loss], dtype=np.float64)
    store_final(out, cfg, algo, list(model.parameters()), list(algo.model_old.parameters()) if cfg["freq"] > 0 else [])
    store_fraction_final(out, algo, fm)
    out["optimizer_count"] = np.int64(len(algo._optimizers))
    np.savez_compressed(os.path.join(OUT, f"{tag.replace('_', '_ref_', 1)}.npz"), **out)
    print(tag, len(out), "arrays; widths", out["init_widths"].min().round(4), "-", out["init_widths"].max().round(4), "; losses",
          [out[f"u{u}_losses"].round(5).tolist() for u in range(cfg["updates"])])


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    for tag in sys.argv[1:] or list(VARIANTS):
        gen(tag, VARIANTS[tag])
