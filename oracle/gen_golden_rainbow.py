"""TEST INFRASTRUCTURE -- golden vectors for Rainbow DQN from the UNMODIFIED reference (thu-ml/tianshou 2.0.1 imported through
oracle/ref_shim.py).

    python -m oracle.gen_golden_rainbow   # writes tests/golden/rainbow_ref_{mlp,cnn,per,nonoisy,nodueling}.npz

``rainbow_mlp`` is the shape of test/discrete/test_rainbow.py shrunk: ``Net(softmax=True, num_atoms=51, dueling_param=...)``
with noisy Q and V heads at ``noisy_std`` 0.1, 3-step returns and lagged refreshes inside the run (``target_update_freq`` 2).
``rainbow_cnn`` is ``RainbowNet`` behind ``ScaledObsInputActionReprNet`` on small stacked uint8 frames with a lagged network.
``rainbow_per`` draws from a prioritised buffer with 21 atoms on the asymmetric support [-3, 7] and rewards scaled by 6 (the
returns are clamped at both ends), on a noisy trunk (``Net(linear_layer=noisy)``) with a noisy Q head and a plain V head, each
with a hidden layer.  ``rainbow_nonoisy`` and ``rainbow_nodueling`` are ``RainbowNet(is_noisy=False)`` and
``RainbowNet(is_dueling=False)`` (the latter without a lagged network).
Captured as in gen_golden_c51.py -- per ``update()`` the sampled indices, n-step returns, loss and priorities (PER: the
importance weights and the tree leaves) -- plus the noise each ``_sample_noise`` drew (``u<i>_noise_on`` / ``u<i>_noise_old``,
every eps_p, eps_q in ``modules()`` order, concatenated) and both networks' noise after the update (``u<i>_eps_on`` /
``u<i>_eps_old``).  After the last update: every trainable parameter with its Adam moments, the lagged model's trainable
parameters, ``_iter``, the keys of ``state_dict()`` and the optimiser's param indices and the indices with state.  Every variant
is ``compact`` (seeded initial weights, tensors stored as ``golden_view`` samples).

On ``rainbow_mlp`` the generator checks that two alternatives give losses measurably different from the reference's: keeping
the lagged network's own noise on a tick, and forming the target with the mu weights only (eval mode).
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch
from torch import nn

from oracle.gen_golden_c51 import fill_per_buffer  # noqa: E402  (imports the reference)
from oracle.gen_golden_discrete_bcq import OUT, fill_buffer  # noqa: E402
from oracle import oracle_rainbow as orb  # noqa: E402
from oracle.oracle_discrete_sac import flat_obs, golden_view, seeded_params  # noqa: E402
from gymnasium.spaces import Discrete  # noqa: E402  (shim stand-in)
from tianshou.algorithm.modelfree.c51 import C51Policy  # noqa: E402
from tianshou.algorithm.modelfree.rainbow import RainbowDQN  # noqa: E402
from tianshou.algorithm.optim import AdamOptimizerFactory  # noqa: E402
from tianshou.env.atari.atari_network import RainbowNet, ScaledObsInputActionReprNet  # noqa: E402
from tianshou.utils.net.common import Net  # noqa: E402
from tianshou.utils.net.discrete import NoisyLinear  # noqa: E402
from tianshou.utils.torch_utils import policy_within_training_step  # noqa: E402

_MLP = dict(kind="mlp", obs=4, A=2, N=51, v_min=-10.0, v_max=10.0, E=4, cap=40, steps=36, per=False, compact=True)
_CNN = dict(kind="cnn", H=44, W=44, scale=True, A=6, N=51, v_min=-10.0, v_max=10.0, E=4, cap=32, steps=28, bs=16, n_step=1,
            gamma=0.99, lr=1e-4, updates=3, per=False, compact=True, noisy_std=0.5)
VARIANTS = {
    "rainbow_mlp": dict(_MLP, hidden=(64, 64), q_hidden=(), v_hidden=(), trunk_noisy=False, v_noisy=True, noisy_std=0.1, bs=64,
                        n_step=3, freq=2, gamma=0.9, lr=1e-2, updates=8, init_seed=71),
    "rainbow_cnn": dict(_CNN, noisy=True, dueling=True, freq=2, init_seed=72),
    "rainbow_per": dict(_MLP, A=3, N=21, v_min=-3.0, v_max=7.0, rew_scale=6.0, hidden=(64,), q_hidden=(32,), v_hidden=(32,),
                        trunk_noisy=True, v_noisy=False, noisy_std=0.5, bs=48, n_step=2, freq=3, gamma=0.95, lr=1e-3, updates=4,
                        per=True, alpha=0.6, beta=0.4, init_seed=73),
    "rainbow_nonoisy": dict(_CNN, noisy=False, dueling=True, freq=2, init_seed=74),
    "rainbow_nodueling": dict(_CNN, noisy=True, dueling=False, freq=0, init_seed=75),
}


def make_model(cfg):
    if cfg["kind"] == "cnn":
        net = RainbowNet(c=4, h=cfg["H"], w=cfg["W"], action_shape=cfg["A"], num_atoms=cfg["N"], noisy_std=cfg["noisy_std"],
                         is_dueling=cfg["dueling"], is_noisy=cfg["noisy"])
        return ScaledObsInputActionReprNet(net) if cfg["scale"] else net

    def noisy(x: int, y: int) -> NoisyLinear:
        return NoisyLinear(x, y, cfg["noisy_std"])

    return Net(state_shape=(cfg["obs"],), action_shape=cfg["A"], hidden_sizes=cfg["hidden"], softmax=True, num_atoms=cfg["N"],
               linear_layer=noisy if cfg["trunk_noisy"] else nn.Linear,
               dueling_param=({"hidden_sizes": cfg["q_hidden"], "linear_layer": noisy},
                              {"hidden_sizes": cfg["v_hidden"], "linear_layer": noisy if cfg["v_noisy"] else nn.Linear}))


def noise_of(model) -> np.ndarray:
    ts = [e for m in model.modules() if isinstance(m, NoisyLinear) for e in (m.eps_p, m.eps_q)]
    return np.concatenate([t.detach().numpy().reshape(-1) for t in ts]) if ts else np.zeros(0, np.float32)


def store_final(out, algo, policy):
    """The trainable parameters in the optimiser's order with their Adam moments, the lagged trainable parameters, ``_iter``,
    the state_dict keys and the optimiser's param indices and the indices that have state."""
    opt = algo.optim._optim
    params = [p for p in policy.model.parameters() if p.requires_grad]
    assert opt.param_groups[0]["params"][0] is policy.support
    for p in policy.model.parameters():
        if not p.requires_grad:
            assert p not in opt.state, "the noise must never get optimiser state"
    for i, p in enumerate(params):
        st = opt.state[p]
        out[f"pf_{i}"], out[f"m_{i}"], out[f"v_{i}"] = golden_view(p), golden_view(st["exp_avg"]), golden_view(st["exp_avg_sq"])
        out["adam_step"] = np.int64(int(st["step"]))
    old = [p for p in algo.model_old.parameters() if p.requires_grad] if algo.use_target_network else []
    for i, p in enumerate(old):
        out[f"old_{i}"] = golden_view(p)
    out["iter"] = np.int64(algo._iter)
    sd = algo.state_dict()
    out["state_dict_keys"] = np.asarray(list(sd.keys()))
    osd = sd["_optimizers"][0]
    out["opt_param_ids"] = np.asarray(osd["param_groups"][0]["params"], dtype=np.int64)
    out["opt_state_ids"] = np.asarray(sorted(osd["state"].keys()), dtype=np.int64)


def check_order_is_pinned(cfg, out):
    """The restatement on the reference's draws and noise, in the reference's way and in the two alternatives: each must give
    other losses, else the golden would not tell it apart."""
    E, cap = cfg["E"], cfg["cap"]
    buf = dict(obs=out["buf_obs"], obs_next=out["buf_obs_next"], act=out["buf_act"], rew=out["buf_rew"], done=out["buf_done"],
               terminated=out["buf_terminated"], offset=np.arange(E + 1) * cap, last_index=out["meta_last_index"],
               lengths=out["meta_lengths"])
    obs_of = flat_obs(buf["obs"], "cpu")
    losses = {}
    for alt in ("reference", "keep_lagged_noise", "target_eval"):
        net = orb.rainbow_net(cfg)
        seeded_params(net, cfg["init_seed"])
        s = orb.RainbowState(net, cfg["lr"], cfg["freq"], cfg["v_min"], cfg["v_max"])
        losses[alt] = np.array([orb.rainbow_update(s, obs_of, buf, out[f"u{u}_indices"], None, cfg["gamma"], cfg["n_step"],
                                                   out[f"u{u}_noise_on"], out[f"u{u}_noise_old"],
                                                   keep_lagged_noise=alt == "keep_lagged_noise",
                                                   target_eval=alt == "target_eval")["loss"] for u in range(cfg["updates"])])
    ref = np.array([out[f"u{u}_losses"][0] for u in range(cfg["updates"])])
    assert np.allclose(losses["reference"], ref, rtol=1e-5, atol=1e-6), (losses["reference"], ref)
    for alt in ("keep_lagged_noise", "target_eval"):
        gap = np.abs(losses[alt] - ref).max()
        assert gap > 1e-3 * np.abs(ref).max(), f"{alt} is within {gap:.2e} of the reference's losses"
        print(f"  {alt} off by", float(gap))


def gen(tag: str, cfg: dict) -> None:
    torch.manual_seed(0)
    model = make_model(cfg)
    seeded_params(model, cfg["init_seed"])
    policy = C51Policy(model=model, action_space=Discrete(cfg["A"]), num_atoms=cfg["N"], v_min=cfg["v_min"], v_max=cfg["v_max"])
    algo = RainbowDQN(policy=policy, optim=AdamOptimizerFactory(lr=cfg["lr"]), gamma=cfg["gamma"],
                      n_step_return_horizon=cfg["n_step"], target_update_freq=cfg["freq"])
    out = {"cfg_" + k: np.asarray(v) for k, v in cfg.items()}
    buf = fill_per_buffer(cfg, out) if cfg["per"] else fill_buffer(cfg, out)
    captured = {}
    orig_pre, orig_post, orig_noise = algo._preprocess_batch, algo._postprocess_batch, algo._sample_noise

    def pre(batch, buffer, indices):
        if cfg["per"]:
            captured["is_weight"] = np.asarray(batch.weight).copy()
        b = orig_pre(batch, buffer, indices)
        captured["indices"], captured["returns"] = np.asarray(indices).copy(), b.returns.detach().numpy().copy()
        return b

    def post(batch, buffer, indices):
        captured["prio"] = batch.weight.detach().numpy().copy()
        return orig_post(batch, buffer, indices)

    def noise(m):
        found = orig_noise(m)
        captured["noise_on" if m is policy.model else "noise_old"] = noise_of(m)
        return found

    algo._preprocess_batch, algo._postprocess_batch, algo._sample_noise = pre, post, noise
    for u in range(cfg["updates"]):
        np.random.seed(500 + u)
        captured["noise_old"] = np.zeros(0, np.float32)
        with policy_within_training_step(algo.policy):
            stats = algo.update(buffer=buf, sample_size=cfg["bs"])
        o = f"u{u}_"
        out[o + "indices"], out[o + "returns"], out[o + "prio"] = captured["indices"], captured["returns"], captured["prio"]
        out[o + "noise_on"], out[o + "noise_old"] = captured["noise_on"], captured["noise_old"]
        out[o + "eps_on"] = noise_of(policy.model)
        out[o + "eps_old"] = noise_of(algo.model_old) if algo.use_target_network else np.zeros(0, np.float32)
        if cfg["per"]:
            out[o + "is_weight"] = captured["is_weight"]
            out[o + "tree_leaves"] = np.asarray(buf.weight[np.arange(len(buf))]).copy()
        out[o + "losses"] = np.array([stats.loss], dtype=np.float64)
    if cfg["per"]:
        ret = np.concatenate([out[f"u{u}_returns"].reshape(-1) for u in range(cfg["updates"])])
        assert ret.min() < cfg["v_min"] and ret.max() > cfg["v_max"], "the returns must be clamped at both ends"
    store_final(out, algo, policy)
    if tag == "rainbow_mlp":
        check_order_is_pinned(cfg, out)
    np.savez_compressed(os.path.join(OUT, f"{tag.replace('_', '_ref_', 1)}.npz"), **out)
    print(tag, len(out), "arrays; losses", [out[f"u{u}_losses"].round(5).tolist() for u in range(cfg["updates"])])


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    for tag in sys.argv[1:] or list(VARIANTS):
        gen(tag, VARIANTS[tag])
