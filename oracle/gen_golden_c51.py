"""TEST INFRASTRUCTURE -- golden vectors for C51 from the UNMODIFIED reference (thu-ml/tianshou 2.0.1 imported through
oracle/ref_shim.py).

    python -m oracle.gen_golden_c51       # writes tests/golden/c51_ref_{mlp,cnn,per}.npz

``c51_mlp`` is the shape of test/discrete/test_c51.py shrunk (obs 4, ``Net(softmax=True)`` hidden [128, 128], 2 actions, 51
atoms, 3-step returns, lagged copies inside the run); ``c51_cnn`` is ``C51Net`` behind ``ScaledObsInputActionReprNet`` on small
stacked uint8 frames with ``target_update_freq = 0`` and 1-step returns; ``c51_per`` draws from a prioritised buffer with 21
atoms on the asymmetric support [-3, 7] and rewards scaled by 6, so the returns are clamped at both ends.
Captured as in gen_golden_qrdqn.py -- per ``update()`` the sampled indices, n-step returns and loss (PER: the importance
weights, the priorities written back and the tree leaves), after the last update every trainable parameter with its Adam
moments, the lagged model, ``_iter``, the keys of ``state_dict()`` and the optimiser's param indices (``support`` is index 0
and has no state).  Every variant is ``compact`` (seeded initial weights, tensors stored as ``golden_view`` samples).

On ``c51_mlp`` the generator checks that forming the target before the lagged refresh (QR-DQN's order) gives other losses
than the reference's order, so the golden pins the order.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

from oracle.gen_golden_discrete_bcq import OUT, fill_buffer  # noqa: E402  (imports the reference)
from oracle.gen_golden_discrete_sac import mlp_rollout  # noqa: E402
from oracle import oracle_c51 as oc  # noqa: E402
from oracle.oracle_discrete_sac import flat_obs, golden_view, seeded_params  # noqa: E402
from gymnasium.spaces import Discrete  # noqa: E402  (shim stand-in)
from tianshou.algorithm.modelfree.c51 import C51, C51Policy  # noqa: E402
from tianshou.algorithm.optim import AdamOptimizerFactory  # noqa: E402
from tianshou.data import Batch, PrioritizedVectorReplayBuffer  # noqa: E402
from tianshou.env.atari.atari_network import C51Net, ScaledObsInputActionReprNet  # noqa: E402
from tianshou.utils.net.common import Net  # noqa: E402
from tianshou.utils.torch_utils import policy_within_training_step  # noqa: E402

VARIANTS = {
    "c51_mlp": dict(kind="mlp", obs=4, hidden=(128, 128), A=2, N=51, v_min=-10.0, v_max=10.0, E=4, cap=40, steps=36, bs=64,
                    n_step=3, freq=2, gamma=0.9, lr=3e-3, updates=6, per=False, compact=True, init_seed=61),
    "c51_cnn": dict(kind="cnn", H=44, W=44, scale=True, A=6, N=51, v_min=-10.0, v_max=10.0, E=4, cap=32, steps=28, bs=16,
                    n_step=1, freq=0, gamma=0.99, lr=1e-4, updates=3, per=False, compact=True, init_seed=62),
    "c51_per": dict(kind="mlp", obs=4, hidden=(64,), A=3, N=21, v_min=-3.0, v_max=7.0, rew_scale=6.0, E=4, cap=40, steps=36, bs=48,
                    n_step=2, freq=3, gamma=0.95, lr=1e-3, updates=4, per=True, alpha=0.6, beta=0.4, compact=True, init_seed=63),
}


def make_model(cfg):
    if cfg["kind"] == "cnn":
        net = C51Net(c=4, h=cfg["H"], w=cfg["W"], action_shape=cfg["A"], num_atoms=cfg["N"])
        return ScaledObsInputActionReprNet(net) if cfg["scale"] else net
    return Net(state_shape=(cfg["obs"],), action_shape=cfg["A"], hidden_sizes=cfg["hidden"], softmax=True, num_atoms=cfg["N"])


def fill_per_buffer(cfg, out):
    """``fill_buffer``'s flat rollout, rewards times ``rew_scale``, into a ``PrioritizedVectorReplayBuffer``."""
    E, cap = cfg["E"], cfg["cap"]
    buf = PrioritizedVectorReplayBuffer(E * cap, E, alpha=cfg["alpha"], beta=cfg["beta"])
    for i, s in enumerate(mlp_rollout(np.random.default_rng(5), E, cfg["steps"], cfg["obs"], cfg["A"])):
        s = dict(s, rew=s["rew"] * cfg["rew_scale"])
        for k, v in s.items():
            out[f"roll{i}_{k}"] = v
        buf.add(Batch(info=Batch(), **s), buffer_ids=np.arange(E))
    for k in ("obs", "act", "rew", "terminated", "done", "obs_next"):
        out["buf_" + k] = np.asarray(buf._meta[k]).copy()
    out["meta_last_index"] = np.asarray(buf.last_index, dtype=np.int64)
    out["meta_lengths"] = np.asarray(buf._lengths, dtype=np.int64)
    return buf


def store_final(out, algo, policy):
    """The trainable parameters in the optimiser's order (after ``support``) with their Adam moments, the lagged parameters,
    ``_iter``, the state_dict keys and the optimiser's param indices and the indices that have state."""
    opt = algo.optim._optim
    params = list(policy.model.parameters())
    assert [id(p) for p in opt.param_groups[0]["params"]] == [id(policy.support)] + [id(p) for p in params]
    assert policy.support not in opt.state
    for i, p in enumerate(params):
        st = opt.state[p]
        out[f"pf_{i}"], out[f"m_{i}"], out[f"v_{i}"] = golden_view(p), golden_view(st["exp_avg"]), golden_view(st["exp_avg_sq"])
        out["adam_step"] = np.int64(int(st["step"]))
    for i, p in enumerate(algo.model_old.parameters() if algo.use_target_network else []):
        out[f"old_{i}"] = golden_view(p)
    out["iter"] = np.int64(algo._iter)
    sd = algo.state_dict()
    out["state_dict_keys"] = np.asarray(list(sd.keys()))
    osd = sd["_optimizers"][0]
    out["opt_param_ids"] = np.asarray(osd["param_groups"][0]["params"], dtype=np.int64)
    out["opt_state_ids"] = np.asarray(sorted(osd["state"].keys()), dtype=np.int64)


def check_order_is_pinned(cfg, out):
    """The float64 restatement on the reference's draws, once in the reference's order and once with the target formed before
    the lagged refresh: the two must give other losses, else the golden would not tell the orders apart."""
    E, cap = cfg["E"], cfg["cap"]
    buf = dict(obs=out["buf_obs"], obs_next=out["buf_obs_next"], act=out["buf_act"], rew=out["buf_rew"], done=out["buf_done"],
               terminated=out["buf_terminated"], offset=np.arange(E + 1) * cap, last_index=out["meta_last_index"],
               lengths=out["meta_lengths"])
    obs_of = flat_obs(buf["obs"], "cpu")
    losses = {}
    for swapped in (False, True):
        net = oc.net_from_cfg({"cfg_" + k: v for k, v in cfg.items()})
        seeded_params(net, cfg["init_seed"])
        s = oc.C51State(net, cfg["lr"], cfg["freq"], cfg["v_min"], cfg["v_max"])
        losses[swapped] = np.array([oc.c51_update(s, obs_of, buf, out[f"u{u}_indices"], None, cfg["gamma"], cfg["n_step"],
                                                  target_before_tick=swapped)["loss"] for u in range(cfg["updates"])])
    ref = np.array([out[f"u{u}_losses"][0] for u in range(cfg["updates"])])
    assert np.allclose(losses[False], ref, rtol=1e-5, atol=1e-6), (losses[False], ref)
    gap = np.abs(losses[True] - ref).max()
    assert gap > 1e-3 * np.abs(ref).max(), f"the target-before-tick order is within {gap:.2e} of the reference's losses"
    print("  target-before-tick order off by", float(gap))


def gen(tag: str, cfg: dict) -> None:
    torch.manual_seed(0)
    model = make_model(cfg)
    seeded_params(model, cfg["init_seed"])
    policy = C51Policy(model=model, action_space=Discrete(cfg["A"]), num_atoms=cfg["N"], v_min=cfg["v_min"], v_max=cfg["v_max"])
    algo = C51(policy=policy, optim=AdamOptimizerFactory(lr=cfg["lr"]), gamma=cfg["gamma"], n_step_return_horizon=cfg["n_step"],
               target_update_freq=cfg["freq"])
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
        out[o + "losses"] = np.array([stats.loss], dtype=np.float64)
    if cfg["per"]:
        ret = np.concatenate([out[f"u{u}_returns"].reshape(-1) for u in range(cfg["updates"])])
        assert ret.min() < cfg["v_min"] and ret.max() > cfg["v_max"], "the returns must be clamped at both ends"
    store_final(out, algo, policy)
    if tag == "c51_mlp":
        check_order_is_pinned(cfg, out)
    np.savez_compressed(os.path.join(OUT, f"{tag.replace('_', '_ref_', 1)}.npz"), **out)
    print(tag, len(out), "arrays; losses", [out[f"u{u}_losses"].round(5).tolist() for u in range(cfg["updates"])])


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    for tag in sys.argv[1:] or list(VARIANTS):
        gen(tag, VARIANTS[tag])
