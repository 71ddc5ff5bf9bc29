"""TEST INFRASTRUCTURE -- golden vectors for DRQN (DQN on ``Recurrent``) from the UNMODIFIED reference (thu-ml/tianshou 2.0.1
imported through oracle/ref_shim.py).

    python -m oracle.gen_golden_drqn       # writes tests/golden/drqn_ref_{mlp,per,s1}.npz

``drqn_mlp`` is test/discrete/test_drqn.py shrunk (obs 4, 2 actions, ``Recurrent(layer_num=2, hidden 128)``, a ``stack_num=4``
buffer with ``ignore_obs_next=True``, 3-step returns, gamma 0.95, lagged copies inside the run); ``drqn_per`` draws from a
prioritised buffer that stores ``obs_next``, one LSTM layer of 64, ``stack_num=3``, plain (non-double) targets and a Huber loss;
``drqn_s1`` is a ``stack_num=1`` buffer (sequences of one step) with three layers of width 5 and no target network.  Episodes end
inside every buffer, so stacks and n-step chains cross episode starts.
Captured as in gen_golden_c51.py -- per ``update()`` the sampled indices, n-step returns, loss and priorities written back, after
the last update every parameter with its Adam moments, the lagged model, ``_iter``, the keys of ``state_dict()`` and the
optimiser's param indices.  Every variant is ``compact`` (seeded initial weights, tensors stored as ``golden_view`` samples).

On ``drqn_mlp`` the generator checks that the float64 restatement (oracle_drqn.py) reproduces the reference's losses, and that
feeding the newest observation only, or the stack newest first, moves them measurably: the golden pins the sequence order.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

from oracle.gen_golden_discrete_bcq import OUT  # noqa: E402  (imports the reference)
from oracle.gen_golden_discrete_sac import mlp_rollout  # noqa: E402
from oracle import oracle_drqn as od  # noqa: E402
from oracle.oracle_discrete_sac import golden_view, seeded_params  # noqa: E402
from gymnasium.spaces import Discrete  # noqa: E402  (shim stand-in)
from tianshou.algorithm import DQN  # noqa: E402
from tianshou.algorithm.modelfree.dqn import DiscreteQLearningPolicy  # noqa: E402
from tianshou.algorithm.optim import AdamOptimizerFactory  # noqa: E402
from tianshou.data import Batch, PrioritizedVectorReplayBuffer, VectorReplayBuffer  # noqa: E402
from tianshou.utils.net.common import Recurrent  # noqa: E402
from tianshou.utils.torch_utils import policy_within_training_step  # noqa: E402

VARIANTS = {
    "drqn_mlp": dict(obs=4, A=2, layers=2, hidden=128, stack=4, E=4, cap=40, steps=36, bs=64, n_step=3, freq=2, gamma=0.95,
                     lr=1e-3, updates=8, per=False, obs_next=False, double=True, huber=0.0, compact=True, init_seed=71),
    "drqn_per": dict(obs=4, A=3, layers=1, hidden=64, stack=3, E=4, cap=40, steps=36, bs=48, n_step=2, freq=3, gamma=0.9,
                     lr=1e-3, updates=5, per=True, alpha=0.6, beta=0.4, obs_next=True, double=False, huber=1.0, compact=True,
                     init_seed=72),
    "drqn_s1": dict(obs=4, A=2, layers=3, hidden=5, stack=1, E=4, cap=40, steps=36, bs=32, n_step=1, freq=0, gamma=0.99, lr=3e-3,
                    updates=5, per=False, obs_next=False, double=True, huber=0.0, compact=True, init_seed=73),
}


def fill(cfg, out):
    """The flat rollout of gen_golden_discrete_sac into the variant's (prioritised) vector buffer."""
    E, cap = cfg["E"], cfg["cap"]
    kw = dict(stack_num=cfg["stack"], ignore_obs_next=not cfg["obs_next"])
    if cfg["per"]:
        buf = PrioritizedVectorReplayBuffer(E * cap, E, alpha=cfg["alpha"], beta=cfg["beta"], **kw)
    else:
        buf = VectorReplayBuffer(E * cap, E, **kw)
    for i, s in enumerate(mlp_rollout(np.random.default_rng(5), E, cfg["steps"], cfg["obs"], cfg["A"])):
        for k, v in s.items():
            out[f"roll{i}_{k}"] = v
        buf.add(Batch(info=Batch(), **s), buffer_ids=np.arange(E))
    for k in ("obs", "act", "rew", "terminated", "done") + (("obs_next",) if cfg["obs_next"] else ()):
        out["buf_" + k] = np.asarray(buf._meta[k]).copy()
    out["meta_last_index"] = np.asarray(buf.last_index, dtype=np.int64)
    out["meta_lengths"] = np.asarray(buf._lengths, dtype=np.int64)
    return buf


def oracle_losses(cfg, out, order):
    """The float64 restatement's losses on the reference's draws, the sequence fed in ``order``."""
    E, cap = cfg["E"], cfg["cap"]
    buf = {k: out["buf_" + k] for k in ("obs", "act", "rew", "terminated", "done")}
    buf.update(offset=np.arange(E + 1) * cap, last_index=out["meta_last_index"], lengths=out["meta_lengths"])
    ref = Recurrent(layer_num=cfg["layers"], state_shape=cfg["obs"], action_shape=cfg["A"], hidden_layer_size=cfg["hidden"])
    seeded_params(ref, cfg["init_seed"])
    net = od.DrqnNet(cfg["layers"], cfg["obs"], cfg["A"], cfg["hidden"])
    od.load_from(net, list(ref.parameters()))
    old = od.DrqnNet(cfg["layers"], cfg["obs"], cfg["A"], cfg["hidden"]) if cfg["freq"] > 0 else None
    opt = torch.optim.Adam(net.parameters(), lr=cfg["lr"])
    losses = []
    for u in range(cfg["updates"]):
        sync = cfg["freq"] > 0 and u % cfg["freq"] == 0
        if sync and u == 0:
            old.load_state_dict(net.state_dict())
        losses.append(od.drqn_update(net, old, opt, buf, out[f"u{u}_indices"], None, cfg["gamma"], cfg["n_step"], cfg["double"],
                                     cfg["huber"] or None, cfg["stack"], cfg["obs_next"], sync_target=sync and u > 0,
                                     order=order)["loss"])
    return np.array(losses)


def check_order_is_pinned(cfg, out):
    ref = np.array([out[f"u{u}_losses"][0] for u in range(cfg["updates"])])
    mine = oracle_losses(cfg, out, "ref")
    assert np.allclose(mine, ref, rtol=1e-4, atol=1e-6), (mine, ref)
    for order in ("newest_only", "newest_first"):
        gap = np.abs(oracle_losses(cfg, out, order) - ref).max()
        assert gap > 1e-3 * np.abs(ref).max(), f"feeding the stack {order} is within {gap:.2e} of the reference's losses"
        print(f"  {order} off by", float(gap))


def store_final(out, algo, model):
    opt = algo.optim._optim
    params = list(model.parameters())
    assert [id(p) for p in opt.param_groups[0]["params"]] == [id(p) for p in params]
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


def gen(tag: str, cfg: dict) -> None:
    torch.manual_seed(0)
    model = Recurrent(layer_num=cfg["layers"], state_shape=cfg["obs"], action_shape=cfg["A"], hidden_layer_size=cfg["hidden"])
    seeded_params(model, cfg["init_seed"])
    policy = DiscreteQLearningPolicy(model=model, action_space=Discrete(cfg["A"]))
    algo = DQN(policy=policy, optim=AdamOptimizerFactory(lr=cfg["lr"]), gamma=cfg["gamma"], n_step_return_horizon=cfg["n_step"],
               target_update_freq=cfg["freq"], is_double=cfg["double"], huber_loss_delta=cfg["huber"] or None)
    out = {"cfg_" + k: np.asarray(v) for k, v in cfg.items()}
    buf = fill(cfg, out)
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
        np.random.seed(700 + u)
        with policy_within_training_step(algo.policy):
            stats = algo.update(buffer=buf, sample_size=cfg["bs"])
        o = f"u{u}_"
        out[o + "indices"], out[o + "returns"], out[o + "prio"] = captured["indices"], captured["returns"], captured["prio"]
        if cfg["per"]:
            out[o + "is_weight"] = captured["is_weight"]
        out[o + "losses"] = np.array([stats.loss], dtype=np.float64)
    store_final(out, algo, model)
    if tag == "drqn_mlp":
        check_order_is_pinned(cfg, out)
    np.savez_compressed(os.path.join(OUT, f"{tag.replace('_', '_ref_', 1)}.npz"), **out)
    print(tag, len(out), "arrays; losses", [out[f"u{u}_losses"].round(5).tolist() for u in range(cfg["updates"])])


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    for tag in sys.argv[1:] or list(VARIANTS):
        gen(tag, VARIANTS[tag])
