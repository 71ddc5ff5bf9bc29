"""TEST INFRASTRUCTURE -- golden vectors for the intrinsic curiosity module from the UNMODIFIED reference (thu-ml/tianshou 2.0.1
imported through oracle/ref_shim.py).

    python -m oracle.gen_golden_icm       # writes tests/golden/icm_ref_{dqn_mlp,dqn_per,dqn_cnn,ppo_shared,a2c_sep}.npz

``dqn_mlp`` is test/modelbased/test_dqn_icm.py's construction at reduced widths (``Net`` Q-network, ``MLP`` feature net, ICM hidden
``hidden_sizes[-1:]``, n-step 3, a lagged network); ``dqn_per`` the same on a ``PrioritizedVectorReplayBuffer``; ``dqn_cnn``
examples/atari/atari_dqn.py's ICM branch on small uint8 frames (``DQNet(features_only=True).net`` reading raw frames, the Q-network
behind ``ScaledObsInputActionReprNet``, ``stack_num=4``); ``ppo_shared`` test/modelbased/test_ppo_icm.py's shared ``Net`` under
``DiscreteActor`` / ``DiscreteCritic`` with ``recompute_advantage``; ``a2c_sep`` separate actor and critic nets with an
``LRSchedulerFactoryLinear`` on the ICM optimiser.  Every network starts from ``seeded_params``.

Captured per ``update()``: the sampled indices, the batch's obs / act / obs_next as the reference's buffer delivered them, the
intrinsic reward of every row (the batch's reward after the ICM preprocess minus before), the three ICM losses, the wrapped stats
and, on-policy, the returns and advantages of the first pass.  After the last update: every ICM and wrapped parameter (golden_view)
with its Adam moments, the ICM learning rate, and the keys of ``state_dict()``.
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

from oracle.oracle_discrete_sac import golden_view  # noqa: E402
from oracle.oracle_icm import build, reference_mods  # noqa: E402
from oracle.ref_shim import import_reference  # noqa: E402

ts = import_reference()
from tianshou.data import Batch, PrioritizedVectorReplayBuffer, VectorReplayBuffer  # noqa: E402
from tianshou.utils.torch_utils import policy_within_training_step  # noqa: E402

_OFF = dict(algo="dqn", A=3, E=4, cap=40, steps=36, bs=32, lr=1e-3, updates=4, n_step=3, freq=2, lr_scale=0.3, reward_scale=0.1,
            w=0.2, init_seed=11, icm_seed=12)
VARIANTS = {
    "dqn_mlp": dict(_OFF, kind="mlp", obs=4, hidden=(32, 32), F=32, feat_hidden=(32,), icm_hidden=(32,)),
    "dqn_per": dict(_OFF, kind="mlp", obs=6, A=5, hidden=(24,), F=20, feat_hidden=(24,), icm_hidden=(16,), per=True, alpha=0.6,
                    beta=0.4, w=0.6, lr_scale=2.0),
    "dqn_cnn": dict(_OFF, kind="cnn", H=36, A=6, icm_hidden=(48,), E=4, cap=16, steps=14, bs=12, updates=2, lr=1e-4),
    "ppo_shared": dict(algo="ppo", kind="mlp", obs=4, A=2, hidden=(64, 64), shared=True, F=64, feat_hidden=(64,), icm_hidden=(64,),
                       E=4, steps=32, bs=32, repeat=2, updates=2, lr=1e-3, lr_scale=1.0, reward_scale=0.01, w=0.2, init_seed=21,
                       icm_seed=22),
    "a2c_sep": dict(algo="a2c", kind="mlp", obs=5, A=3, hidden=(48,), shared=False, F=24, feat_hidden=(32,), icm_hidden=(16,),
                    E=4, steps=24, bs=32, repeat=1, updates=3, lr=1e-3, lr_scale=0.5, reward_scale=0.5, w=0.5, init_seed=31,
                    icm_seed=32, sched=True),
}


def rollout(rng, cfg):
    E, A = cfg["E"], cfg["A"]
    out = []
    for _ in range(cfg["steps"]):
        if cfg["kind"] == "cnn":
            obs = rng.integers(0, 256, (E, cfg["H"], cfg["H"]), dtype=np.uint8)
        else:
            obs = rng.standard_normal((E, cfg["obs"])).astype(np.float32)
        term = rng.random(E) < 0.06
        trunc = (rng.random(E) < 0.04) & ~term
        s = dict(obs=obs, act=rng.integers(0, A, E), rew=rng.standard_normal(E), terminated=term, truncated=trunc)
        if cfg["kind"] != "cnn":
            s["obs_next"] = rng.standard_normal((E, cfg["obs"])).astype(np.float32)
        out.append(s)
    return out


def fill_buffer(cfg, out):
    """The rollout into the reference's buffer as tests/offpolicy_testutil.vector_buffer_from_golden replays it (on-policy: a
    buffer of exactly the rollout's size)."""
    E = cfg["E"]
    cap = cfg.get("cap", cfg["steps"])
    cnn = cfg["kind"] == "cnn"
    kw = dict(stack_num=4, ignore_obs_next=True, save_only_last_obs=True) if cnn else {}
    if cfg.get("per"):
        buf = PrioritizedVectorReplayBuffer(E * cap, E, alpha=cfg["alpha"], beta=cfg["beta"], **kw)
    else:
        buf = VectorReplayBuffer(E * cap, E, **kw)
    for i, s in enumerate(rollout(np.random.default_rng(5), cfg)):
        for k, v in s.items():
            out[f"roll{i}_{k}"] = v
        if cnn:
            st = np.repeat(s["obs"][:, None], 4, axis=1)
            s = dict(s, obs=st, obs_next=st)
        buf.add(Batch(info=Batch(), **s), buffer_ids=np.arange(E))
    return buf


def gen(tag: str, cfg: dict) -> None:
    cfg = dict(cfg, compact=True)
    wrapper, algo, icm = build(cfg, reference_mods())
    on_policy = cfg["algo"] in ("ppo", "a2c")
    out = {"cfg_" + k: np.asarray(v) for k, v in cfg.items()}
    buf = fill_buffer(cfg, out)
    cap: dict = {}
    pre_icm, post = wrapper._icm_preprocess_batch, wrapper._postprocess_batch
    pre_wrapped = algo._preprocess_batch

    def icm_pre(batch):
        cap.update(obs=np.asarray(batch.obs).copy(), act=np.asarray(batch.act).copy(), obs_next=np.asarray(batch.obs_next).copy(),
                   rew0=np.asarray(batch.rew, dtype=np.float64).copy())
        pre_icm(batch)
        cap["intrinsic"] = np.asarray(batch.rew, dtype=np.float64) - cap["rew0"]

    def wrapped_pre(batch, buffer, indices):
        cap["indices"] = np.asarray(indices).copy()
        b = pre_wrapped(batch, buffer, indices)
        if on_policy:
            cap["returns"], cap["adv"] = np.asarray(b.returns, np.float64).copy(), np.asarray(b.adv, np.float64).copy()
        return b

    def wrapped_post(batch, buffer, indices):
        post(batch, buffer, indices)
        if cfg.get("per"):
            cap["prio"] = torch.as_tensor(batch.weight).detach().numpy().copy()

    wrapper._icm_preprocess_batch, algo._preprocess_batch, wrapper._postprocess_batch = icm_pre, wrapped_pre, wrapped_post
    for u in range(cfg["updates"]):
        np.random.seed(500 + u)
        with policy_within_training_step(wrapper.policy):
            if on_policy:
                stats = wrapper.update(buffer=buf, batch_size=cfg["bs"], repeat=cfg["repeat"])
            else:
                stats = wrapper.update(buffer=buf, sample_size=cfg["bs"])
        keys = ["indices", "act", "intrinsic"] + (["returns", "adv"] if on_policy else ["obs", "obs_next"])
        keys += ["prio"] if cfg.get("per") else []
        for k in keys:
            out[f"u{u}_{k}"] = cap[k]
        for k in ("icm_loss", "icm_forward_loss", "icm_inverse_loss"):
            out[f"u{u}_{k}"] = np.float64(getattr(stats, k))
        if on_policy:
            out[f"u{u}_loss"] = np.asarray(stats.loss.mean, np.float64)
            if u == 0:
                out["u0_obs"], out["u0_obs_next"] = cap["obs"], cap["obs_next"]
        else:
            out[f"u{u}_loss"] = np.float64(stats.loss)
        out[f"u{u}_icm_lr"] = np.float64(wrapper.optim._optim.param_groups[0]["lr"])
        out[f"u{u}_wrapped_lr"] = np.float64(algo.optim._optim.param_groups[0]["lr"])
    for name, opt, params in (("icm", wrapper.optim._optim, list(icm.parameters())),
                              ("w", algo.optim._optim, list(algo.optim._optim.param_groups[0]["params"]))):
        for i, p in enumerate(params):
            st = opt.state[p]
            out[f"{name}_pf_{i}"], out[f"{name}_m_{i}"], out[f"{name}_v_{i}"] = (golden_view(p), golden_view(st["exp_avg"]),
                                                                                golden_view(st["exp_avg_sq"]))
            out[f"{name}_adam_step"] = np.int64(int(st["step"]))
    sd = wrapper.state_dict()
    out["state_dict_keys"] = np.asarray(list(sd.keys()))
    np.savez_compressed(os.path.join(OUT, f"icm_ref_{tag}.npz"), **out)
    size = os.path.getsize(os.path.join(OUT, f"icm_ref_{tag}.npz"))
    print(f"icm_ref_{tag}.npz {size} bytes; icm losses", [round(float(out[f"u{u}_icm_loss"]), 6) for u in range(cfg["updates"])])


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    for tag in sys.argv[1:] or list(VARIANTS):
        gen(tag, VARIANTS[tag])
