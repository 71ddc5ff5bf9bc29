"""TEST INFRASTRUCTURE -- golden vectors for the on-policy update with torch.optim.RMSprop, from the UNMODIFIED reference
(thu-ml/tianshou 2.0.1 imported from /root/reference through oracle/ref_shim.py).

    python -m oracle.gen_golden_rmsprop      # writes tests/golden/a2c_rmsprop_ref*.npz, tests/golden/npg_rmsprop_ref.npz

  a2c_rmsprop_ref.npz     A2C with examples/mujoco/mujoco_a2c.py's optimiser (RMSprop lr 7e-4, eps 1e-5, alpha 0.99),
                          max_grad_norm 0.5 and a linear LR schedule that halves the lr for the second update; obs 17 /
                          act 6, tanh [64, 64] actor and critic (the fused tensor-core shape).
  a2c_rmsprop_ref_C1.npz  A2C with the same optimiser on the reference's discrete shared-ReLU-trunk network
                          (test/discrete/test_ppo_discrete.py:90-100, the ppo_ref_C1 family; the SIMT kernels).
  npg_rmsprop_ref.npz     NPG whose critic optimiser is RMSprop (the layer-wise critic step), built by gen_golden_npg.

Same capture as gen_golden.gen_a2c / gen_golden_npg.gen, plus the lr every update ran at (``u{u}_lr``).
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

from oracle import gen_golden as gg  # noqa: E402  (imports the reference)

import tianshou.algorithm.modelfree.a2c as ref_a2c  # noqa: E402
from tianshou.algorithm import A2C  # noqa: E402
from tianshou.algorithm.optim import LRSchedulerFactoryLinear, RMSpropOptimizerFactory  # noqa: E402
from tianshou.data import VectorReplayBuffer  # noqa: E402
from tianshou.utils.torch_utils import policy_within_training_step  # noqa: E402

# examples/mujoco/mujoco_a2c.py:117-121 (and mujoco_a2c_hl.py:69)
RMSPROP = dict(lr=7e-4, eps=1e-5, alpha=0.99)
# max_update_num = ceil(epoch_num_steps / collection_step_num_env_steps) * max_epochs = 2: lr 7e-4, then 3.5e-4
LR_SCHEDULE = dict(max_epochs=1, epoch_num_steps=1024, collection_step_num_env_steps=512)


def rmsprop_factory(lr_schedule: bool) -> RMSpropOptimizerFactory:
    f = RMSpropOptimizerFactory(**RMSPROP)
    if lr_schedule:
        f.with_lr_scheduler_factory(LRSchedulerFactoryLinear(**LR_SCHEDULE))
    return f


def capture_a2c(name: str, algo, named, steps, steps2, cfg: dict) -> None:
    """Two A2C updates on fresh rollouts: buffer, permutations, v_s / returns / adv, loss table, parameters, ret_rms."""
    buf = VectorReplayBuffer(cfg["E"] * cfg["cap"], cfg["E"])
    gg.fill(buf, steps)
    out = {"p0_" + k: v.detach().numpy().copy() for k, v in named().items()}
    captured = {"pre": [], "seq": []}
    orig_pre = algo._preprocess_batch

    def pre_hook(batch, buffer, indices):
        b = orig_pre(batch, buffer, indices)
        captured["pre"].append({k: b[k].detach().numpy().copy() for k in ("v_s", "returns", "adv")}
                               | {"indices": np.asarray(indices).copy()})
        return b

    algo._preprocess_batch = pre_hook
    orig_from = ref_a2c.SequenceSummaryStats.from_sequence

    def rec(seq):
        captured["seq"].append(np.asarray(seq, dtype=np.float64))
        return orig_from(seq)

    ref_a2c.SequenceSummaryStats.from_sequence = rec
    try:
        for u, st in enumerate([steps, steps2]):
            if u == 1:
                buf.reset(keep_statistics=True)
                gg.fill(buf, st)
            out[f"u{u}_lr"] = float(algo.optim._optim.param_groups[0]["lr"])
            np.random.seed(1000 + u)
            torch.manual_seed(2000 + u)
            N = len(buf)
            with policy_within_training_step(algo.policy):
                stats = algo.update(buffer=buf, batch_size=cfg["bs"], repeat=cfg["repeat"])
            np.random.seed(1000 + u)
            perms = np.stack([np.random.permutation(N) for _ in range(cfg["repeat"])])
            pre = captured["pre"][u]
            seqs = captured["seq"][4 * u: 4 * u + 4]
            o = f"u{u}_"
            out.update({o + "perms": perms, o + "indices": pre["indices"], o + "v_s": pre["v_s"], o + "returns": pre["returns"],
                        o + "adv": pre["adv"], o + "losses": np.stack(seqs, axis=1), o + "gradient_steps": stats.gradient_steps,
                        o + "rms": np.array([float(algo.ret_rms.mean), float(algo.ret_rms.var), float(algo.ret_rms.count)])})
            out.update({o + "p_" + k: v.detach().numpy().copy() for k, v in named().items()})
            for key in ("obs", "act", "rew", "terminated", "truncated", "obs_next", "done"):
                out[o + "buf_" + key] = np.asarray(buf._meta[key]).copy()
            out.update({o + "meta_" + k: v for k, v in gg.meta_of(buf).items()})
            out[o + "unfinished"] = buf.unfinished_index()
    finally:
        ref_a2c.SequenceSummaryStats.from_sequence = orig_from
        algo._preprocess_batch = orig_pre
    out["cfg_E"], out["cfg_cap"], out["cfg_steps"], out["cfg_bs"], out["cfg_repeat"] = cfg["E"], cfg["cap"], cfg["steps"], cfg["bs"], cfg["repeat"]
    for k, v in cfg["kw"].items():
        out["kw_" + k] = np.nan if v is None else v
    for k, v in RMSPROP.items():
        out["opt_" + k] = v
    np.savez_compressed(os.path.join(OUT, f"{name}.npz"), **out)
    print(f"{name}.npz", len(out), "arrays; gradient_steps", int(out["u0_gradient_steps"]), "lr", out["u0_lr"], out["u1_lr"])


def gen_a2c_gauss() -> None:
    obs_dim, act_dim = 17, 6
    cfg = dict(E=16, cap=32, steps=32, bs=128, repeat=2, seed=5,
               kw=dict(gamma=0.99, gae_lambda=0.95, max_grad_norm=0.5, vf_coef=0.5, ent_coef=0.01, return_scaling=True))
    rng = np.random.default_rng(510)
    ppo_algo, actor, critic = gg.build_ref_ppo(obs_dim, act_dim, cfg["seed"])     # nets + policy, PPO wrapper discarded
    algo = A2C(policy=ppo_algo.policy, critic=critic, optim=rmsprop_factory(True), **cfg["kw"])
    steps = gg.synth_rollout(rng, cfg["E"], cfg["steps"], obs_dim, act_dim, 0.03, 20)
    steps2 = gg.synth_rollout(rng, cfg["E"], cfg["steps"], obs_dim, act_dim, 0.03, 20)
    capture_a2c("a2c_rmsprop_ref", algo, lambda: gg.flat_named_params(actor, critic), steps, steps2, cfg)


def gen_a2c_discrete() -> None:
    obs_dim, n_act = 4, 2
    cfg = dict(E=10, cap=40, steps=40, bs=64, repeat=2, seed=0,
               kw=dict(gamma=0.99, gae_lambda=0.95, max_grad_norm=0.5, vf_coef=0.5, ent_coef=0.01, return_scaling=False))
    rng = np.random.default_rng(520)
    ppo_algo, actor, critic = gg.build_ref_ppo_discrete(obs_dim, n_act, cfg["seed"], shared=True)
    algo = A2C(policy=ppo_algo.policy, critic=critic, optim=rmsprop_factory(True), **cfg["kw"])
    steps = gg.synth_rollout_discrete(rng, cfg["E"], cfg["steps"], obs_dim, n_act, 0.04, 25)
    steps2 = gg.synth_rollout_discrete(rng, cfg["E"], cfg["steps"], obs_dim, n_act, 0.04, 25)
    capture_a2c("a2c_rmsprop_ref_C1", algo, lambda: gg.discrete_named_params(actor, critic), steps, steps2, cfg)


def gen_npg() -> None:
    """gen_golden_npg's capture with the critic optimiser swapped for RMSprop (lr 1e-3 as the Adam NPG goldens use)."""
    from oracle import gen_golden_npg as gn
    name = "npg_rmsprop_ref"
    gn.VARIANTS[name] = ("npg", "gauss", 11, 3, 8, 16, None, 2, 8,
                         dict(return_scaling=True, advantage_normalization=True, optim_critic_iters=5, trust_region_size=0.02))
    adam_factory = gn.AdamOptimizerFactory
    gn.AdamOptimizerFactory = lambda lr: RMSpropOptimizerFactory(lr=lr, eps=RMSPROP["eps"], alpha=RMSPROP["alpha"])
    try:
        gn.gen(name)
    finally:
        gn.AdamOptimizerFactory = adam_factory
    path = os.path.join(OUT, f"{name}.npz")
    with np.load(path) as z:
        out = dict(z)
    out.update({"opt_alpha": RMSPROP["alpha"], "opt_eps": RMSPROP["eps"]})
    np.savez_compressed(path, **out)


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    jobs = {"a2c": gen_a2c_gauss, "a2c_discrete": gen_a2c_discrete, "npg": gen_npg}
    for w in sys.argv[1:] or list(jobs):
        jobs[w]()
