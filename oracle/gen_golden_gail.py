"""TEST INFRASTRUCTURE -- golden vectors for GAIL from the UNMODIFIED reference (thu-ml/tianshou 2.0.1 imported through
oracle/ref_shim.py).

    python -m oracle.gen_golden_gail          # writes tests/golden/gail_ref_*.npz

Captured per ``update()`` (two consecutive updates on fresh rollouts): the rollout in ``restore_vector_buffer`` format, the
numpy seed, the per-row rewards the discriminator produced and v_s / returns / adv / logp_old, the per-step discriminator loss /
acc_pi / acc_exp with the smallest |logit| on each side (the decision margins behind the accuracy counts), the expert indices
each step drew, PPO's loss table, every actor / critic / discriminator parameter after the update, the discriminator's learning
rate during the update, and the generator states after it: numpy's global one and the expert buffer's (for a
VectorReplayBuffer the manager's and each sub-buffer's).  The expert buffer and the initial parameters are stored once.
``oracle/oracle_gail.py`` and the GPU tests are pinned to these files.
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

from oracle.gen_golden import fill, meta_of, synth_rollout  # noqa: E402  (imports the reference)

from gymnasium.spaces import Box  # noqa: E402  (shim stand-in)
from tianshou.algorithm import GAIL  # noqa: E402
from tianshou.algorithm.modelfree.reinforce import ProbabilisticActorPolicy  # noqa: E402
from tianshou.algorithm.optim import AdamOptimizerFactory, LRSchedulerFactoryLinear  # noqa: E402
from tianshou.data import ReplayBuffer, SequenceSummaryStats, VectorReplayBuffer  # noqa: E402
from tianshou.utils.net.common import Net  # noqa: E402
from tianshou.utils.net.continuous import ContinuousActorProbabilistic, ContinuousCritic  # noqa: E402
from tianshou.utils.torch_utils import policy_within_training_step  # noqa: E402

VARIANTS = {
    # name: (obs, act, hidden, disc activation, E, steps, batch_size, repeat, disc_update_num, seed, vector expert, disc lr
    #        schedule, keyword arguments)
    "gail_ref_tc": (11, 3, (64, 64), "tanh", 16, 16, 64, 2, 2, 0, False, False,
                    dict(return_scaling=True, value_clip=True, advantage_normalization=True, max_grad_norm=0.5, vf_coef=0.25,
                         ent_coef=0.001)),
    "gail_ref_merge": (11, 3, (64, 64), "tanh", 8, 16, 50, 2, 3, 1, True, True,
                       dict(recompute_advantage=True, advantage_normalization=False, max_grad_norm=0.5)),
    "gail_ref_steps": (11, 3, (64, 64), "tanh", 8, 15, 40, 1, 11, 2, False, False, dict()),
    "gail_ref_layered": (17, 6, (128, 128), "relu", 8, 16, 64, 2, 2, 5, False, False,
                         dict(return_scaling=True, max_grad_norm=0.5)),
}
EXPERT_E, EXPERT_CAP = 4, 50            # vector expert buffer: 4 sub-buffers of 50 (one of them partly filled)
EXPERT_ROWS = 300                       # plain expert buffer (ReplayBuffer.from_data)
LR, DISC_LR = 3e-4, 5e-4


def build(O: int, A: int, hidden: tuple[int, ...], disc_act: str, seed: int, dun: int, expert, sched: bool, kw: dict):
    torch.manual_seed(seed)
    actor = ContinuousActorProbabilistic(preprocess_net=Net(state_shape=(O,), hidden_sizes=hidden, activation=torch.nn.Tanh),
                                         action_shape=(A,), unbounded=True)
    critic = ContinuousCritic(preprocess_net=Net(state_shape=(O,), hidden_sizes=hidden, activation=torch.nn.Tanh))
    act_cls = torch.nn.Tanh if disc_act == "tanh" else torch.nn.ReLU
    disc = ContinuousCritic(preprocess_net=Net(state_shape=(O,), action_shape=(A,), hidden_sizes=hidden, activation=act_cls,
                                               concat=True))
    torch.nn.init.constant_(actor.sigma_param, -0.5)
    for m in list(actor.modules()) + list(critic.modules()) + list(disc.modules()):
        if isinstance(m, torch.nn.Linear):          # irl_gail.py:137-144, 164-168
            torch.nn.init.orthogonal_(m.weight, gain=np.sqrt(2))
            torch.nn.init.zeros_(m.bias)
    for m in actor.mu.modules():
        if isinstance(m, torch.nn.Linear):
            torch.nn.init.zeros_(m.bias)
            m.weight.data.copy_(0.01 * m.weight.data)

    def dist(loc_scale):
        loc, scale = loc_scale
        return torch.distributions.Independent(torch.distributions.Normal(loc, scale), 1)

    policy = ProbabilisticActorPolicy(actor=actor, dist_fn=dist, action_scaling=True, action_bound_method="clip",
                                      action_space=Box(-1.0, 1.0, (A,)))
    disc_optim = AdamOptimizerFactory(lr=DISC_LR)
    if sched:
        disc_optim.with_lr_scheduler_factory(LRSchedulerFactoryLinear(max_epochs=2, epoch_num_steps=8, collection_step_num_env_steps=4))
    algo = GAIL(policy=policy, critic=critic, optim=AdamOptimizerFactory(lr=LR), expert_buffer=expert, disc_net=disc,
                disc_optim=disc_optim, disc_update_num=dun, **kw)
    return algo, actor, critic, disc


def params(mod: torch.nn.Module, prefix: str) -> dict[str, np.ndarray]:
    return {f"{prefix}{i}": p.detach().numpy().copy() for i, p in enumerate(mod.parameters())}


def rng_state(prefix: str, st: tuple) -> dict[str, np.ndarray]:
    return {prefix + "key": np.asarray(st[1], dtype=np.uint32).copy(), prefix + "pos": np.int64(st[2]),
            prefix + "gauss": np.array([float(st[3]), float(st[4])])}


def expert_states(buf, vector: bool) -> dict[str, np.ndarray]:
    out = rng_state("rng_exp_", buf._random_state.get_state())
    if vector:
        for e, sub in enumerate(buf.buffers):
            out.update(rng_state(f"rng_exp{e}_", sub._random_state.get_state()))
    return out


def expert_rollout(rng, E, steps, O, A):
    """Expert-like rows: actions shifted by +0.5, so the discriminator has something to separate."""
    roll = synth_rollout(rng, E, steps, O, A, 0.05, 12)
    for s in roll:
        s["act"] = (s["act"] + 0.5).astype(np.float32)
    return roll


def gen(name: str) -> None:
    O, A, hidden, disc_act, E, steps, bs, repeat, dun, seed, vector, sched, kw = VARIANTS[name]
    rng = np.random.default_rng(900 + seed)
    out = {"cfg_obs": O, "cfg_act": A, "cfg_hidden": np.array(hidden), "cfg_disc_relu": int(disc_act == "relu"), "cfg_E": E,
           "cfg_cap": steps, "cfg_bs": bs, "cfg_repeat": repeat, "cfg_dun": dun, "cfg_lr": LR, "cfg_disc_lr": DISC_LR,
           "cfg_vector_expert": int(vector), "cfg_sched": int(sched)}
    for k, v in kw.items():
        out["kw_" + k] = v
    if vector:
        expert = VectorReplayBuffer(EXPERT_E * EXPERT_CAP, EXPERT_E)
        roll = expert_rollout(rng, EXPERT_E, EXPERT_CAP, O, A)
        fill(expert, roll)
        s = expert_rollout(rng, EXPERT_E, 1, O, A)[0]     # a few more rows: sub-buffers 0 and 2 wrap
        ids = np.array([0, 2])
        from tianshou.data import Batch
        expert.add(Batch(obs=s["obs"][ids], act=s["act"][ids], rew=s["rew"][ids], terminated=s["terminated"][ids],
                         truncated=s["truncated"][ids], obs_next=s["obs_next"][ids]), buffer_ids=ids)
        for key in ("obs", "act", "rew", "terminated", "truncated", "obs_next", "done"):
            out["exp_buf_" + key] = np.asarray(expert._meta[key]).copy()
        out.update({"exp_meta_" + k: v for k, v in meta_of(expert).items()})
    else:
        n = EXPERT_ROWS
        eo = rng.standard_normal((n, O)).astype(np.float32)
        ea = (rng.standard_normal((n, A)) + 0.5).astype(np.float32)
        er = rng.standard_normal(n)
        et = rng.random(n) < 0.05
        etr = np.zeros(n, dtype=bool)
        en = rng.standard_normal((n, O)).astype(np.float32)
        expert = ReplayBuffer.from_data(eo, ea, er, et, etr, et | etr, en)
        out.update({"exp_obs": eo, "exp_act": ea, "exp_rew": er, "exp_terminated": et, "exp_truncated": etr, "exp_obs_next": en})
    algo, actor, critic, disc = build(O, A, hidden, disc_act, seed, dun, expert, sched, kw)
    out.update(params(actor, "p0_actor_"))
    out.update(params(critic, "p0_critic_"))
    out.update(params(disc, "p0_disc_"))
    rolls = [synth_rollout(rng, E, steps, O, A, 0.05, 12) for _ in range(2)]

    cap: dict = {"logits": [], "exp_idx": []}
    orig_pre, orig_disc, orig_sample = algo._preprocess_batch, algo.disc, expert.sample

    def pre(batch, buffer, indices):
        b = orig_pre(batch, buffer, indices)
        cap["pre"] = {k: np.asarray(b[k].detach().numpy() if isinstance(b[k], torch.Tensor) else b[k]).copy()
                      for k in ("rew", "v_s", "returns", "adv", "logp_old")}
        return b

    def disc_fn(batch):
        y = orig_disc(batch)
        cap["logits"].append(y.detach().numpy().reshape(-1).copy())
        return y

    def sample(bsz):
        b, idx = orig_sample(bsz)
        cap["exp_idx"].append(np.asarray(idx, dtype=np.int64).copy())
        return b, idx

    seqs: list[np.ndarray] = []
    orig_from = SequenceSummaryStats.from_sequence

    def rec(seq):
        seqs.append(np.asarray(seq, dtype=np.float64))
        return orig_from(seq)

    algo._preprocess_batch, algo.disc, expert.sample = pre, disc_fn, sample
    SequenceSummaryStats.from_sequence = staticmethod(rec)
    buf = VectorReplayBuffer(E * steps, E)
    try:
        for u in range(2):
            if u == 1:
                buf.reset(keep_statistics=True)
            fill(buf, rolls[u])
            cap["logits"], cap["exp_idx"], seqs[:] = [], [], []
            np.random.seed(1000 + u)
            out[f"u{u}_disc_lr"] = float(algo.disc_optim._optim.param_groups[0]["lr"])
            with policy_within_training_step(algo.policy):
                algo.update(buffer=buf, batch_size=bs, repeat=repeat)
            o = f"u{u}_"
            for key in ("obs", "act", "rew", "terminated", "truncated", "obs_next", "done"):
                out[o + "buf_" + key] = np.asarray(buf._meta[key]).copy()
            out.update({o + "meta_" + k: v for k, v in meta_of(buf).items()})
            out[o + "np_seed"] = 1000 + u
            out.update({o + k: v for k, v in cap["pre"].items()})
            out[o + "losses"] = np.stack(seqs[:4], axis=1)               # loss, clip, vf, ent per PPO step
            out[o + "disc_loss"], out[o + "acc_pi"], out[o + "acc_exp"] = seqs[4], seqs[5], seqs[6]
            step_logits = cap["logits"][1:]                              # [0] is the reward pass
            out[o + "reward_logits"] = cap["logits"][0]
            out[o + "margin_pi"] = np.array([np.abs(x).min() for x in step_logits[0::2]])
            out[o + "margin_exp"] = np.array([np.abs(x).min() for x in step_logits[1::2]])
            out[o + "exp_idx"] = np.concatenate(cap["exp_idx"])
            out.update(params(actor, o + "actor_"))
            out.update(params(critic, o + "critic_"))
            out.update(params(disc, o + "disc_"))
            out.update(rng_state(o + "rng_np_", np.random.get_state()))
            out.update({o + k: v for k, v in expert_states(expert, vector).items()})
    finally:
        SequenceSummaryStats.from_sequence = orig_from
    np.savez_compressed(os.path.join(OUT, f"{name}.npz"), **out)
    print(name, {k: np.round(np.asarray(out[k]), 4).tolist() for k in out if k.startswith("u") and k.endswith(("disc_loss", "acc_pi", "acc_exp"))})


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    for n in sys.argv[1:] or list(VARIANTS):
        gen(n)
