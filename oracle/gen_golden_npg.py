"""TEST INFRASTRUCTURE -- golden vectors for NPG / TRPO from the UNMODIFIED reference (thu-ml/tianshou 2.0.1 imported from
/root/reference through oracle/ref_shim.py).

    python -m oracle.gen_golden_npg          # writes tests/golden/npg_ref_*.npz, tests/golden/trpo_ref_*.npz

Captured per ``update()`` (two consecutive updates on fresh rollouts): the buffer in ``restore_vector_buffer`` format, the
numpy seed, v_s / returns / adv (after normalisation) / logp_old, the per-minibatch actor_loss / vf_loss / kl (/ step_size),
the warnings, every actor and critic parameter after the update, the conjugate-gradient iterations run and the margins of
every discrete decision: r.r against the residual tolerance (reconstructed from the reference's own Fisher-vector products),
and for every evaluated line-search candidate kl - max_kl and new_loss - actor_loss.  ``oracle/oracle_npg.py`` and the GPU
tests are pinned to these files.
"""
from __future__ import annotations

import os
import sys
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "tests", "golden")

from oracle.gen_golden import fill, meta_of, synth_rollout, synth_rollout_discrete  # noqa: E402  (imports the reference)

import tianshou.algorithm.modelfree.npg as ref_npg  # noqa: E402
import tianshou.algorithm.modelfree.trpo as ref_trpo  # noqa: E402
from gymnasium.spaces import Box, Discrete  # noqa: E402  (shim stand-ins)
from tianshou.algorithm import NPG, TRPO  # noqa: E402
from tianshou.algorithm.modelfree.reinforce import DiscreteActorPolicy, ProbabilisticActorPolicy  # noqa: E402
from tianshou.algorithm.optim import AdamOptimizerFactory  # noqa: E402
from tianshou.data import VectorReplayBuffer  # noqa: E402
from tianshou.utils.net.common import Net  # noqa: E402
from tianshou.utils.net.continuous import ContinuousActorProbabilistic, ContinuousCritic  # noqa: E402
from tianshou.utils.net.discrete import DiscreteActor, DiscreteCritic  # noqa: E402
from tianshou.utils.torch_utils import policy_within_training_step  # noqa: E402

RESIDUAL_TOL = 1e-10

VARIANTS = {
    # name: (algorithm, net, obs, act, E, steps, batch_size, repeat, seed, keyword arguments)
    "npg_ref_gauss": ("npg", "gauss", 11, 3, 8, 16, None, 2, 0,
                      dict(return_scaling=True, advantage_normalization=True, optim_critic_iters=5, trust_region_size=0.02)),
    "trpo_ref_gauss": ("trpo", "gauss", 11, 3, 8, 16, None, 2, 1,
                       dict(return_scaling=True, advantage_normalization=True, optim_critic_iters=5)),
    "npg_ref_mb": ("npg", "gauss", 17, 6, 8, 16, 50, 1, 2,
                   dict(advantage_normalization=False, optim_critic_iters=3, trust_region_size=0.01)),
    "trpo_ref_mb": ("trpo", "gauss", 17, 6, 8, 16, 50, 1, 3,
                    dict(advantage_normalization=False, optim_critic_iters=3)),
    "npg_ref_cat": ("npg", "cat", 6, 5, 8, 16, None, 1, 4, dict(optim_critic_iters=2, trust_region_size=0.02)),
    "trpo_ref_cat": ("trpo", "cat", 6, 5, 8, 16, 64, 1, 5, dict(optim_critic_iters=2)),
    "trpo_ref_backtrack": ("trpo", "gauss", 11, 3, 8, 16, None, 1, 6, dict(max_kl=2.0)),
    "trpo_ref_fail": ("trpo", "gauss", 11, 3, 8, 16, None, 1, 6, dict(max_kl=2.0, max_backtracks=1)),
    "trpo_ref_nobt": ("trpo", "gauss", 11, 3, 8, 16, None, 1, 7, dict(max_backtracks=0)),
}


def build(net: str, O: int, A: int, seed: int, algo: str, kw: dict):
    torch.manual_seed(seed)
    if net == "gauss":
        actor = ContinuousActorProbabilistic(preprocess_net=Net(state_shape=(O,), hidden_sizes=(64, 64), activation=torch.nn.Tanh),
                                             action_shape=(A,), unbounded=True)
        critic = ContinuousCritic(preprocess_net=Net(state_shape=(O,), hidden_sizes=(64, 64), activation=torch.nn.Tanh))
        with torch.no_grad():
            actor.sigma_param.copy_(torch.linspace(-0.9, -0.3, A).reshape(actor.sigma_param.shape))

        def dist(loc_scale):
            loc, scale = loc_scale
            return torch.distributions.Independent(torch.distributions.Normal(loc, scale), 1)

        policy = ProbabilisticActorPolicy(actor=actor, dist_fn=dist, action_scaling=True, action_bound_method="clip",
                                          action_space=Box(-1.0, 1.0, (A,)))
    else:
        actor = DiscreteActor(preprocess_net=Net(state_shape=(O,), hidden_sizes=(64, 64)), action_shape=(A,))
        critic = DiscreteCritic(preprocess_net=Net(state_shape=(O,), hidden_sizes=(64, 64)))
        policy = DiscreteActorPolicy(actor=actor, dist_fn=torch.distributions.Categorical, action_space=Discrete(A))
    cls = NPG if algo == "npg" else TRPO
    return cls(policy=policy, critic=critic, optim=AdamOptimizerFactory(lr=1e-3), **kw), actor, critic


def params(mod: torch.nn.Module, prefix: str) -> dict[str, np.ndarray]:
    return {f"{prefix}{i}": p.detach().numpy().copy() for i, p in enumerate(mod.parameters())}


def gen(name: str) -> None:
    algo_name, net, O, A, E, steps, bs, repeat, seed, kw = VARIANTS[name]
    algo, actor, critic = build(net, O, A, seed, algo_name, kw)
    rng = np.random.default_rng(700 + seed)
    rolls = [synth_rollout(rng, E, steps, O, A, 0.05, 12) if net == "gauss" else synth_rollout_discrete(rng, E, steps, O, A, 0.05, 12)
             for _ in range(2)]
    out = {"cfg_obs": O, "cfg_act": A, "cfg_E": E, "cfg_cap": steps, "cfg_bs": -1 if bs is None else bs, "cfg_repeat": repeat,
           "cfg_categorical": int(net == "cat"), "cfg_trpo": int(algo_name == "trpo"), "cfg_lr": 1e-3}
    for k, v in kw.items():
        out["kw_" + k] = v
    out.update(params(actor, "p0_actor_"))
    out.update(params(critic, "p0_critic_"))

    cap = {}
    orig_pre, orig_cg, orig_mvp = algo._preprocess_batch, algo._conjugate_gradients, algo._MVP
    orig_fwd = algo.policy.forward

    def pre(batch, buffer, indices):
        b = orig_pre(batch, buffer, indices)
        cap["pre"] = {k: b[k].detach().numpy().copy() for k in ("v_s", "returns", "adv", "logp_old")}
        return b

    def mvp(v, flat_kl_grad):
        z = orig_mvp(v, flat_kl_grad)
        if cap.get("pairs") is not None:
            cap["pairs"].append((v.detach().clone(), z.detach().clone()))
        return z

    def cg(b, flat_kl_grad, nsteps=10, residual_tol=RESIDUAL_TOL):
        cap["pairs"], cap["cands"], cap["kls"] = [], [], []
        x = orig_cg(b, flat_kl_grad, nsteps=nsteps, residual_tol=residual_tol)
        # r.r after every iteration, replayed from the reference's own products (npg.py:212-218 arithmetic, fp32)
        r, rdotr, rr = b.detach().clone(), None, []
        rdotr = r.dot(r)
        for p, z in cap["pairs"]:
            alpha = rdotr / p.dot(z)
            r = r - alpha * z
            rdotr = r.dot(r)
            rr.append(float(rdotr))
        cap["mb"].append({"cg_iters": len(cap["pairs"]), "rdotr": rr, "cands": cap["cands"], "kls": cap["kls"]})
        cap["pairs"] = None
        return x

    def fwd(batch, state=None, **kwargs):
        res = orig_fwd(batch, state, **kwargs)
        if cap.get("cands") is not None and cap.get("pairs") is None and not torch.is_grad_enabled():
            with torch.no_grad():
                lp = res.dist.log_prob(batch.act)
                cap["cands"].append(float(-((lp - batch.logp_old).exp().float() * batch.adv).mean()))
        return res

    orig_kl = ref_trpo.kl_divergence

    def kl(p, q):
        t = orig_kl(p, q)
        if cap.get("cands") is not None and cap.get("pairs") is None:
            cap["kls"].append(float(t.mean()))
        return t

    orig_critic = algo.critic.forward

    def critic_fwd(*args, **kwargs):          # the critic steps follow the line search: it is over
        cap["cands"] = None
        return orig_critic(*args, **kwargs)

    seqs: list[np.ndarray] = []
    orig_from = ref_npg.SequenceSummaryStats.from_sequence

    def rec(seq):
        seqs.append(np.asarray(seq, dtype=np.float64))
        return orig_from(seq)

    algo._preprocess_batch, algo._conjugate_gradients, algo._MVP = pre, cg, mvp
    algo.policy.forward, algo.critic.forward = fwd, critic_fwd
    ref_trpo.kl_divergence = kl
    ref_npg.SequenceSummaryStats.from_sequence = rec
    ref_trpo.SequenceSummaryStats.from_sequence = rec
    buf = VectorReplayBuffer(E * steps, E)
    try:
        for u in range(2):
            if u == 1:
                buf.reset(keep_statistics=True)
            fill(buf, rolls[u])
            cap["mb"], seqs[:] = [], []
            np.random.seed(1000 + u)
            with warnings.catch_warnings(record=True) as w, policy_within_training_step(algo.policy):
                warnings.simplefilter("always")
                algo.update(buffer=buf, batch_size=bs, repeat=repeat)
            o = f"u{u}_"
            for key in ("obs", "act", "rew", "terminated", "truncated", "obs_next", "done"):
                out[o + "buf_" + key] = np.asarray(buf._meta[key]).copy()
            out.update({o + "meta_" + k: v for k, v in meta_of(buf).items()})
            out[o + "np_seed"] = 1000 + u
            out.update({o + k: v for k, v in cap["pre"].items()})
            out[o + "actor_loss"], out[o + "vf_loss"], out[o + "kl"] = seqs[0], seqs[1], seqs[2]
            if algo_name == "trpo":
                out[o + "step_size"] = seqs[3]
            out[o + "warnings"] = np.array([str(x.message) for x in w if issubclass(x.category, UserWarning)], dtype=np.str_)
            out[o + "cg_iters"] = np.array([m["cg_iters"] for m in cap["mb"]], dtype=np.int64)
            out[o + "cg_log10_rdotr_margin"] = np.array([min(abs(np.log10(max(v, 1e-300) / RESIDUAL_TOL)) for v in m["rdotr"])
                                                         for m in cap["mb"]])
            if algo_name == "trpo":         # every evaluated line-search candidate, in order
                out[o + "ls_count"] = np.array([len(m["kls"]) for m in cap["mb"]], dtype=np.int64)
                out[o + "ls_kl"] = np.array([v for m in cap["mb"] for v in m["kls"]], dtype=np.float64)
                out[o + "ls_new_loss"] = np.array([v for m in cap["mb"] for v in m["cands"]], dtype=np.float64)
            out.update(params(actor, o + "actor_"))
            out.update(params(critic, o + "critic_"))
    finally:
        algo.policy.forward, algo.critic.forward = orig_fwd, orig_critic
        ref_trpo.kl_divergence = orig_kl
        ref_npg.SequenceSummaryStats.from_sequence = orig_from
        ref_trpo.SequenceSummaryStats.from_sequence = orig_from
    np.savez_compressed(os.path.join(OUT, f"{name}.npz"), **out)
    print(name, {k: np.asarray(out[k]).tolist() for k in out if k.startswith("u") and k.endswith(("warnings", "cg_iters", "step_size", "kl"))})


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    for n in sys.argv[1:] or list(VARIANTS):
        gen(n)
