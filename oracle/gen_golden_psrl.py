"""TEST INFRASTRUCTURE -- golden vectors for PSRL from the UNMODIFIED reference (thu-ml/tianshou 2.0.1 imported through
oracle/ref_shim.py).

    python -m oracle.gen_golden_psrl       # writes tests/golden/psrl_ref_{chain,chain_f32_done,lake,wide}.npz

Each variant runs rounds of: a synthetic rollout into a ``VectorReplayBuffer`` -> ``PSRL.update`` -> one ``forward`` (the lazy
solve) -> ``buffer.reset()``.  ``chain`` is NChain (5 x 2, slip 0.2) with test_psrl.py's priors and float64 rewards;
``chain_f32_done`` the same with ``add_done_loop=True``, terminated and truncated rows and float32 rewards (the
buffer's rewards plus noise, handed to ``_update_with_batch`` in the batch: the buffer itself stores float64); ``lake`` a random
16 x 4 MDP with a Dirichlet prior of 0.5, a reward prior of 0.3 / 2.0, gamma 0.95 and eps 1e-3; ``wide`` a sparse random 80 x 3
MDP whose rollouts leave many (s, a) pairs unvisited.  ``lake`` pays 0 / 1 rewards, as FrozenLake does: with a reward count
prior of eps = 1e-3, a pair seen once with a reward strictly between 0 and 2 x 0.3 gets a negative variance estimate and the
reference's rew_std turns NaN, after which its value iteration never ends.

Captured per round ``r<i>_``: numpy's global state before and after the update (pack_numpy_state), the buffer's rows in
``buffer.sample(0)``'s order, the five posterior arrays and the two stats after the update, the three draws of the solve
(``sample_trans_prob``, ``sample_reward`` and the ``np.random.randn`` tie-break noise, recorded by wrapping them at run time),
the policy and value, the sweep count (calls of ``np.allclose``) and the smallest gap between the best and second-best noised Q.
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

from oracle import oracle_psrl as op  # noqa: E402
from oracle.ref_shim import import_reference  # noqa: E402
from tianshou_b200.algorithm.minibatch_order import pack_numpy_state  # noqa: E402

ts = import_reference()
import gymnasium as gym  # noqa: E402  (ref_shim's stand-in)
from tianshou.algorithm import PSRL  # noqa: E402
from tianshou.algorithm.modelbased.psrl import PSRLPolicy  # noqa: E402
from tianshou.data import Batch, VectorReplayBuffer  # noqa: E402
from tianshou.utils.torch_utils import policy_within_training_step  # noqa: E402

VARIANTS = {
    "chain": dict(kind="chain", n_s=5, n_a=2, E=2, T=60, rounds=3, tc=1.0, rm=0.0, rs=1.0, gamma=0.99, eps=0.01, done_loop=False,
                  f32=False, seed=1),
    "chain_f32_done": dict(kind="chain", n_s=5, n_a=2, E=3, T=40, rounds=3, tc=1.0, rm=0.0, rs=1.0, gamma=0.99, eps=0.01,
                           done_loop=True, f32=True, p_term=0.08, p_trunc=0.05, seed=2),
    "lake": dict(kind="random", n_s=16, n_a=4, E=4, T=60, rounds=3, tc=0.5, rm=0.3, rs=2.0, gamma=0.95, eps=1e-3, done_loop=False,
                 f32=False, p_term=0.03, seed=3, visit=16, binary=True),
    "wide": dict(kind="random", n_s=80, n_a=3, E=4, T=80, rounds=2, tc=1.0, rm=0.0, rs=1.0, gamma=0.9, eps=0.01, done_loop=False,
                 f32=False, seed=4, visit=40),
}


def rollout(rng, cfg, true_P, true_R):
    """[T] steps of E rows: obs, act, rew, terminated, truncated, obs_next."""
    n_s, n_a, E = cfg["n_s"], cfg["n_a"], cfg["E"]
    steps = []
    s = rng.integers(0, cfg.get("visit", n_s), E)
    for _ in range(cfg["T"]):
        a = rng.integers(0, n_a, E)
        if cfg["kind"] == "chain":
            nxt, r = zip(*(op.nchain_step(rng, int(si), int(ai)) for si, ai in zip(s, a)))
            nxt, r = np.array(nxt), np.array(r)
        else:
            nxt = np.array([rng.choice(n_s, p=true_P[si, ai]) for si, ai in zip(s, a)])
            r = (rng.random(E) < true_R[s, a]).astype(float) if cfg.get("binary") else true_R[s, a] + 0.5 * rng.standard_normal(E)
        r = r.astype(np.float32 if cfg["f32"] else np.float64)
        term = rng.random(E) < cfg.get("p_term", 0.0)
        trunc = ~term & (rng.random(E) < cfg.get("p_trunc", 0.0))
        steps.append(dict(obs=s.astype(np.int64), act=a.astype(np.int64), rew=r, terminated=term, truncated=trunc,
                          obs_next=nxt.astype(np.int64)))
        s = np.where(term | trunc, rng.integers(0, cfg.get("visit", n_s), E), nxt)
    return steps


def true_model(rng, cfg):
    n_s, n_a = cfg["n_s"], cfg["n_a"]
    if cfg["kind"] == "chain":
        return op.nchain_model(n_s)
    visit = cfg.get("visit", n_s)
    P = np.zeros((n_s, n_a, n_s))
    for s in range(n_s):
        for a in range(n_a):
            nxt = rng.choice(visit, size=3, replace=False)
            P[s, a, nxt] = rng.dirichlet(np.ones(3))
    return P, (rng.random((n_s, n_a)) * 0.3 if cfg.get("binary") else rng.standard_normal((n_s, n_a)))


def generate(name, cfg):
    n_s, n_a = cfg["n_s"], cfg["n_a"]
    rng = np.random.default_rng(cfg["seed"])
    true_P, true_R = true_model(rng, cfg)
    tc_prior = np.full((n_s, n_a, n_s), cfg["tc"])
    rm_prior = np.full((n_s, n_a), cfg["rm"])
    rs_prior = np.full((n_s, n_a), cfg["rs"])
    out = dict(cfg_n_s=n_s, cfg_n_a=n_a, cfg_gamma=cfg["gamma"], cfg_eps=cfg["eps"], cfg_add_done_loop=cfg["done_loop"],
               cfg_rounds=cfg["rounds"], cfg_E=cfg["E"], trans_count_prior=tc_prior.copy(), rew_mean_prior=rm_prior.copy(),
               rew_std_prior=rs_prior.copy())
    policy = PSRLPolicy(trans_count_prior=tc_prior, rew_mean_prior=rm_prior, rew_std_prior=rs_prior,
                        action_space=gym.spaces.Discrete(n_a), discount_factor=cfg["gamma"], epsilon=cfg["eps"])
    algo = PSRL(policy=policy, add_done_loop=cfg["done_loop"])
    model = policy.model
    buf = VectorReplayBuffer(cfg["E"] * cfg["T"], cfg["E"])
    np.random.seed(cfg["seed"] + 100)
    torch.manual_seed(cfg["seed"] + 100)
    for r in range(cfg["rounds"]):
        buf.reset()
        for st in rollout(rng, cfg, true_P, true_R):
            buf.add(Batch(**st, info=Batch()), buffer_ids=np.arange(cfg["E"]))
        rows, _ = buf.sample(0)
        if cfg["f32"]:
            # the buffer widens rewards to float64 on its first add; float32 rewards reach the update in a batch of their own
            rows.rew = (rows.rew + 0.1 * rng.standard_normal(len(rows))).astype(np.float32)
        p = f"r{r}_"
        for k in ("obs", "act", "rew", "done", "obs_next"):
            out[p + k] = np.asarray(rows[k]).copy()
        out[p + "value_before"] = model.value.copy()
        out[p + "np_state"] = pack_numpy_state(np.random.get_state())
        with policy_within_training_step(policy):
            stats = algo._update_with_batch(rows, 0, 1) if cfg["f32"] else algo.update(buffer=buf, batch_size=0, repeat=1)
        out[p + "np_state_after"] = pack_numpy_state(np.random.get_state())
        for k in ("trans_count", "rew_mean", "rew_std", "rew_square_sum", "rew_count"):
            out[p + k] = np.array(getattr(model, k), dtype=np.float64)
        out[p + "stat_mean"], out[p + "stat_std"] = stats.psrl_rew_mean, stats.psrl_rew_std
        draws = {}
        orig_tp, orig_rw, orig_randn, orig_close = model.sample_trans_prob, model.sample_reward, np.random.randn, np.allclose
        calls = [0]

        def tp():
            draws["P"] = orig_tp()
            return draws["P"]

        def rw():
            draws["R"] = orig_rw()
            return draws["R"]

        def randn(*shape):
            draws["noise"] = orig_randn(*shape)
            return draws["noise"]

        def allclose(*a, **k):
            calls[0] += 1
            return orig_close(*a, **k)

        model.sample_trans_prob, model.sample_reward = tp, rw
        np.random.randn, np.allclose = randn, allclose
        try:
            act = policy(Batch(obs=np.arange(n_s), info=Batch())).act
        finally:
            del model.sample_trans_prob, model.sample_reward
            np.random.randn, np.allclose = orig_randn, orig_close
        out[p + "P"], out[p + "R"], out[p + "noise"] = draws["P"], draws["R"], draws["noise"]
        out[p + "policy"], out[p + "value"], out[p + "sweeps"] = np.asarray(act), model.value.copy(), calls[0]
        pol, val, sweeps, qn = op.value_iteration(draws["P"], draws["R"], cfg["gamma"], cfg["eps"], out[p + "value_before"],
                                                  draws["noise"])
        assert sweeps == calls[0] and np.array_equal(pol, act) and np.array_equal(val, model.value), name
        out[p + "gap"] = op.tie_gap(qn)
        assert out[p + "gap"] > 1e-9 * max(1.0, float(np.abs(qn).max())), (name, r, out[p + "gap"])
    out["state_dict_keys"] = np.array(sorted(algo.state_dict().keys()))
    path = os.path.join(OUT, f"psrl_ref_{name}.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes;", {k: int(out[f"r{k}_sweeps"]) for k in range(cfg["rounds"])})


if __name__ == "__main__":
    for n in sys.argv[1:] or VARIANTS:
        generate(n, VARIANTS[n])
