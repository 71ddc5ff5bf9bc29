"""TEST INFRASTRUCTURE -- numpy float64 restatement of PSRL (tianshou/algorithm/modelbased/psrl.py).

``update_rows`` is the reference's per-row loop of ``PSRL._update_with_batch`` (:253-270) given the permutation that
``batch.split(size=1)`` drew; ``observe`` is ``PSRLModel.observe`` (:65-98); ``value_iteration`` is ``PSRLModel.value_iteration``
(:116-150) with the tie-break noise passed in, returning the number of sweeps (evaluations of Q) as well.
"""
from __future__ import annotations

import numpy as np

EPS32 = np.finfo(np.float32).eps.item()


def update_rows(n_s, n_a, obs, act, obs_next, rew, done, perm, add_done_loop):
    """The batch's (trans_count, rew_sum, rew_square_sum, rew_count), the rows taken one at a time in ``perm``'s order.  ``rew``
    keeps its dtype: a float32 reward is squared in float32."""
    trans_count = np.zeros((n_s, n_a, n_s))
    rew_sum = np.zeros((n_s, n_a))
    rew_square_sum = np.zeros((n_s, n_a))
    rew_count = np.zeros((n_s, n_a))
    for j in perm:
        s, a, t, r = obs[j], act[j], obs_next[j], rew[j:j + 1]      # r: a one-row array, as split(size=1) yields it
        trans_count[s, a, t] += 1
        rew_sum[s, a] += r[0]
        rew_square_sum[s, a] += (r**2)[0]         # an array's square is x * x in its dtype (a scalar's ** is pow)
        rew_count[s, a] += 1
        if add_done_loop and done[j]:
            trans_count[t, :, t] += 1
            rew_count[t, :] += 1
    return trans_count, rew_sum, rew_square_sum, rew_count


def initial_state(trans_count_prior, rew_mean_prior, rew_std_prior, epsilon):
    """The model's posterior before any update, as float64 copies."""
    return dict(trans_count=np.array(trans_count_prior, dtype=np.float64), rew_mean=np.array(rew_mean_prior, dtype=np.float64),
                rew_std=np.array(rew_std_prior, dtype=np.float64), rew_square_sum=np.zeros(np.shape(rew_mean_prior)),
                rew_count=np.full(np.shape(rew_mean_prior), float(epsilon)))


def observe(state, rew_std_prior, trans_count, rew_sum, rew_square_sum, rew_count):
    """PSRLModel.observe on the dict of the five posterior arrays, in place and in the reference's operation order."""
    state["trans_count"] += trans_count
    sum_count = state["rew_count"] + rew_count
    state["rew_mean"] = (state["rew_mean"] * state["rew_count"] + rew_sum) / sum_count
    state["rew_square_sum"] += rew_square_sum
    raw_std2 = state["rew_square_sum"] / sum_count - state["rew_mean"] ** 2
    state["rew_std"] = np.sqrt(1 / (sum_count / (raw_std2 + EPS32) + 1 / rew_std_prior**2))
    state["rew_count"] = sum_count
    return state


def value_iteration(trans_prob, rew, gamma, eps, value, noise, max_sweeps=None):
    """(policy, value, sweeps, noised Q).  ``max_sweeps`` bounds the loop for tests that build slow MDPs (None: the reference's
    unbounded loop); past it the result is (None, None, sweeps, None)."""
    Q = rew + gamma * trans_prob.dot(value)
    new_value = Q.max(axis=1)
    sweeps = 1
    while not np.allclose(new_value, value, eps):
        if max_sweeps is not None and sweeps >= max_sweeps:
            return None, None, sweeps, None
        value = new_value
        Q = rew + gamma * trans_prob.dot(value)
        new_value = Q.max(axis=1)
        sweeps += 1
    Q = Q + eps * noise
    return Q.argmax(axis=1), new_value, sweeps, Q


def tie_gap(q_noised):
    """The smallest gap between the best and the second-best action over the states (inf with one action)."""
    if q_noised.shape[1] < 2:
        return np.inf
    s = np.sort(q_noised, axis=1)
    return float((s[:, -1] - s[:, -2]).min())


def nchain_step(rng, s, a, n=5, slip=0.2, small=2.0, large=10.0):
    """NChain (gym's NChain-v0): action 0 moves forward (the last state pays ``large`` and stays), action 1 returns to the start
    paying ``small``; with probability ``slip`` the other action happens."""
    if rng.random() < slip:
        a = 1 - a
    if a == 1:
        return 0, small
    if s < n - 1:
        return s + 1, 0.0
    return s, large


def nchain_model(n=5, slip=0.2, small=2.0, large=10.0):
    """NChain's true (P [n][2][n], expected reward [n][2])."""
    P = np.zeros((n, 2, n))
    R = np.zeros((n, 2))
    for s in range(n):
        fwd = min(s + 1, n - 1)
        P[s, 0, fwd] += 1 - slip
        P[s, 0, 0] += slip
        P[s, 1, 0] += 1 - slip
        P[s, 1, fwd] += slip
        r_fwd = large if s == n - 1 else 0.0
        R[s, 0] = (1 - slip) * r_fwd + slip * small
        R[s, 1] = (1 - slip) * small + slip * r_fwd
    return P, R
