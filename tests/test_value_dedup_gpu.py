"""One critic evaluation per distinct observation in the value pass: the next-observation alias map
(``ts_next_alias_map``) against numpy, ``ts_critic_forward_dedup`` against ``ts_critic_forward`` bit for bit, and whole
updates with the map against the same updates without it."""
import numpy as np
import pytest
import torch

from ts_testutil import build_ppo, perturb_params, synth_rollout

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _alias_ref(obs: np.ndarray, obs_next: np.ndarray):
    """alias / extra by the definition: bitwise equality of obs_next[i] and obs[i + 1]."""
    n = obs.shape[0]
    a, b = obs_next.view(np.uint32).reshape(n, -1), obs.view(np.uint32).reshape(n, -1)
    alias = np.zeros(n, dtype=np.uint8)
    if n > 1:
        alias[:-1] = (a[:-1] == b[1:]).all(axis=1)
    return alias, np.flatnonzero(alias == 0).astype(np.int32)


def _check_map(obs: np.ndarray, obs_next: np.ndarray):
    from tianshou_b200 import ops
    obs, obs_next = np.ascontiguousarray(obs, np.float32), np.ascontiguousarray(obs_next, np.float32)
    amap = ops.next_alias_map(torch.from_numpy(obs).to(DEV), torch.from_numpy(obs_next).to(DEV))
    alias, extra = _alias_ref(obs, obs_next)
    m = int(amap.count.item())
    assert m == len(extra)
    assert np.array_equal(amap.alias.cpu().numpy(), alias) and alias[-1] == 0
    assert np.array_equal(amap.extra[:m].cpu().numpy(), extra)       # ascending, complete
    return alias, extra


def _rollout(E, T, obs_dim, act_dim=2, seed=0, **kw):
    """Row-major-by-env obs / obs_next of a synthetic rollout (row = e * T + t)."""
    steps = list(synth_rollout(np.random.default_rng(seed), E, T, obs_dim, act_dim, **kw))
    obs = np.stack([s["obs"] for s in steps], axis=1).reshape(E * T, obs_dim)
    obs_next = np.stack([s["obs_next"] for s in steps], axis=1).reshape(E * T, obs_dim)
    return np.ascontiguousarray(obs), np.ascontiguousarray(obs_next)


def _buffer(E, T, obs_dim, act_dim, steps=None, **buf_kw):
    from tianshou_b200.data import Batch, VectorReplayBuffer
    buf = VectorReplayBuffer(E * T, E, device=DEV, **buf_kw)
    for s in list(synth_rollout(np.random.default_rng(3), E, T, obs_dim, act_dim, p_term=0.03, trunc_len=40))[:steps]:
        buf.add(Batch(**s), buffer_ids=np.arange(E))
    return buf


# ------------------------------------------------------------------------------------------------ alias map
@pytest.mark.parametrize("E,T,obs_dim", [(8, 50, 17), (3, 43, 5), (1, 1, 17), (1, 300, 32), (5, 77, 1)])
def test_alias_map_of_a_rollout(E, T, obs_dim):
    obs, obs_next = _rollout(E, T, obs_dim, p_term=0.05, trunc_len=20)
    alias, extra = _check_map(obs, obs_next)
    if E * T > 1:
        assert len(extra) >= E and alias.sum() > 0          # every env's last row, and some rows do alias


def test_alias_map_is_a_bitwise_test():
    obs, obs_next = _rollout(4, 64, 8, p_term=0.0)
    obs[10, 3], obs_next[9, 3] = 0.0, -0.0                  # equal as floats, different words: not aliased
    obs[20, 0] = obs_next[19, 0] = np.nan                   # the same NaN word on both sides: aliased
    obs_next[30, 1] = np.nan                                # NaN against a number
    obs[41, 2] = np.float32(-0.0)
    obs_next[40, 2] = np.float32(-0.0)
    alias, _ = _check_map(obs, obs_next)
    assert alias[9] == 0 and alias[19] == 1 and alias[30] == 0 and alias[40] == 1


def test_alias_map_of_a_shuffled_batch_lists_every_row():
    obs, obs_next = _rollout(16, 32, 17)
    p = np.random.default_rng(1).permutation(len(obs))
    _, extra = _check_map(obs[p], obs_next[p])
    assert len(extra) >= len(obs) - 16                      # a chance neighbour pair aside, nothing aliases


@pytest.mark.parametrize("ignore_obs_next,steps", [(True, None), (False, 11), (True, 11)],
                         ids=["gathered_obs_next", "partly_filled", "partly_filled_gathered"])
def test_alias_map_of_sampled_buffers(ignore_obs_next, steps):
    """What ``_sample`` hands the value pass: obs_next gathered through ``next_index`` when the buffer does not store it,
    and gathered columns when the buffer is not full."""
    from tianshou_b200.utils import policy_within_training_step
    algo, _, _ = build_ppo(17, 6, DEV)
    buf = _buffer(6, 24, 17, 6, steps=steps, ignore_obs_next=ignore_obs_next)
    with policy_within_training_step(algo.policy):
        batch, _ = algo._sample(buf, 0)
    alias, extra = _check_map(batch.obs.cpu().numpy(), batch.obs_next.cpu().numpy())
    assert 0 < len(extra) < len(alias)


# --------------------------------------------------------------------------------- de-duplicated value pass
@pytest.mark.parametrize("obs_dim", [1, 16, 17, 32, 48])
def test_dedup_value_pass_is_bit_equal(obs_dim):
    """obs 1 .. 16 / 17 .. 32: the tensor-core kernel at both padded widths; obs 48: the fp32 SIMT kernel.  Few extra rows
    (a rollout), none but the last (one long segment), all of them (a shuffled batch); row counts off the tile size."""
    from tianshou_b200 import ops
    algo, actor, critic = build_ppo(obs_dim, 3, DEV)
    perturb_params(actor, critic, seed=obs_dim)
    assert (algo._flat.weight_image is not None) == (obs_dim <= 32)
    f, desc = algo._flat.flat, algo._desc
    cases = [_rollout(7, 300, obs_dim, p_term=0.02), _rollout(1, 1, obs_dim), _rollout(1, 129, obs_dim, p_term=0.0),
             _rollout(3, 128 * 5 // 3 + 1, obs_dim, p_term=0.0), _rollout(40, 1000, obs_dim, seed=2, p_term=0.01)]
    o, on = _rollout(9, 131, obs_dim)
    p = np.random.default_rng(5).permutation(len(o))
    cases.append((o[p], on[p]))
    for obs, obs_next in cases:
        obs_t, next_t = torch.from_numpy(obs).to(DEV), torch.from_numpy(obs_next).to(DEV)
        amap = ops.next_alias_map(obs_t, next_t)
        v_s, v_next = ops.critic_forward(f, desc, obs_t, next_t)
        d_s = torch.full_like(v_s, float("nan"))
        d_next = torch.full_like(v_next, float("nan"))        # every element must be written
        ops.critic_forward_dedup(f, desc, obs_t, next_t, amap, out=d_s, out2=d_next)
        assert torch.equal(v_s, d_s) and torch.equal(v_next, d_next), (obs_dim, len(obs), int(amap.count.item()))


# --------------------------------------------------------------------------------------------- whole updates
def _update(algo_name: str, with_map: bool, monkeypatch):
    from tianshou_b200.algorithm.modelfree.a2c import ActorCriticOnPolicyAlgorithm
    from tianshou_b200.utils import policy_within_training_step
    if algo_name == "ppo":
        algo, actor, critic = build_ppo(17, 6, DEV, recompute_advantage=True, value_clip=True, return_scaling=True,
                                        advantage_normalization=False)
    else:
        from tianshou_b200.algorithm import A2C, AdamOptimizerFactory, ProbabilisticActorPolicy
        from ts_testutil import Box, build_actor_critic, gaussian_dist
        actor, critic = build_actor_critic(17, 6, DEV)
        policy = ProbabilisticActorPolicy(actor=actor, dist_fn=gaussian_dist, action_scaling=True, action_bound_method="clip",
                                          action_space=Box(6))
        algo = A2C(policy=policy, critic=critic, optim=AdamOptimizerFactory(lr=3e-4), return_scaling=True)
    perturb_params(actor, critic, seed=7)
    used = []
    real = ActorCriticOnPolicyAlgorithm._next_alias_map

    def next_alias_map(self, batch, build=False):
        amap = real(self, batch, build) if with_map else None
        used.append(amap is not None)
        return amap
    buf = _buffer(64, 128, 17, 6)
    np.random.seed(11)
    with monkeypatch.context() as mp, policy_within_training_step(algo.policy):
        mp.setattr(ActorCriticOnPolicyAlgorithm, "_next_alias_map", next_alias_map)
        algo.update(buffer=buf, batch_size=2048, repeat=3)
    # the preprocess call, and for PPO the one C call that recomputes the advantages of passes 1 and 2
    assert used == [with_map] * (2 if algo_name == "ppo" else 1)
    return algo._flat.flat.detach().clone(), algo.last_loss_table.copy()


@pytest.mark.parametrize("algo_name", ["ppo", "a2c"])
def test_update_with_the_map_equals_update_without(algo_name, monkeypatch):
    p1, t1 = _update(algo_name, True, monkeypatch)
    p0, t0 = _update(algo_name, False, monkeypatch)
    assert torch.equal(p1, p0)
    assert np.array_equal(t1, t0)
