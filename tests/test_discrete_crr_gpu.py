"""Discrete CRR on the GPU: the rows kernel against float64 (the restatement pinned to autograd in test_oracle_discrete_crr),
``DiscreteCRR.update()`` against outputs of the imported reference (tests/golden/dcrr_ref_*.npz from
oracle/gen_golden_discrete_crr.py), the flat gradient of one update against float64 autograd, ``state_dict()`` keys and round
trip, and the refusals."""
import copy

import numpy as np
import pytest
import torch
from torch.distributions import Categorical

from oracle import oracle_discrete_crr as odc
from offpolicy_testutil import (DEV, EPS, Discrete, capture_batches, capture_grads, check_final_state, stream,
                                vector_buffer_from_golden)
from test_discrete_bcq_gpu import A_CASES, TRUNK_CASES, chain64, check_flat_grads, copy64, heads_from_golden, make_heads, past_grid_rows
from ts_testutil import load_golden, record_parity

gpu = pytest.mark.gpu


def _crr_rows(q, z, act, qo, zo, rew, done, gamma, mode, beta, bound, w):
    from tianshou_b200._cabi import ABI, call, ptr
    B, A = q.shape
    dq, dz = torch.empty(B, A, device=DEV), torch.empty(B, A, device=DEV)
    rows, losses = torch.empty(4 * B + 2, device=DEV), torch.empty(4, device=DEV)
    code = ABI.consts[{"exp": "TS_CRR_EXP", "binary": "TS_CRR_BINARY", "all": "TS_CRR_ALL"}[mode]]
    call("ts_discrete_crr_rows", ptr(q), ptr(z), ptr(act), ptr(qo), ptr(zo), ptr(rew), ptr(done), B, A, gamma, code, beta, bound, w,
         ptr(dq), ptr(dz), ptr(rows), ptr(losses), stream())
    torch.cuda.synchronize()
    return losses.cpu().numpy(), dq.cpu().numpy(), dz.cpu().numpy()


@gpu
@pytest.mark.parametrize("mode", ["exp", "binary", "all"])
@pytest.mark.parametrize("A", A_CASES)
def test_rows_kernel_vs_fp64(A, mode):
    """Losses and both gradients against float64 on rows with ``done``, advantages of both signs and exactly 0, the clamp
    saturated and not, and logit spreads that underflow probabilities.  A row's sums carry ~(A / 32 + 10) eps of the magnitudes
    of their terms; exp(adv / beta) multiplies the advantage's absolute error by 1 / beta; rows whose float64 advantage or
    coefficient sits within that error of a branch point (adv = 0, the clamp's bound) may fall on either side in fp32 and are
    left out of the element-wise comparison."""
    g = torch.Generator().manual_seed(100 + A)
    B = past_grid_rows() if A == 6 else 301
    gamma, beta, bound, w = 0.9, 0.7, 2.0, 3.0
    q = torch.randn(B, A, generator=g) * 2
    z = torch.randn(B, A, generator=g) * 3
    z[: B // 4] *= 40.0
    qo, zo = torch.randn(B, A, generator=g) * 2, torch.randn(B, A, generator=g) * 3
    act = torch.randint(0, A, (B,), generator=g)
    q[5:9] = 0.0                                   # every q zero: the advantage is exactly 0 in any precision
    rew = torch.randn(B, generator=g)
    done = (torch.rand(B, generator=g) < 0.3).float()
    dev = [t.to(DEV) for t in (q, z, act, qo, zo, rew, done)]
    losses, dq, dz = _crr_rows(*dev, gamma, mode, beta, bound, w)
    r = odc.crr_rows(q.numpy(), z.numpy(), act.numpy(), qo.numpy(), zo.numpy(), rew.numpy(), done.numpy(), gamma, mode, beta, bound, w)
    assert done.sum() > 0 and (r["adv"][5:9] == 0).all()
    if A > 1:
        assert (r["adv"] > 0).any() and (r["adv"] < 0).any()
    if mode == "exp" and A > 1:
        assert (r["coef"] == bound).any() and (r["coef"] < bound).any()
    k = (np.ceil(A / 32) + 10) * EPS
    adv_err = k * (np.abs(q.double().numpy()).sum(-1) + 1.0) * 4
    e64 = np.exp(np.minimum(r["adv"] / beta, 50.0))
    near = {"exp": np.abs(e64 - bound) <= e64 * adv_err / beta * 2, "binary": (np.abs(r["adv"]) <= adv_err) & (r["adv"] != 0),
            "all": np.zeros(B, bool)}[mode]
    assert near.mean() < 0.05
    tag = f"dcrr_rows/A{A}_{mode}"
    scale = np.abs(r["losses"]).max()
    # the four means: row errors average, the block sum adds (B / 1024 + 12) eps; near-branch rows move actor_loss by <= 1 / B each
    atol = 64 * k * scale + near.sum() * bound * abs(r["losses"][1]) / B + 1e-6
    record_parity(f"{tag}/losses", losses, r["losses"], rtol=1e-5, atol=float(atol))
    keep = ~near
    if near.any():        # a flipped row changes mean(coef), which scales every row's dlogits
        return
    row_scale = np.abs(r["dq"]).max(-1, keepdims=True) + 1.0 / B
    record_parity(f"{tag}/dq", (dq / row_scale)[keep], (r["dq"] / row_scale)[keep], rtol=0.0, atol=float(256 * k * (1 + 1 / beta)))
    row_scale = np.abs(r["dlogits"]).max(-1, keepdims=True) + 1.0 / B
    record_parity(f"{tag}/dlogits", (dz / row_scale)[keep], (r["dlogits"] / row_scale)[keep], rtol=0.0, atol=float(256 * k * (1 + 1 / beta)))
    again = _crr_rows(*dev, gamma, mode, beta, bound, w)
    assert all(np.array_equal(a, b) for a, b in zip((losses, dq, dz), again)), "two calls must be bit-identical"


def build_crr(g, **over):
    from tianshou_b200.algorithm import AdamOptimizerFactory, DiscreteActorPolicy, DiscreteCRR
    actor, critic = heads_from_golden(g, critic_b=True)
    kw = dict(gamma=float(g["cfg_gamma"]), policy_improvement_mode=str(g["cfg_mode"]), ratio_upper_bound=float(g["cfg_bound"]),
              beta=float(g["cfg_beta"]), min_q_weight=float(g["cfg_min_q_weight"]), target_update_freq=int(g["cfg_freq"]),
              return_standardization=bool(g["cfg_ret_std"]))
    kw.update(over)
    return DiscreteCRR(policy=DiscreteActorPolicy(actor=actor, action_space=Discrete(int(g["cfg_A"]))), critic=critic,
                       optim=AdamOptimizerFactory(lr=float(g["cfg_lr"])), **kw)


@gpu
@pytest.mark.parametrize("variant,mirror", [("mlp", False), ("mlp", True), ("cnn", False), ("cnn", True), ("sep", False)])
def test_update_matches_reference(variant, mirror):
    """All three modes, ``target_update_freq`` 0 (cnn) and several lagged copies (mlp, sep), which must fall on the updates the
    reference copies on: the golden's lagged parameters are the last copy's."""
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden(f"dcrr_ref_{variant}.npz")
    algo, buf = build_crr(g), vector_buffer_from_golden(g, mirror)
    assert list(algo.state_dict().keys()) == [str(k) for k in g["state_dict_keys"]]
    with capture_batches(algo) as cap:
        for u in range(int(g["cfg_updates"])):
            np.random.seed(500 + u)
            with policy_within_training_step(algo.policy):
                stats = algo.update(buffer=buf, sample_size=int(g["cfg_bs"]))
            assert np.array_equal(cap["indices"], g[f"u{u}_indices"]), "sampled indices differ from the reference's"
            got = np.array([stats.loss, stats.actor_loss, stats.critic_loss, stats.cql_loss])
            record_parity(f"dcrr_{variant}_m{int(mirror)}_u{u}/losses", got, g[f"u{u}_losses"], rtol=2e-5, atol=2e-6)
    lagged = [*algo.actor_old.parameters(), *algo.critic_old.parameters()] if int(g["cfg_freq"]) > 0 else []
    check_final_state(f"dcrr_{variant}_m{int(mirror)}", g, algo, lagged)
    # return standardisation changes nothing: the loss never reads the returns
    if variant == "sep" and not mirror:
        other, buf2 = build_crr(g, return_standardization=False), vector_buffer_from_golden(g)
        for u in range(int(g["cfg_updates"])):
            np.random.seed(500 + u)
            with policy_within_training_step(other.policy):
                other.update(buffer=buf2, sample_size=int(g["cfg_bs"]))
        assert torch.equal(other._group.flat, algo._group.flat)


@gpu
@pytest.mark.parametrize("mode", ["exp", "binary", "all"])
@pytest.mark.parametrize("name,kind,shared,kw", TRUNK_CASES[:4], ids=[c[0] for c in TRUNK_CASES[:4]])
def test_update_gradient_vs_fp64_autograd(name, kind, shared, kw, mode):
    grad_case(name, kind, shared, kw, mode)


def grad_case(name, kind, shared, kw, mode, B=64, edge=""):
    """One update at batch ``B`` (64 in the suite's own cases) with a lagged copy: the flat gradient before its Adam step
    against float64 autograd of the reference loss
    (discrete_crr.py:131-158, its [B] x [B, 1] broadcast included) on copies of the modules."""
    from tianshou_b200.algorithm import AdamOptimizerFactory, DiscreteActorPolicy, DiscreteCRR
    from tianshou_b200.algorithm.shared_trunk import two_head_parameters
    from tianshou_b200.data import Batch, VectorReplayBuffer
    from tianshou_b200.utils import policy_within_training_step
    torch.manual_seed(9 + len(name))
    rng = np.random.default_rng(len(name) + len(mode))
    A, E, T, gamma, beta, bound, w = 6, 4, 48, 0.9, 0.5, 1.1, 3.0
    actor, critic = make_heads(kind, shared, A, (24,), critic_b=True, **kw)
    algo = DiscreteCRR(policy=DiscreteActorPolicy(actor=actor, action_space=Discrete(A)), critic=critic, optim=AdamOptimizerFactory(lr=1e-3),
                       gamma=gamma, policy_improvement_mode=mode, ratio_upper_bound=bound, beta=beta, min_q_weight=w, target_update_freq=2)
    with torch.no_grad():         # the lagged networks differ from the online ones
        for p in [*algo.actor_old.parameters(), *algo.critic_old.parameters()]:
            p.mul_(1.1)
        if shared:
            for tp, sp in zip(algo.critic_old.module.preprocess.parameters(), algo.actor_old.module.preprocess.parameters()):
                tp.copy_(sp)
    algo._iter = 1                # no copy in this update
    cnn = kind == "cnn"
    buf = VectorReplayBuffer(E * T, E, device=DEV, **(dict(stack_num=1, ignore_obs_next=True) if cnn else {}))
    obs_fn = (lambda: rng.integers(0, 256, (E, 4, 44, 44), dtype=np.uint8)) if cnn else (lambda: rng.standard_normal((E, 11)).astype(np.float32))
    obs = obs_fn()
    for t in range(T):
        nxt = obs_fn()
        term = rng.random(E) < 0.1
        buf.add(Batch(obs=obs, act=rng.integers(0, A, E), rew=rng.standard_normal(E) * 2, terminated=term,
                      truncated=np.full(E, t % 17 == 16) & ~term, obs_next=nxt), buffer_ids=np.arange(E))
        obs = nxt
    grp = algo._group
    ref, ref_old = copy64(actor, critic), copy64(algo.actor_old.module, algo.critic_old.module)
    np.random.seed(7)
    with capture_batches(algo) as cap, capture_grads(grp) as grads, policy_within_training_step(algo.policy):
        stats = algo.update(buffer=buf, sample_size=B)
    idx = cap["indices"]
    rd = lambda a: torch.as_tensor((a.astype(np.float64) / 255.0).astype(np.float32) if cnn else a).double()
    x = rd(np.asarray(buf.obs)[idx])
    xn = rd(np.asarray(buf.obs)[buf.next(idx)] if cnn else np.asarray(buf.obs_next)[idx])
    act = torch.as_tensor(np.asarray(buf.act)[idx].astype(np.int64))
    rew = torch.as_tensor(np.asarray(buf.rew)[idx].astype(np.float32)).double()
    done = torch.as_tensor(np.asarray(buf.done)[idx])
    z, q = chain64(ref[0])(x), chain64(ref[1])(x)
    qa = q.gather(1, act.unsqueeze(1))
    with torch.no_grad():
        eq = (chain64(ref_old[1])(xn) * Categorical(logits=chain64(ref_old[0])(xn)).probs).sum(-1, keepdim=True)
        eq[done > 0] = 0.0
        target = rew.unsqueeze(1) + gamma * eq
    critic_loss = 0.5 * torch.nn.functional.mse_loss(qa, target)
    dist = Categorical(logits=z)
    adv = qa - (q * dist.probs).sum(-1, keepdim=True)
    coef = {"binary": (adv > 0).double(), "exp": (adv / beta).exp().clamp(0, bound), "all": 1.0}[mode]
    actor_loss = (-dist.log_prob(act) * coef).mean()
    cql = (q.logsumexp(1) - qa.squeeze(-1)).mean()
    loss = actor_loss + critic_loss + w * cql
    loss.backward()
    check_flat_grads(f"dcrr_grad{edge}/{name}_{mode}", grp.params, grp, grads[-1], two_head_parameters(ref[0], ref[1]))
    record_parity(f"dcrr_grad{edge}/{name}_{mode}/losses", np.array([stats.loss, stats.actor_loss, stats.critic_loss, stats.cql_loss]),
                  np.array([loss.item(), actor_loss.item(), critic_loss.item(), cql.item()]), rtol=5e-5, atol=5e-6)
    assert len(idx) == B, "the update must run on the B sampled rows"


@gpu
def test_state_dict_round_trip_continues_identically():
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden("dcrr_ref_mlp.npz")
    a, buf_a = build_crr(g), vector_buffer_from_golden(g)
    for u in range(3):
        np.random.seed(u)
        with policy_within_training_step(a.policy):
            a.update(buffer=buf_a, sample_size=int(g["cfg_bs"]))
    b = build_crr(g)
    with torch.no_grad():
        for p in b.parameters():
            p.add_(0.01)
    b.load_state_dict(copy.deepcopy(a.state_dict()))
    b._iter = a._iter             # a plain attribute, as in the reference: whoever restores a run restores it too
    for algo in (a, b):
        buf = vector_buffer_from_golden(g)
        for u in range(3):
            np.random.seed(10 + u)
            with policy_within_training_step(algo.policy):
                algo.update(buffer=buf, sample_size=int(g["cfg_bs"]))
    for ga, gb in ((a._group, b._group), (a._g_old, b._g_old)):
        assert torch.equal(ga.flat, gb.flat) and torch.equal(ga.exp_avg, gb.exp_avg) and torch.equal(ga.exp_avg_sq, gb.exp_avg_sq)


@gpu
def test_refusals():
    from tianshou_b200.algorithm import AdamOptimizerFactory, DiscreteActorPolicy, DiscreteCRR, UnsupportedModelError
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.discrete import DiscreteActor, DiscreteCritic
    A = 3
    trunk = Net(state_shape=(11,), hidden_sizes=(16,))

    def make(actor=None, critic=None, n=A):
        actor = actor or DiscreteActor(preprocess_net=trunk, action_shape=A, softmax_output=False)
        critic = critic or DiscreteCritic(preprocess_net=trunk, last_size=A)
        return DiscreteCRR(policy=DiscreteActorPolicy(actor=actor.to(DEV), action_space=Discrete(n)), critic=critic.to(DEV),
                           optim=AdamOptimizerFactory(lr=1e-3))

    make()
    with pytest.raises(UnsupportedModelError, match="softmax_output=True"):
        make(DiscreteActor(preprocess_net=trunk, action_shape=A, softmax_output=True))
    with pytest.raises(UnsupportedModelError, match="critic has 1 outputs for 3 actions"):
        make(critic=DiscreteCritic(preprocess_net=trunk))
    with pytest.raises(UnsupportedModelError, match="must read it the same way"):
        make(critic=DiscreteCritic(preprocess_net=Net(state_shape=(5,), hidden_sizes=(16,)), last_size=A))
