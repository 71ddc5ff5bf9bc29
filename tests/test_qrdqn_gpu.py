"""QR-DQN and discrete CQL on the GPU: the target and rows kernels against the float64 restatement (oracle/oracle_qrdqn.py),
``QRDQN.update()`` / ``DiscreteCQL.update()`` against outputs of the imported reference (tests/golden/{qrdqn,dcql}_ref_*.npz
from oracle/gen_golden_qrdqn.py), one update's gradient against float64 autograd, the ``state_dict()`` round trip, the
policy's torch path, the refusals and the kernels' register report."""
import copy

import numpy as np
import pytest
import torch

from oracle import oracle_discrete_sac as ods
from oracle import oracle_qrdqn as oq
from offpolicy_testutil import (DEV, EPS, Discrete, assert_spill_free, capture_batches, capture_grads, check_final_state,
                                ptxas_report, sm_count, stream, vector_buffer_from_golden)
from ts_testutil import load_golden, record_parity

gpu = pytest.mark.gpu
A_CASES = (1, 2, 6, 18)
N_CASES = (2, 200, 201)
VARIANTS = ["qrdqn_ref_mlp", "qrdqn_ref_cnn", "qrdqn_ref_per", "dcql_ref_mlp", "dcql_ref_cnn"]


# ------------------------------------------------------------------------------------------------------------ target kernel
@gpu
@pytest.mark.parametrize("N", N_CASES)
@pytest.mark.parametrize("A", A_CASES)
def test_target_kernel_matches_oracle(A, N):
    """Exact.  Integer-valued quantiles make every quantile sum exact in fp32 and float64 alike, so the means order the actions
    the same way in both and equal sums are exact ties: the first action of a tie must win.  B runs past the one-warp-per-row
    grid (16 blocks of 8 warps per SM) in one case."""
    from tianshou_b200._cabi import call, ptr
    g = torch.Generator().manual_seed(A * 1000 + N)
    B = sm_count() * 16 * 8 + 37 if (A, N) == (6, 200) else 301
    q = torch.randint(-3, 4, (B, A, N), generator=g).float()
    q_next = torch.randn(B, A, N, generator=g)
    if A > 1:
        q[: B // 3, A - 1] = q[: B // 3, 0]                          # two equal blocks: the first wins where they lead
    out, act = torch.empty(B, N, device=DEV), torch.empty(B, dtype=torch.int64, device=DEV)
    qd, nd = q.to(DEV), q_next.to(DEV)
    call("ts_qrdqn_target", ptr(qd), ptr(nd), B, A, N, ptr(out), ptr(act), stream())
    torch.cuda.synchronize()
    ref_a = oq.qr_select(q.numpy())
    assert np.array_equal(act.cpu().numpy(), ref_a) and np.array_equal(ref_a, q.mean(2).argmax(1).numpy())
    assert torch.equal(out.cpu(), q_next[torch.arange(B), torch.as_tensor(ref_a)])
    if A > 1:
        lead = q[: B // 3].sum(2).argmax(1) == 0
        assert bool(lead.any()) and bool((act.cpu()[: B // 3][lead] == 0).all())
    call("ts_qrdqn_target", ptr(qd), ptr(qd), B, A, N, ptr(out), None, stream())      # target_update_freq = 0: q_next is q_online
    torch.cuda.synchronize()
    assert torch.equal(out.cpu(), q[torch.arange(B), torch.as_tensor(ref_a)])


# ------------------------------------------------------------------------------------------------------------ rows kernel
def _rows(q, act, ret, tau, w, mqw):
    from tianshou_b200._cabi import call, ptr
    B, A, N = q.shape
    dq, prio = torch.empty(B, A, N, device=DEV), torch.empty(B, device=DEV)
    rows, losses = torch.empty(3, B, device=DEV), torch.empty(4, device=DEV)
    call("ts_qrdqn_rows", ptr(q), ptr(act), ptr(ret), ptr(tau), ptr(w), B, A, N, float(mqw), ptr(dq), ptr(prio), ptr(rows), ptr(losses),
         stream())
    torch.cuda.synchronize()
    return losses.cpu().numpy(), dq.cpu().numpy(), prio.cpu().numpy()


def oracle_rows_chunked(q, act, ret, tau, w, mqw, chunk=128):
    """``oq.qr_rows`` over row chunks (its [B, N, N] pair tensors stay small), recombined into batch means."""
    B = q.shape[0]
    losses, dqs, prios = np.zeros(3), [], []
    for s in range(0, B, chunk):
        e = min(B, s + chunk)
        r = oq.qr_rows(q[s:e], act[s:e], ret[s:e], tau, None if w is None else w[s:e], mqw)
        losses += r["losses"] * (e - s) / B
        dqs.append(r["dq"] * (e - s) / B)
        prios.append(r["prio"])
    return losses, np.concatenate(dqs), np.concatenate(prios)


def pair_terms(q, act, ret, tau):
    """Per row and current quantile i: sum_j h_ij w_ij, sum_j h_ij and sum_j |w_ij clip(u_ij)| in float64 (the magnitudes the
    error model scales with), in row chunks."""
    out = []
    for s in range(0, q.shape[0], 128):
        c = q[s:s + 128][np.arange(min(128, q.shape[0] - s)), act[s:s + 128], :]
        u = ret[s:s + 128, None, :] - c[:, :, None]
        au = np.abs(u)
        h = np.where(au < 1.0, 0.5 * u * u, au - 0.5)
        wt = np.abs(tau[None, :, None] - (u <= 0.0))
        out.append(np.stack([(h * wt).sum(-1), h.sum(-1), np.abs(wt * np.clip(u, -1, 1)).sum(-1)]))
    return np.concatenate(out, axis=1)            # [3, B, N]


@gpu
@pytest.mark.parametrize("mqw", [0.0, 10.0])
@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("N", N_CASES)
@pytest.mark.parametrize("A", A_CASES)
def test_rows_kernel_vs_fp64(A, N, weighted, mqw):
    """Losses, priorities and d loss / d q against the float64 restatement (pinned to autograd of the reference's expression in
    test_oracle_qrdqn), with pairs at u == 0 exactly (indicator true) and |u| == 1 exactly (the Huber knee).

    Error model (fp32, eps = 2^-23): u = t - c is one rounding, h and |tau - 1[u <= 0]| a few more, and each thread sums its N
    pair terms in order: a row's quantile sum is off by at most (N + 4) eps times the sum of its terms' magnitudes; the CTA then
    adds ceil(N / 256) per-thread partials, five butterfly levels and eight warp partials, (N + 20) eps in all for qr_b and
    prio_b (every term is >= 0).  A quantile mean is off by (N / 32 + 6) eps times the mean magnitude of its row (lanes add
    ceil(N / 32) values, then five levels); softmax and logsumexp over A add (A / 32 + 10) eps.  The batch means come from
    row_sums3_kernel: (B / 1024 + 12) eps times the mean magnitude."""
    rng = np.random.default_rng(A * 7919 + N * 31 + weighted * 3 + int(mqw))
    B = sm_count() * 8 + 37 if (A, N, weighted) == (6, 200, True) else 41
    q = (rng.standard_normal((B, A, N)) * 2).astype(np.float32)
    act = rng.integers(0, A, B)
    ret = (q[np.arange(B), act, :] + rng.standard_normal((B, N)) * 1.5).astype(np.float32)
    ret[0, 0] = q[0, act[0], N - 1]                                       # u = 0 exactly
    q[1, act[1], 0], ret[1, 0], ret[1, 1] = 0.5, -0.5, 1.5                # |u| = 1 exactly, both signs
    w = rng.uniform(0.2, 1.0, B).astype(np.float32) if weighted else None
    tau32 = oq.tau_hat(N)
    tau = tau32.astype(np.float64)
    dev = lambda a, dt=torch.float32: torch.as_tensor(a, dtype=dt, device=DEV)
    args = (dev(q), dev(act, torch.int64), dev(ret), dev(tau32), None if w is None else dev(w), mqw)
    losses, dq, prio = _rows(*args)
    q64, ret64 = q.astype(np.float64), ret.astype(np.float64)
    ref_l, ref_dq, ref_p = oracle_rows_chunked(q64, act, ret64, tau, None if w is None else w.astype(np.float64), mqw)
    terms = pair_terms(q64, act, ret64, tau)                    # [3, B, N]
    wb = np.ones(B) if w is None else w.astype(np.float64)
    qr_b = terms[0].sum(1) / N
    rel = (N + 20) * EPS
    tag = f"qrdqn_rows/A{A}_N{N}_w{int(weighted)}_m{int(mqw)}"
    record_parity(f"{tag}/prio", prio, ref_p, rtol=rel, atol=1e-30)
    m = q64.mean(2)
    dm = (N / 32 + 6) * EPS * np.abs(q64).mean(2)               # [B, A]
    lse = m.max(1) + np.log(np.exp(m - m.max(1, keepdims=True)).sum(1))
    p = np.exp(m - lse[:, None])
    soft = (A / 32 + 10) * EPS
    cql_rows = lse - m[np.arange(B), act]
    cql_err = 2 * dm.max(1) + soft * np.abs(lse) + EPS * (np.abs(lse) + np.abs(m[np.arange(B), act]))
    bounds = np.array([0.0, (wb * qr_b * rel).mean() + (np.ceil(B / 1024) + 12) * EPS * (wb * qr_b).mean(),
                       (cql_err.mean() + (np.ceil(B / 1024) + 12) * EPS * np.abs(cql_rows).mean()) if mqw else 0.0])
    bounds[0] = bounds[1] + mqw * bounds[2] + 4 * EPS * abs(ref_l[0])
    err = np.abs(losses[:3] - ref_l)
    assert np.all(err <= bounds + 1e-30), f"{tag}: losses off by {err} past {bounds}"
    record_parity(f"{tag}/losses", losses[:3], ref_l, rtol=0.0, atol=float(bounds.max()) + 1e-30)
    # d loss / d q: the taken block's quantile term, plus (CQL) min_q_weight / (B N) (p_a - 1[a == act]) on every element
    bound = np.zeros((B, A, N))
    bound[np.arange(B), act, :] = (N + 4) * EPS * terms[2] * (wb / (B * N))[:, None]
    if mqw:
        rel_p = 2 * dm.max(1, keepdims=True) + soft + 4 * EPS + EPS * (m.max(1, keepdims=True) - m)
        bound += (mqw / (B * N)) * (p * rel_p + 2 * EPS * (p + 1.0))[:, :, None]
    bound += 4 * EPS * np.abs(ref_dq) + 1e-30
    e = np.abs(dq - ref_dq)
    assert np.all(e <= bound), f"{tag}: dq error {float((e - bound).max()):.3e} past its bound"
    record_parity(f"{tag}/dq", dq, ref_dq, rtol=0.0, atol=float(bound.max()))
    again = _rows(*args)
    assert all(np.array_equal(a, b) for a, b in zip((losses, dq, prio), again)), "two calls must be bit-identical"


@gpu
def test_rows_kernel_refuses_what_shared_memory_cannot_hold():
    from tianshou_b200._cabi import call, ptr
    x = torch.zeros(16, device=DEV)
    a = torch.zeros(1, dtype=torch.int64, device=DEV)
    for A, N, mqw in ((1, 6145, 0.0), (100, 6100, 1.0), (1, 1, 0.0)):
        with pytest.raises(RuntimeError, match="ts_qrdqn_rows"):
            call("ts_qrdqn_rows", ptr(x), ptr(a), ptr(x), ptr(x), None, 1, A, N, mqw, ptr(x), ptr(x), ptr(x), ptr(x), stream())


# ------------------------------------------------------------------------------------------------------------ vs reference
def model_from_cfg(kind, A, N, obs=4, hidden=(64,), H=44, W=44, scale=True):
    from tianshou_b200.env.atari import QRDQNet, ScaledObsInputActionReprNet
    from tianshou_b200.utils.net.common import Net
    if kind == "cnn":
        net = QRDQNet(c=4, h=H, w=W, action_shape=A, num_quantiles=N)
        return (ScaledObsInputActionReprNet(net) if scale else net).to(DEV)
    return Net(state_shape=(obs,), action_shape=A, hidden_sizes=hidden, num_atoms=N).to(DEV)


def build_from_golden(g):
    from tianshou_b200.algorithm import AdamOptimizerFactory, DiscreteCQL, QRDQN, QRDQNPolicy
    kind = str(g["cfg_kind"])
    kw = (dict(H=int(g["cfg_H"]), W=int(g["cfg_W"]), scale=bool(g["cfg_scale"])) if kind == "cnn"
          else dict(obs=int(g["cfg_obs"]), hidden=tuple(int(x) for x in g["cfg_hidden"])))
    A, N = int(g["cfg_A"]), int(g["cfg_N"])
    model = model_from_cfg(kind, A, N, **kw)
    ods.seeded_params(model, int(g["cfg_init_seed"]))
    policy = QRDQNPolicy(model=model, action_space=Discrete(A))
    akw = dict(policy=policy, optim=AdamOptimizerFactory(lr=float(g["cfg_lr"])), gamma=float(g["cfg_gamma"]), num_quantiles=N,
               n_step_return_horizon=int(g["cfg_n_step"]), target_update_freq=int(g["cfg_freq"]))
    if str(g["cfg_algo"]) == "dcql":
        return DiscreteCQL(min_q_weight=float(g["cfg_min_q_weight"]), **akw)
    return QRDQN(**akw)


@gpu
@pytest.mark.parametrize("mirror", [False, True])
@pytest.mark.parametrize("variant", VARIANTS)
def test_update_matches_reference(variant, mirror):
    """Update after update against the reference's run: the same sampled indices, n-step returns over N columns, losses, the
    priorities written back (PER: and the sum-tree leaves), then the final state."""
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden(f"{variant}.npz")
    algo, buf = build_from_golden(g), vector_buffer_from_golden(g, mirror)
    keys = [str(k) for k in g["state_dict_keys"]]
    assert list(algo.state_dict().keys()) == keys
    dcql = str(g["cfg_algo"]) == "dcql"
    with capture_batches(algo) as cap:
        for u in range(int(g["cfg_updates"])):
            np.random.seed(500 + u)
            with policy_within_training_step(algo.policy):
                stats = algo.update(buffer=buf, sample_size=int(g["cfg_bs"]))
            tag = f"{variant}_m{int(mirror)}_u{u}"
            assert np.array_equal(cap["indices"], g[f"u{u}_indices"]), "sampled indices differ from the reference's"
            ref_ret = g[f"u{u}_returns"]
            record_parity(f"{tag}/returns", cap["returns"].cpu().numpy(), ref_ret, rtol=1e-5, atol=1e-5 * float(np.abs(ref_ret).max()))
            got = np.array([stats.loss, stats.qr_loss, stats.cql_loss] if dcql else [stats.loss])
            record_parity(f"{tag}/losses", got, g[f"u{u}_losses"], rtol=2e-5, atol=2e-6)
            record_parity(f"{tag}/prio", cap["prio"].cpu().numpy(), g[f"u{u}_prio"], rtol=2e-5, atol=2e-6)
            if bool(g["cfg_per"]):
                leaves = np.asarray(buf.weight[np.arange(len(buf))])
                record_parity(f"{tag}/tree_leaves", leaves, g[f"u{u}_tree_leaves"], rtol=2e-5, atol=1e-7)
    check_final_state(f"{variant}_m{int(mirror)}", g, algo)
    assert list(algo.state_dict().keys()) == keys


def make_buffer(kind, A, rng, E=4, T=48):
    from tianshou_b200.data import Batch, VectorReplayBuffer
    cnn = kind == "cnn"
    buf = VectorReplayBuffer(E * T, E, device=DEV, **(dict(stack_num=1, ignore_obs_next=True) if cnn else {}))
    obs_fn = (lambda: rng.integers(0, 256, (E, 4, 44, 44), dtype=np.uint8)) if cnn else (lambda: rng.standard_normal((E, 4)).astype(np.float32))
    obs = obs_fn()
    for t in range(T):
        nxt = obs_fn()
        term = rng.random(E) < 0.1
        buf.add(Batch(obs=obs, act=rng.integers(0, A, E), rew=rng.standard_normal(E) * 2, terminated=term,
                      truncated=np.full(E, t % 17 == 16) & ~term, obs_next=nxt), buffer_ids=np.arange(E))
        obs = nxt
    return buf


@gpu
@pytest.mark.parametrize("kind,mqw", [("mlp", 0.0), ("mlp", 10.0), ("cnn", 10.0)])
def test_update_gradient_vs_fp64_autograd(kind, mqw):
    grad_case(kind, mqw)


def grad_case(kind, mqw, B=64, edge=""):
    """One update at batch ``B`` (64 in the suite's own cases): the flat gradient, snapshotted before its Adam step, against
    float64 autograd of the reference's loss
    (qrdqn.py:114-128, discrete_cql.py:86-106) on a copy of the module with the same weights, batch and returns.  Adam's first
    step is lr * sign(g), so a gradient off by a constant factor leaves the parameters unchanged; this is the check that sees it.
    The GEMMs are fp32-faithful (bf16x3) and a weight gradient sums B products per element: 2e-4 relative plus 1e-4 of the
    tensor's largest value, as in test_discrete_bcq_gpu."""
    from tianshou_b200.algorithm import AdamOptimizerFactory, DiscreteCQL, QRDQN, QRDQNPolicy
    from tianshou_b200.utils import policy_within_training_step
    torch.manual_seed(3)
    rng = np.random.default_rng(4)
    A, N = 5, 33
    model = model_from_cfg(kind, A, N, hidden=(48, 40))
    policy = QRDQNPolicy(model=model, action_space=Discrete(A))
    kw = dict(policy=policy, optim=AdamOptimizerFactory(lr=1e-3), gamma=0.9, num_quantiles=N, n_step_return_horizon=2,
              target_update_freq=3)
    algo = DiscreteCQL(min_q_weight=mqw, **kw) if mqw else QRDQN(**kw)
    buf = make_buffer(kind, A, rng)
    grp = algo._group
    ref = copy.deepcopy(model).to("cpu", torch.float64)         # the weights before the step
    np.random.seed(7)
    with capture_batches(algo) as cap, capture_grads(grp) as grads, policy_within_training_step(algo.policy):
        stats = algo.update(buffer=buf, sample_size=B)
    idx, returns = cap["indices"], cap["returns"].cpu().double()
    raw = np.asarray(buf.obs)[idx]
    x = torch.as_tensor((raw.astype(np.float64) / 255.0).astype(np.float32) if kind == "cnn" else raw).double()
    inner = ref.module if kind == "cnn" else ref
    chain = inner.net if kind == "cnn" else inner.model.model
    q = chain(x).view(B, A, N)
    act = np.asarray(buf.act)[idx].astype(np.int64)
    loss, qr, cql, _ = oq.reference_loss(q, act, returns, torch.as_tensor(oq.tau_hat(N), dtype=torch.float64), 1.0, mqw)
    loss.backward()
    ref_params = [p for m in chain.modules() if isinstance(m, (torch.nn.Linear, torch.nn.Conv2d)) for p in (m.weight, m.bias)]
    for i, (p, r) in enumerate(zip(grp.params, ref_params, strict=True)):
        want = r.grad.numpy()
        got = grp.view(grads[-1], p).view(p.shape).cpu().numpy()
        record_parity(f"qrdqn_grad{edge}/{kind}_m{int(mqw)}/grad_{i}", got, want, rtol=2e-4, atol=1e-4 * float(np.abs(want).max()) + 1e-12)
    got = [stats.loss, stats.qr_loss, stats.cql_loss] if mqw else [stats.loss]
    want = [loss.item(), qr.item(), cql.item()] if mqw else [loss.item()]
    record_parity(f"qrdqn_grad{edge}/{kind}_m{int(mqw)}/losses", np.array(got), np.array(want), rtol=2e-5, atol=2e-6)
    assert len(idx) == B and returns.shape[0] == B, "the update must run on the B sampled rows"


# ------------------------------------------------------------------------------------------------------------ state_dict
@gpu
@pytest.mark.parametrize("variant", ["dcql_ref_mlp", "qrdqn_ref_cnn"])
def test_state_dict_round_trip_continues_identically(variant):
    """A fresh algorithm loaded from another's ``state_dict()`` continues bit for bit: online, lagged and optimiser state.
    ``_iter`` is a plain attribute, as in the reference: whoever restores a run restores it too."""
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden(f"{variant}.npz")
    a, buf_a = build_from_golden(g), vector_buffer_from_golden(g)
    for u in range(3):
        np.random.seed(u)
        with policy_within_training_step(a.policy):
            a.update(buffer=buf_a, sample_size=int(g["cfg_bs"]))
    b = build_from_golden(g)
    with torch.no_grad():
        for p in b.policy.parameters():
            p.add_(0.01)
    b.load_state_dict(copy.deepcopy(a.state_dict()))
    b._iter = a._iter
    assert torch.equal(a.tau_hat, b.tau_hat)
    for algo in (a, b):
        buf = vector_buffer_from_golden(g)
        for u in range(3):
            np.random.seed(10 + u)
            with policy_within_training_step(algo.policy):
                algo.update(buffer=buf, sample_size=int(g["cfg_bs"]))
    pairs = [(a._group, b._group)] + ([(a._g_old, b._g_old)] if a._g_old is not None else [])
    for ga, gb in pairs:
        assert torch.equal(ga.flat, gb.flat) and torch.equal(ga.exp_avg, gb.exp_avg) and torch.equal(ga.exp_avg_sq, gb.exp_avg_sq)
    assert a._group.step == b._group.step


# ------------------------------------------------------------------------------------------------------------ policy
@gpu
def test_policy_forward_takes_arg_max_of_quantile_means():
    from tianshou_b200.algorithm import QRDQNPolicy
    from tianshou_b200.data import Batch
    torch.manual_seed(0)
    model = model_from_cfg("mlp", 5, 17, obs=4, hidden=(32,))
    policy = QRDQNPolicy(model=model, action_space=Discrete(5))
    obs = np.random.default_rng(0).standard_normal((300, 4)).astype(np.float32)
    out = policy(Batch(obs=obs, info=Batch()))
    logits, _ = model(obs)
    assert out.logits.shape == (300, 5, 17) and torch.equal(out.logits, logits)
    assert np.array_equal(out.act, logits.mean(2).argmax(1).cpu().numpy())


# ------------------------------------------------------------------------------------------------------------ refusals
@gpu
def test_refusals():
    from tianshou_b200.algorithm import (AdamOptimizerFactory, DiscreteCQL, QRDQN, QRDQNPolicy, RMSpropOptimizerFactory,
                                         UnsupportedModelError)
    from tianshou_b200.data import Batch, VectorReplayBuffer
    from tianshou_b200.utils import policy_within_training_step
    from tianshou_b200.utils.net.common import Net
    A, N = 3, 8

    def make(model=None, opt=AdamOptimizerFactory, n=A, cls=QRDQN, **kw):
        model = model or model_from_cfg("mlp", A, N, hidden=(16,))
        return cls(policy=QRDQNPolicy(model=model, action_space=Discrete(n)), optim=opt(lr=1e-3), num_quantiles=N, **kw)

    algo = make()
    with pytest.raises(UnsupportedModelError, match="softmax"):
        make(Net(state_shape=(4,), action_shape=A, hidden_sizes=(16,), num_atoms=N, softmax=True).to(DEV))
    with pytest.raises(UnsupportedModelError, match="outputs, not 3 actions x 8 quantiles"):
        make(model_from_cfg("mlp", A, N + 1, hidden=(16,)))
    with pytest.raises(UnsupportedModelError, match="outputs, not 4 actions"):
        make(n=4)
    with pytest.raises(UnsupportedModelError, match="Adam"):
        make(opt=RMSpropOptimizerFactory)
    with pytest.raises(UnsupportedModelError, match="no CPU path"):
        make(model_from_cfg("mlp", A, N, hidden=(16,)).cpu())
    for kw in (dict(gamma=1.5), dict(n_step_return_horizon=0)):
        with pytest.raises(AssertionError):
            make(**kw)
    with pytest.raises(AssertionError, match="num_quantiles"):
        QRDQN(policy=QRDQNPolicy(model=model_from_cfg("mlp", A, 1, hidden=(16,)), action_space=Discrete(A)),
              optim=AdamOptimizerFactory(lr=1e-3), num_quantiles=1)
    with pytest.raises(ValueError, match="min_q_weight"):
        make(cls=DiscreteCQL, min_q_weight=-1.0)
    # an action the network has no quantiles for is refused on the host, before any kernel indexes with it
    buf = VectorReplayBuffer(40, 4, device=DEV)
    rng = np.random.default_rng(0)
    for _ in range(8):
        buf.add(Batch(obs=rng.standard_normal((4, 4)).astype(np.float32), act=np.array([0, 1, 2, A]), rew=np.zeros(4),
                      terminated=np.zeros(4, bool), truncated=np.zeros(4, bool), obs_next=rng.standard_normal((4, 4)).astype(np.float32)),
                buffer_ids=np.arange(4))
    with pytest.raises(ValueError, match="actions in"), policy_within_training_step(algo.policy):
        algo.update(buffer=buf, sample_size=32)


# ------------------------------------------------------------------------------------------------------------ resources
def test_kernels_have_no_stack_frame_or_spills(tmp_path):
    report = ptxas_report("qrdqn.cu", tmp_path)
    kernels = ("qrdqn_rows_kernel", "qrdqn_target_kernel", "row_sums3_kernel")
    assert len(report) == 3 and all(any(k in e for k in kernels) for e in report), report
    assert_spill_free(report)
