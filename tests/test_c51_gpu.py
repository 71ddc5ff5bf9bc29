"""C51 on the GPU: the target and rows kernels against the float64 restatement (oracle/oracle_c51.py), ``C51.update()`` against
outputs of the imported reference (tests/golden/c51_ref_*.npz from oracle/gen_golden_c51.py), one update's gradient against
float64 autograd, the batch sizes the kernels and GEMMs split on, the ``state_dict()`` round trip, the policy's torch path, the
refusals and the kernels' register report."""
import copy
import math

import numpy as np
import pytest
import torch

from oracle import oracle_c51 as oc
from oracle import oracle_discrete_sac as ods
from offpolicy_testutil import (B_LARGE, B_SMALL, DEV, EPS, GEMM_BK, Discrete, assert_spill_free, capture_batches, capture_grads,
                                check_final_state, check_second_batch_size, gemm_splits_k, grid_caps, ptxas_report, sm_count,
                                stream, vector_buffer_from_golden)
from test_qrdqn_gpu import make_buffer
from ts_testutil import load_golden, record_parity

gpu = pytest.mark.gpu
A_CASES = (1, 2, 6, 18)
N_CASES = (2, 51, 201)
VARIANTS = ["c51_ref_mlp", "c51_ref_cnn", "c51_ref_per"]


# ------------------------------------------------------------------------------------------------------------ target kernel
@gpu
@pytest.mark.parametrize("N", N_CASES)
@pytest.mark.parametrize("A", A_CASES)
def test_target_kernel_matches_oracle(A, N):
    """The action exactly, the distribution within fp32 rounding.  Integer-valued logits make two equal action blocks compute
    equal expected values, so they are exact ties and the first action must win; on every other row the action must be the
    float64 arg-max wherever the two best expected values are further apart than fp32 can blur.  B runs past the
    one-warp-per-row grid (16 blocks of 8 warps per SM) in one case; ``logits_next == logits_online`` is the
    ``target_update_freq == 0`` case."""
    from tianshou_b200._cabi import call, ptr
    g = torch.Generator().manual_seed(A * 1000 + N)
    B = sm_count() * 16 * 8 + 37 if (A, N) == (6, 51) else 301
    lo = torch.randint(-3, 4, (B, A, N), generator=g).float()
    ln = torch.randn(B, A, N, generator=g) * 2
    if A > 1:
        lo[: B // 3, A - 1] = lo[: B // 3, 0]                        # two equal blocks: the first wins where they lead
    z32 = oc.support(N, -10.0, 10.0)
    z = torch.as_tensor(z32, device=DEV)
    out, act = torch.empty(B, N, device=DEV), torch.empty(B, dtype=torch.int64, device=DEV)
    lod, lnd = lo.to(DEV), ln.to(DEV)
    q64 = (oc.softmax(lo.numpy()) * z32.astype(np.float64)).sum(2)
    ref_a = q64.argmax(1)
    top2 = np.sort(q64, 1)[:, -2:] if A > 1 else np.zeros((B, 2))
    clear = (top2[:, 1] - top2[:, 0]) > 1e-4 * 10.0 if A > 1 else np.ones(B, bool)
    for nxt, src in ((lnd, ln), (lod, lo)):
        call("ts_c51_target", ptr(lod), ptr(nxt), ptr(z), B, A, N, ptr(out), ptr(act), stream())
        torch.cuda.synchronize()
        got_a = act.cpu().numpy()
        assert np.array_equal(got_a[clear], ref_a[clear])
        if A > 1:
            tie = got_a[: B // 3]
            assert not np.any(tie == A - 1) and np.any(tie == 0), "the first of two equal blocks must win"
        want = oc.softmax(src.numpy()[np.arange(B), got_a])
        bound = (N / 32 + 8 + 2 * 2 * float(src.abs().max())) * EPS * want + 1e-30
        assert np.all(np.abs(out.cpu().numpy() - want) <= bound)
    call("ts_c51_target", ptr(lod), ptr(lod), ptr(z), 0, A, N, ptr(out), None, stream())      # B == 0: nothing to do
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------------ rows kernel
def _rows(logits, act, ret, z, v_min, v_max, dz, nd, w):
    from tianshou_b200._cabi import call, ptr
    B, A, N = logits.shape
    dl, prio = torch.empty(B, A, N, device=DEV), torch.empty(B, device=DEV)
    rows, losses = torch.empty(3, B, device=DEV), torch.empty(4, device=DEV)
    call("ts_c51_rows", ptr(logits), ptr(act), ptr(ret), ptr(z), v_min, v_max, dz, ptr(nd), ptr(w), B, A, N, ptr(dl), ptr(prio),
         ptr(rows), ptr(losses), stream())
    torch.cuda.synchronize()
    return losses.cpu().numpy(), dl.cpu().numpy(), prio.cpu().numpy()


@gpu
@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("N", N_CASES)
@pytest.mark.parametrize("A", A_CASES)
def test_rows_kernel_vs_fp64(A, N, weighted):
    """Loss, priorities and d loss / d logits against the float64 restatement (pinned to autograd of the reference's expression
    in test_oracle_c51), with returns exactly on an atom, exactly delta_z from one, and clamped at both ends.

    Error model (fp32, eps = 2^-23; the float64 side runs on the same fp32 inputs):
      - a projection weight clamp(1 - |t_k - z_j| / delta_z, 0, 1) is three roundings plus delta_z's own: 5 eps absolute;
        target_j sums N of them times next_dist_k in order: (N + 6) eps times sum_k next_dist_k.
      - p = softmax: x - max carries eps |x| + eps |max|, exp two more, the sum (N / 128 + 12) eps:
        rel_p = (N / 128 + 14 + 2 max|x|) eps.
      - CE_b: each term's target error times |log(p_j + 1e-8)|, plus target_j rel_p (d log(p + c) <= dp / p), plus the in-order
        and block sum, (N + 12) eps times sum_j target_j |log(p_j + 1e-8)|.
      - pg_j = -(w / B) target_j p_j / (p_j + 1e-8) is off by (w / B) (err_target_j + target_j (rel_p + 4 eps)); their sum S by
        the sum of those plus (N + 12) eps sum |pg|; dlogits_k = pg_k - p_k S adds p_k (err_S + |S| (rel_p + 2 eps)) and one
        rounding.
      - the loss averages w_b CE_b in row_sums3_kernel: (B / 1024 + 12) eps times the mean, on top of the rows' errors."""
    rng = np.random.default_rng(A * 7919 + N * 31 + weighted)
    B = sm_count() * 8 + 37 if (A, N, weighted) == (6, 51, True) else 41
    v_min, v_max = (-3.0, 7.0) if N % 2 else (-10.0, 10.0)
    z32 = oc.support(N, v_min, v_max)
    dz = (v_max - v_min) / (N - 1)
    logits = (rng.standard_normal((B, A, N)) * 2).astype(np.float32)
    act = rng.integers(0, A, B)
    ret = rng.uniform(v_min - 4, v_max + 4, (B, N)).astype(np.float32)
    ret[0, 0] = z32[N // 2]                                                       # on an atom
    ret[0, 1] = np.float32(z32[0] + np.float32(dz))                              # delta_z from atom 0
    ret[1, 0], ret[1, 1] = v_max + 5.0, v_min - 5.0                               # clamped at both ends
    nd = oc.softmax(rng.standard_normal((B, N)) * 2).astype(np.float32)
    w = rng.uniform(0.2, 1.0, B).astype(np.float32) if weighted else None
    dev = lambda a, dt=torch.float32: torch.as_tensor(a, dtype=dt, device=DEV)
    args = (dev(logits), dev(act, torch.int64), dev(ret), dev(z32), v_min, v_max, dz, dev(nd), None if w is None else dev(w))
    losses, dl, prio = _rows(*args)
    l64, ret64, z64, nd64 = (x.astype(np.float64) for x in (logits, ret, z32, nd))
    wb = np.ones(B) if w is None else w.astype(np.float64)
    r = oc.c51_rows(l64, act, ret64, z64, v_min, v_max, dz, nd64, None if w is None else wb)
    tg = r["target"]
    p = oc.softmax(l64[np.arange(B), act])
    L = np.abs(np.log(p + 1e-8))
    err_tg = (N + 6) * EPS * nd64.sum(1, keepdims=True)                          # [B, 1]
    rel_p = (N / 128 + 14 + 2 * np.abs(l64).max()) * EPS
    err_ce = 2 * ((err_tg * L).sum(1) + rel_p * tg.sum(1) + (N + 12) * EPS * (tg * L).sum(1))
    tag = f"c51_rows/A{A}_N{N}_w{int(weighted)}"
    assert np.all(np.abs(prio - r["prio"]) <= err_ce + 1e-30), f"{tag}: priorities off"
    record_parity(f"{tag}/prio", prio, r["prio"], rtol=0.0, atol=float(err_ce.max()) + 1e-30)
    bound_l = (wb * err_ce).mean() + (math.ceil(B / 1024) + 12) * EPS * (wb * r["ce"]).mean()
    want_l = np.array([r["loss"], r["loss"], r["ce"].mean(), 0.0])
    bound_ce_mean = err_ce.mean() + (math.ceil(B / 1024) + 12) * EPS * r["ce"].mean()
    err = np.abs(losses - want_l)
    assert err[0] <= bound_l and err[1] <= bound_l and err[2] <= bound_ce_mean and losses[3] == 0.0, f"{tag}: losses off by {err}"
    record_parity(f"{tag}/losses", losses, want_l, rtol=0.0, atol=float(max(bound_l, bound_ce_mean)))
    s = wb / B
    rr = p / (p + 1e-8)
    pg = -(s[:, None]) * tg * rr
    err_pg = s[:, None] * (err_tg * rr + tg * rr * (rel_p + 4 * EPS))
    S = pg.sum(1, keepdims=True)
    err_S = err_pg.sum(1, keepdims=True) + (N + 12) * EPS * np.abs(pg).sum(1, keepdims=True)
    bound_blk = 2 * (err_pg + p * (err_S + np.abs(S) * (rel_p + 2 * EPS))) + EPS * np.abs(pg - p * S) + 1e-30
    bound = np.zeros((B, A, N)) + 1e-30
    bound[np.arange(B), act, :] = bound_blk
    e = np.abs(dl - r["dlogits"])
    assert np.all(e <= bound), f"{tag}: dlogits error {float((e - bound).max()):.3e} past its bound"
    record_parity(f"{tag}/dlogits", dl, r["dlogits"], rtol=0.0, atol=float(bound.max()))
    again = _rows(*args)
    assert all(np.array_equal(a, b) for a, b in zip((losses, dl, prio), again)), "two calls must be bit-identical"


@gpu
def test_kernels_refuse_bad_arguments():
    from tianshou_b200._cabi import call, ptr
    x = torch.zeros(16, device=DEV)
    a = torch.zeros(1, dtype=torch.int64, device=DEV)

    def rows(N=4, dz=1.0, logits=x, v_min=-1.0, v_max=1.0):
        call("ts_c51_rows", ptr(logits), ptr(a), ptr(x), ptr(x), v_min, v_max, dz, ptr(x), None, 1, 1, N, ptr(x), ptr(x), ptr(x),
             ptr(x), stream())

    for kw in (dict(N=3073), dict(N=1), dict(dz=0.0), dict(dz=-1.0), dict(dz=float("nan")), dict(logits=None), dict(v_min=2.0)):
        with pytest.raises(RuntimeError, match="ts_c51_rows"):
            rows(**kw)
    for N, lo in ((1, x), (4, None)):
        with pytest.raises(RuntimeError, match="ts_c51_target"):
            call("ts_c51_target", ptr(lo), ptr(x), ptr(x), 1, 1, N, ptr(x), None, stream())


# ------------------------------------------------------------------------------------------------------------ vs reference
def model_from_cfg(kind, A, N, obs=4, hidden=(64,), H=44, W=44, scale=True):
    from tianshou_b200.env.atari import C51Net, ScaledObsInputActionReprNet
    from tianshou_b200.utils.net.common import Net
    if kind == "cnn":
        net = C51Net(c=4, h=H, w=W, action_shape=A, num_atoms=N)
        return (ScaledObsInputActionReprNet(net) if scale else net).to(DEV)
    return Net(state_shape=(obs,), action_shape=A, hidden_sizes=hidden, softmax=True, num_atoms=N).to(DEV)


def build_from_golden(g):
    from tianshou_b200.algorithm import AdamOptimizerFactory, C51, C51Policy
    kind = str(g["cfg_kind"])
    kw = (dict(H=int(g["cfg_H"]), W=int(g["cfg_W"]), scale=bool(g["cfg_scale"])) if kind == "cnn"
          else dict(obs=int(g["cfg_obs"]), hidden=tuple(int(x) for x in g["cfg_hidden"])))
    A, N = int(g["cfg_A"]), int(g["cfg_N"])
    model = model_from_cfg(kind, A, N, **kw)
    ods.seeded_params(model, int(g["cfg_init_seed"]))
    policy = C51Policy(model=model, action_space=Discrete(A), num_atoms=N, v_min=float(g["cfg_v_min"]), v_max=float(g["cfg_v_max"]))
    return C51(policy=policy, optim=AdamOptimizerFactory(lr=float(g["cfg_lr"])), gamma=float(g["cfg_gamma"]),
               n_step_return_horizon=int(g["cfg_n_step"]), target_update_freq=int(g["cfg_freq"]))


def _optimizer_layout(algo):
    osd = algo.state_dict()["_optimizers"][0]
    return list(osd["param_groups"][0]["params"]), sorted(osd["state"].keys())


@gpu
@pytest.mark.parametrize("mirror", [False, True])
@pytest.mark.parametrize("variant", VARIANTS)
def test_update_matches_reference(variant, mirror):
    """Update after update against the reference's run: the same sampled indices, n-step returns over the N atoms, loss, the
    priorities written back (PER: and the sum-tree leaves), then the final state, the ``state_dict()`` keys and the
    optimiser's param indices (``support`` at 0, without state)."""
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden(f"{variant}.npz")
    algo, buf = build_from_golden(g), vector_buffer_from_golden(g, mirror)
    keys = [str(k) for k in g["state_dict_keys"]]
    assert list(algo.state_dict().keys()) == keys
    with capture_batches(algo) as cap:
        for u in range(int(g["cfg_updates"])):
            np.random.seed(500 + u)
            with policy_within_training_step(algo.policy):
                stats = algo.update(buffer=buf, sample_size=int(g["cfg_bs"]))
            tag = f"{variant}_m{int(mirror)}_u{u}"
            assert np.array_equal(cap["indices"], g[f"u{u}_indices"]), "sampled indices differ from the reference's"
            ref_ret = g[f"u{u}_returns"]
            record_parity(f"{tag}/returns", cap["returns"].cpu().numpy(), ref_ret, rtol=1e-5, atol=1e-5 * float(np.abs(ref_ret).max()))
            assert isinstance(stats.loss, float)
            record_parity(f"{tag}/losses", np.array([stats.loss]), g[f"u{u}_losses"], rtol=2e-5, atol=2e-6)
            record_parity(f"{tag}/prio", cap["prio"].cpu().numpy(), g[f"u{u}_prio"], rtol=2e-5, atol=2e-6)
            if bool(g["cfg_per"]):
                leaves = np.asarray(buf.weight[np.arange(len(buf))])
                record_parity(f"{tag}/tree_leaves", leaves, g[f"u{u}_tree_leaves"], rtol=2e-5, atol=1e-7)
    check_final_state(f"{variant}_m{int(mirror)}", g, algo)
    assert list(algo.state_dict().keys()) == keys
    ids, state_ids = _optimizer_layout(algo)
    assert ids == [int(i) for i in g["opt_param_ids"]] and state_ids == [int(i) for i in g["opt_state_ids"]]
    assert algo.optim._optim.param_groups[0]["params"][0] is algo.policy.support


def grad_case(kind, B=64, edge=""):
    """One update at batch ``B``: the flat gradient, snapshotted before its Adam step, against float64 autograd of the
    reference's loss (c51.py:113-154) through the module's own softmax, on a copy of the module with the same weights, batch
    and returns.  The lagged copy is refreshed by this first update, so the target comes from the same weights.  The GEMMs are
    fp32-faithful (bf16x3) and a weight gradient sums B products per element: 2e-4 relative plus 1e-4 of the tensor's largest
    value, as in test_qrdqn_gpu."""
    from tianshou_b200.algorithm import AdamOptimizerFactory, C51, C51Policy
    from tianshou_b200.utils import policy_within_training_step
    torch.manual_seed(3)
    rng = np.random.default_rng(4)
    A, N, v_min, v_max = 5, 33, -4.0, 6.0
    model = model_from_cfg(kind, A, N, hidden=(48, 40))
    policy = C51Policy(model=model, action_space=Discrete(A), num_atoms=N, v_min=v_min, v_max=v_max)
    algo = C51(policy=policy, optim=AdamOptimizerFactory(lr=1e-3), gamma=0.9, n_step_return_horizon=2, target_update_freq=3)
    buf = make_buffer(kind, A, rng)
    grp = algo._group
    ref = copy.deepcopy(model).to("cpu", torch.float64)         # the weights before the step
    np.random.seed(7)
    with capture_batches(algo) as cap, capture_grads(grp) as grads, policy_within_training_step(algo.policy):
        stats = algo.update(buffer=buf, sample_size=B)
    idx, returns = cap["indices"], cap["returns"].cpu().double()
    obs = np.asarray(buf.obs)
    obs_next = obs[buf.next(idx)] if kind == "cnn" else np.asarray(buf.obs_next)[idx]
    x_of = lambda raw: torch.as_tensor((raw.astype(np.float64) / 255.0).astype(np.float32) if kind == "cnn" else raw).double()
    inner = ref.module if kind == "cnn" else ref
    chain = inner.net if kind == "cnn" else inner.model.model
    probs = lambda x: chain(x).view(len(x), A, N).softmax(-1)
    z = torch.as_tensor(oc.support(N, v_min, v_max), dtype=torch.float64)
    with torch.no_grad():
        pn = probs(x_of(obs_next))
        nd = pn[torch.arange(B), (pn * z).sum(2).argmax(1)]
        target = oc.reference_target(nd, returns, z, v_min, v_max, (v_max - v_min) / (N - 1))
    act = np.asarray(buf.act)[idx].astype(np.int64)
    loss, _ = oc.reference_loss(probs(x_of(obs[idx])), act, target, 1.0)
    loss.backward()
    ref_params = [p for m in chain.modules() if isinstance(m, (torch.nn.Linear, torch.nn.Conv2d)) for p in (m.weight, m.bias)]
    for i, (p, r) in enumerate(zip(grp.params, ref_params, strict=True)):
        want = r.grad.numpy()
        got = grp.view(grads[-1], p).view(p.shape).cpu().numpy()
        record_parity(f"c51_grad{edge}/{kind}/grad_{i}", got, want, rtol=2e-4, atol=1e-4 * float(np.abs(want).max()) + 1e-12)
    record_parity(f"c51_grad{edge}/{kind}/loss", np.array([stats.loss]), np.array([loss.item()]), rtol=2e-5, atol=2e-6)
    assert len(idx) == B and returns.shape[0] == B, "the update must run on the B sampled rows"


@gpu
@pytest.mark.parametrize("kind", ["mlp", "cnn"])
def test_update_gradient_vs_fp64_autograd(kind):
    grad_case(kind)


def _edge_batch(cls):
    if cls == "B1":
        return 1
    if cls in ("splitK_below", "splitK_above"):
        return GEMM_BK + (cls == "splitK_above")
    caps = grid_caps()                  # past both the target's warp-per-row and the rows kernel's block-per-row grid
    return max(caps["warp_per_row"], caps["block_per_row"]) + 1


@gpu
@pytest.mark.parametrize("cls", ["B1", "splitK_below", "splitK_above", "past_grid"])
def test_update_vs_fp64_autograd_at_batch_edges(cls):
    """The batch sizes of test_offpolicy_batch_edges_gpu applied to C51: B = 1, the largest weight-gradient GEMM at one and at
    two K chunks (unsplit / split K), and the smallest batch past the grid caps of both new kernels."""
    B = _edge_batch(cls)
    if cls.startswith("splitK"):
        assert gemm_splits_k(B) == (cls == "splitK_above")
    if cls == "past_grid":
        caps = grid_caps()
        assert B > caps["warp_per_row"] and B > caps["block_per_row"]
    grad_case("mlp", B=B, edge=f"@{cls}")


@gpu
@pytest.mark.parametrize("order", ["large_then_small", "small_then_large"])
def test_second_batch_size_is_bit_identical_to_a_fresh_instance(order):
    """As test_offpolicy_batch_edges_gpu part 2: one batch size, every scratch tensor poisoned with NaN, then another; the
    second update must equal a fresh instance's, loaded from the same ``state_dict()``, bit for bit."""
    g = load_golden("c51_ref_mlp.npz")
    B1, B2 = (B_LARGE, B_SMALL) if order == "large_then_small" else (B_SMALL, B_LARGE)
    cap, _ = check_second_batch_size(lambda: build_from_golden(g), vector_buffer_from_golden(g, False), B1, B2)
    assert cap["prio"] is not None


# ------------------------------------------------------------------------------------------------------------ state_dict
@gpu
@pytest.mark.parametrize("variant", ["c51_ref_mlp", "c51_ref_cnn"])
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
        for p in b.policy.model.parameters():
            p.add_(0.01)
    b.load_state_dict(copy.deepcopy(a.state_dict()))
    b._iter = a._iter
    assert torch.equal(a.policy.support, b.policy.support)
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
def test_policy_forward_takes_arg_max_of_expected_values():
    from tianshou_b200.algorithm import C51Policy
    from tianshou_b200.data import Batch
    torch.manual_seed(0)
    model = model_from_cfg("mlp", 5, 17, obs=4, hidden=(32,))
    policy = C51Policy(model=model, action_space=Discrete(5), num_atoms=17, v_min=-2.0, v_max=3.0)
    assert policy.support.device == torch.device(DEV)
    rng = np.random.default_rng(0)
    obs = rng.standard_normal((300, 4)).astype(np.float32)
    probs, _ = model(obs)
    q = (probs * policy.support).sum(2)
    out = policy(Batch(obs=obs, info=Batch()))
    assert out.logits.shape == (300, 5, 17) and torch.equal(out.logits, probs)
    assert np.array_equal(out.act, q.argmax(1).cpu().numpy())
    mask = rng.random((300, 5)) < 0.6
    mask[:, 2] = True
    out = policy(Batch(obs=Batch(obs=obs, mask=mask), info=Batch()))
    masked = q + torch.as_tensor(1 - mask.astype(np.float32), device=DEV) * (q.min() - q.max() - 1.0)
    assert np.array_equal(out.act, masked.argmax(1).cpu().numpy()) and mask[np.arange(300), out.act].all()


# ------------------------------------------------------------------------------------------------------------ refusals
@gpu
def test_refusals():
    from tianshou_b200.algorithm import AdamOptimizerFactory, C51, C51Policy, RMSpropOptimizerFactory, UnsupportedModelError
    from tianshou_b200.data import Batch, VectorReplayBuffer
    from tianshou_b200.env.atari import DQNet, QRDQNet
    from tianshou_b200.utils import policy_within_training_step
    from tianshou_b200.utils.net.common import Net
    A, N = 3, 8

    def make(model=None, opt=AdamOptimizerFactory, n=A, **kw):
        model = model or model_from_cfg("mlp", A, N, hidden=(16,))
        return C51(policy=C51Policy(model=model, action_space=Discrete(n), num_atoms=N), optim=opt(lr=1e-3), **kw)

    algo = make()
    for model in (Net(state_shape=(4,), action_shape=A, hidden_sizes=(16,), num_atoms=N),
                  DQNet(4, 44, 44, A * N), QRDQNet(c=4, h=44, w=44, action_shape=A, num_quantiles=N),
                  Net(state_shape=(4,), action_shape=A * N, hidden_sizes=(16,), softmax=True)):
        with pytest.raises(UnsupportedModelError, match="softmax"):
            make(model.to(DEV))
    with pytest.raises(UnsupportedModelError, match="outputs, not 3 actions x 8 atoms"):
        make(model_from_cfg("mlp", A, N + 1, hidden=(16,)))
    with pytest.raises(UnsupportedModelError, match="outputs, not 4 actions"):
        make(n=4)
    with pytest.raises(UnsupportedModelError, match="Adam"):
        make(opt=RMSpropOptimizerFactory)
    with pytest.raises(UnsupportedModelError, match="no CPU path"):
        make(model_from_cfg("mlp", A, N, hidden=(16,)).cpu())
    for kw in (dict(gamma=1.5), dict(gamma=-0.1), dict(n_step_return_horizon=0)):
        with pytest.raises(AssertionError):
            make(**kw)
    for kw in (dict(num_atoms=1), dict(v_min=1.0, v_max=1.0), dict(v_min=2.0, v_max=1.0)):
        with pytest.raises(AssertionError):
            C51Policy(model=model_from_cfg("mlp", A, N, hidden=(16,)), action_space=Discrete(A), **kw)
    # an action the network has no atoms for is refused on the host, before any kernel indexes with it
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
    report = ptxas_report("c51.cu", tmp_path)
    kernels = ("c51_rows_kernel", "c51_target_kernel", "row_sums3_kernel")
    assert len(report) == 3 and all(any(k in e for k in kernels) for e in report), report
    assert_spill_free(report)
