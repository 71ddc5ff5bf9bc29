"""Rainbow DQN on the GPU: the noisy-layer and dueling kernels against torch and float64, ``RainbowDQN.update()`` against
outputs of the imported reference (tests/golden/rainbow_ref_*.npz from oracle/gen_golden_rainbow.py, the reference's noise
injected through the ``_sample_noise`` seam), one update's gradient against float64 autograd through noisy layers and dueling
heads, the noise draws against the eager update's, the batch sizes the kernels and GEMMs split on, the ``state_dict()`` round
trip, the policy's torch path, the refusals, the reference's algorithm constructions and the kernels' register report."""
import copy

import numpy as np
import pytest
import torch
from torch import nn

from oracle import oracle_c51 as oc
from oracle import oracle_discrete_sac as ods
from oracle import oracle_rainbow as orb
from offpolicy_testutil import (B_LARGE, B_SMALL, DEV, EPS, GEMM_BK, Discrete, assert_spill_free, capture_batches, capture_grads,
                                check_final_state, check_second_batch_size, gemm_splits_k, grid_caps, ptxas_report, sm_count,
                                stream, vector_buffer_from_golden)
from test_qrdqn_gpu import make_buffer
from ts_testutil import load_golden, record_parity

gpu = pytest.mark.gpu
A_CASES = (1, 2, 6, 18)
N_CASES = (2, 51, 201)
VARIANTS = ["rainbow_ref_mlp", "rainbow_ref_cnn", "rainbow_ref_per", "rainbow_ref_nonoisy", "rainbow_ref_nodueling"]


# ------------------------------------------------------------------------------------------------------------ noisy kernels
@gpu
@pytest.mark.parametrize("out,inp", [(1, 1), (5, 7), (512, 256), (306, 512), (33, 3136)])
def test_noisy_weight_kernel_is_bit_identical_to_torch(out, inp):
    """torch's train-mode expression, ger then * then +, on the same device tensors."""
    from tianshou_b200._cabi import call, ptr
    g = torch.Generator(device=DEV).manual_seed(out * 31 + inp)
    mu_w, sg_w = torch.randn(out, inp, device=DEV, generator=g), torch.randn(out, inp, device=DEV, generator=g)
    mu_b, sg_b = torch.randn(out, device=DEV, generator=g), torch.randn(out, device=DEV, generator=g)
    ep, eq = torch.randn(inp, device=DEV, generator=g), torch.randn(out, device=DEV, generator=g)
    w, b = torch.empty(out, inp, device=DEV), torch.empty(out, device=DEV)
    call("ts_noisy_weight", ptr(mu_w), ptr(sg_w), ptr(mu_b), ptr(sg_b), ptr(ep), ptr(eq), out, inp, ptr(w), ptr(b), stream())
    torch.cuda.synchronize()
    assert torch.equal(w, mu_w + sg_w * eq.ger(ep)) and torch.equal(b, mu_b + sg_b * eq.clone())


@gpu
@pytest.mark.parametrize("out,inp", [(1, 1), (5, 7), (512, 256), (33, 3136)])
def test_noisy_grad_kernel_matches_torch_expressions(out, inp):
    """Given the same gradient at the effective weight and bias, autograd's gradients of the four trainable tensors exactly."""
    from tianshou_b200._cabi import call, ptr
    g = torch.Generator(device=DEV).manual_seed(out * 7 + inp)
    dw, db = torch.randn(out, inp, device=DEV, generator=g), torch.randn(out, device=DEV, generator=g)
    ep, eq = torch.randn(inp, device=DEV, generator=g), torch.randn(out, device=DEV, generator=g)
    mu_w, sg_w = torch.zeros(out, inp, device=DEV, requires_grad=True), torch.ones(out, inp, device=DEV, requires_grad=True)
    mu_b, sg_b = torch.zeros(out, device=DEV, requires_grad=True), torch.ones(out, device=DEV, requires_grad=True)
    torch.autograd.backward([mu_w + sg_w * eq.ger(ep), mu_b + sg_b * eq.clone()], [dw, db])
    got = [torch.full_like(t, float("nan")) for t in (dw, dw, db, db)]
    call("ts_noisy_grad", ptr(dw), ptr(db), ptr(ep), ptr(eq), out, inp, *(ptr(t) for t in got), stream())
    torch.cuda.synchronize()
    for t, want in zip(got, (mu_w.grad, sg_w.grad, mu_b.grad, sg_b.grad)):
        assert torch.equal(t, want)


# ------------------------------------------------------------------------------------------------------------ dueling kernels
@gpu
@pytest.mark.parametrize("N", N_CASES)
@pytest.mark.parametrize("A", A_CASES)
def test_dueling_kernels_vs_fp64(A, N):
    """Forward and backward against float64 on the same fp32 inputs.  Error model (eps = 2^-23): the mean sums A values in order
    ((A - 1) eps sum_a |q|) and divides (one rounding), q - m and + v round once each: |logits - ref| <= (A + 3) eps (mean_a |q| +
    |q| + |m| + |v|).  dv sums A values in order: (A - 1) eps sum_a |dl|; dq = dl - s / A adds two roundings:
    (A + 2) eps (sum_a |dl| / A + |dl|).  B runs past the kernels' grid cap (8 blocks of 256 threads per SM) in one case."""
    from tianshou_b200._cabi import call, ptr
    rng = np.random.default_rng(A * 1000 + N)
    B = sm_count() * 8 * 256 // N + 29 if (A, N) == (6, 201) else 37
    q = (rng.standard_normal((B, A, N)) * 3).astype(np.float32)
    v = (rng.standard_normal((B, N)) * 3).astype(np.float32)
    dl = rng.standard_normal((B, A, N)).astype(np.float32)
    qd, vd, dld = (torch.as_tensor(a, device=DEV) for a in (q, v, dl))
    logits, dq, dv = torch.empty(B, A, N, device=DEV), torch.empty(B, A, N, device=DEV), torch.empty(B, N, device=DEV)
    call("ts_dueling_atoms", ptr(qd), ptr(vd), B, A, N, ptr(logits), stream())
    call("ts_dueling_atoms_bwd", ptr(dld), B, A, N, ptr(dq), ptr(dv), stream())
    torch.cuda.synchronize()
    q64, v64 = q.astype(np.float64), v.astype(np.float64)
    m = q64.mean(1, keepdims=True)
    want = orb.dueling(q64, v64)
    bound = (A + 3) * EPS * (np.abs(q64).mean(1, keepdims=True) + np.abs(q64) + np.abs(m) + np.abs(v64)[:, None, :])
    got = logits.cpu().numpy()
    assert np.all(np.abs(got - want) <= bound)
    record_parity(f"rainbow_dueling/A{A}_N{N}/logits", got, want, rtol=0.0, atol=float(bound.max()))
    want_dq, want_dv = orb.dueling_bwd(dl)
    s = np.abs(dl.astype(np.float64)).sum(1)
    assert np.all(np.abs(dv.cpu().numpy() - want_dv) <= max(A - 1, 0) * EPS * s + 1e-30)
    assert np.all(np.abs(dq.cpu().numpy() - want_dq) <= (A + 2) * EPS * (s[:, None, :] / A + np.abs(dl)) + 1e-30)
    again = torch.empty_like(dq)
    call("ts_dueling_atoms_bwd", ptr(dld), B, A, N, ptr(again), ptr(dv), stream())
    torch.cuda.synchronize()
    assert torch.equal(again, dq), "two calls must be bit-identical"


@gpu
def test_kernels_refuse_bad_arguments():
    from tianshou_b200._cabi import call, ptr
    x = torch.zeros(16, device=DEV)
    for args in ((None, 2, 2), (ptr(x), 0, 2), (ptr(x), 2, 0)):
        with pytest.raises(RuntimeError, match="ts_noisy_weight"):
            call("ts_noisy_weight", args[0], ptr(x), ptr(x), ptr(x), ptr(x), ptr(x), args[1], args[2], ptr(x), ptr(x), stream())
        with pytest.raises(RuntimeError, match="ts_noisy_grad"):
            call("ts_noisy_grad", args[0], ptr(x), ptr(x), ptr(x), args[1], args[2], ptr(x), ptr(x), ptr(x), ptr(x), stream())
    for args in ((None, 1, 2, 2), (ptr(x), -1, 2, 2), (ptr(x), 1, 0, 2), (ptr(x), 1, 2, 0)):
        with pytest.raises(RuntimeError, match="ts_dueling_atoms"):
            call("ts_dueling_atoms", args[0], ptr(x), args[1], args[2], args[3], ptr(x), stream())
        with pytest.raises(RuntimeError, match="ts_dueling_atoms_bwd"):
            call("ts_dueling_atoms_bwd", args[0], args[1], args[2], args[3], ptr(x), ptr(x), stream())
    call("ts_dueling_atoms", ptr(x), ptr(x), 0, 2, 2, ptr(x), stream())          # B == 0: nothing to do
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------------ vs reference
def model_from_cfg(cfg):
    """Our network of a golden's configuration (the keys of ``oracle_rainbow.rainbow_net``), on the device."""
    from tianshou_b200.env.atari import RainbowNet, ScaledObsInputActionReprNet
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.discrete import NoisyLinear
    A, N = int(cfg["A"]), int(cfg["N"])
    std = float(cfg.get("noisy_std", 0.5))
    if str(cfg["kind"]) == "cnn":
        net = RainbowNet(c=4, h=int(cfg["H"]), w=int(cfg["W"]), action_shape=A, num_atoms=N, noisy_std=std,
                         is_dueling=bool(cfg["dueling"]), is_noisy=bool(cfg["noisy"]))
        return (ScaledObsInputActionReprNet(net) if bool(cfg.get("scale", True)) else net).to(DEV)

    def noisy(x, y):
        return NoisyLinear(x, y, std)

    return Net(state_shape=(int(cfg["obs"]),), action_shape=A, hidden_sizes=[int(h) for h in cfg["hidden"]], softmax=True,
               num_atoms=N, linear_layer=noisy if bool(cfg["trunk_noisy"]) else nn.Linear,
               dueling_param=({"hidden_sizes": [int(h) for h in cfg["q_hidden"]], "linear_layer": noisy},
                              {"hidden_sizes": [int(h) for h in cfg["v_hidden"]],
                               "linear_layer": noisy if bool(cfg["v_noisy"]) else nn.Linear})).to(DEV)


def _cfg(g):
    return {k[4:]: g[k] for k in g.files if k.startswith("cfg_")}


def build_from_golden(g):
    from tianshou_b200.algorithm import AdamOptimizerFactory, C51Policy, RainbowDQN
    A, N = int(g["cfg_A"]), int(g["cfg_N"])
    model = model_from_cfg(_cfg(g))
    ods.seeded_params(model, int(g["cfg_init_seed"]))
    policy = C51Policy(model=model, action_space=Discrete(A), num_atoms=N, v_min=float(g["cfg_v_min"]), v_max=float(g["cfg_v_max"]))
    return RainbowDQN(policy=policy, optim=AdamOptimizerFactory(lr=float(g["cfg_lr"])), gamma=float(g["cfg_gamma"]),
                      n_step_return_horizon=int(g["cfg_n_step"]), target_update_freq=int(g["cfg_freq"]))


def inject_noise(algo, g, u):
    """Replace the noise draw by the reference's draws of update ``u``."""
    def sample(model):
        orb.set_noise(model, g[f"u{u}_noise_on"] if model is algo.policy.model else g[f"u{u}_noise_old"])
        return len(orb.noise_tensors(model)) > 0
    algo._sample_noise = sample


def _optimizer_layout(algo):
    osd = algo.state_dict()["_optimizers"][0]
    return list(osd["param_groups"][0]["params"]), sorted(osd["state"].keys())


@gpu
@pytest.mark.parametrize("mirror", [False, True])
@pytest.mark.parametrize("variant", VARIANTS)
def test_update_matches_reference(variant, mirror):
    """Update after update against the reference's run, with its noise: the sampled indices, n-step returns, loss, priorities
    (PER: the sum-tree leaves), both networks' noise after the update (on a tick the lagged network holds the online network's),
    then the final parameters, Adam moments and lagged parameters, ``_iter``, the ``state_dict()`` keys (``model_old.*``
    unwrapped) and the optimiser's param indices (``support`` and the noise listed, without state)."""
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden(f"{variant}.npz")
    algo, buf = build_from_golden(g), vector_buffer_from_golden(g, mirror)
    keys = [str(k) for k in g["state_dict_keys"]]
    assert list(algo.state_dict().keys()) == keys
    freq = int(g["cfg_freq"])
    with capture_batches(algo) as cap:
        for u in range(int(g["cfg_updates"])):
            inject_noise(algo, g, u)
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
            assert np.array_equal(orb.get_noise(algo.policy.model), g[f"u{u}_eps_on"])
            assert np.array_equal(algo._eps.flat.cpu().numpy(), g[f"u{u}_eps_on"])
            if freq > 0:
                assert np.array_equal(orb.get_noise(algo.model_old), g[f"u{u}_eps_old"])
                assert np.array_equal(algo._eps_old.flat.cpu().numpy(), g[f"u{u}_eps_old"])
    check_final_state(f"{variant}_m{int(mirror)}", g, algo, lagged=orb.trainable(algo.model_old) if freq > 0 else [])
    assert list(algo.state_dict().keys()) == keys
    if freq > 0:        # the lagged network unwrapped: its keys are the online model's under model_old.
        assert [k for k in keys if k.startswith("model_old.")] == ["model_old." + k for k in algo.policy.model.state_dict()]
    ids, state_ids = _optimizer_layout(algo)
    assert ids == [int(i) for i in g["opt_param_ids"]] and state_ids == [int(i) for i in g["opt_state_ids"]]
    assert algo.optim._optim.param_groups[0]["params"][0] is algo.policy.support


GRAD_CFG = {"mlp": dict(kind="mlp", obs=4, hidden=(48, 40), q_hidden=(32,), v_hidden=(), trunk_noisy=True, v_noisy=True, A=5, N=33),
            "cnn": dict(kind="cnn", H=44, W=44, noisy=True, dueling=True, A=5, N=33)}


def grad_case(kind, B=64, edge=""):
    """One update at batch ``B``: the flat gradient, snapshotted before its Adam step, against float64 autograd of the
    reference's loss through the oracle network (train mode: the noise this update drew) with the same weights, batch and
    returns.  The lagged copy is refreshed by this first update, so the target comes from the same weights and noise.  The
    GEMMs are fp32-faithful (bf16x3) and a weight gradient sums B products per element: 2e-4 relative plus 1e-4 of the tensor's
    largest value, as in test_c51_gpu."""
    from tianshou_b200.algorithm import AdamOptimizerFactory, C51Policy, RainbowDQN
    from tianshou_b200.utils import policy_within_training_step
    torch.manual_seed(3)
    rng = np.random.default_rng(4)
    cfg = GRAD_CFG[kind]
    A, N, v_min, v_max = cfg["A"], cfg["N"], -4.0, 6.0
    model = model_from_cfg(cfg)
    policy = C51Policy(model=model, action_space=Discrete(A), num_atoms=N, v_min=v_min, v_max=v_max)
    algo = RainbowDQN(policy=policy, optim=AdamOptimizerFactory(lr=1e-3), gamma=0.9, n_step_return_horizon=2, target_update_freq=3)
    buf = make_buffer(kind, A, rng)
    grp = algo._group
    ref = orb.rainbow_net(cfg).double()
    with torch.no_grad():                                           # the weights before the step
        for r, p in zip(ref.parameters(), model.parameters(), strict=True):
            r.copy_(p)
    np.random.seed(7)
    with capture_batches(algo) as cap, capture_grads(grp) as grads, policy_within_training_step(algo.policy):
        stats = algo.update(buffer=buf, sample_size=B)
    orb.set_noise(ref, orb.get_noise(model))                        # the noise the update drew
    idx, returns = cap["indices"], cap["returns"].cpu().double()
    obs = np.asarray(buf.obs)
    obs_next = obs[buf.next(idx)] if kind == "cnn" else np.asarray(buf.obs_next)[idx]
    x_of = lambda raw: torch.as_tensor((raw.astype(np.float64) / 255.0).astype(np.float32) if kind == "cnn" else raw).double()
    z = torch.as_tensor(oc.support(N, v_min, v_max), dtype=torch.float64)
    with torch.no_grad():
        pn = ref(x_of(obs_next))
        nd = pn[torch.arange(B), (pn * z).sum(2).argmax(1)]
        target = oc.reference_target(nd, returns, z, v_min, v_max, (v_max - v_min) / (N - 1))
    act = np.asarray(buf.act)[idx].astype(np.int64)
    loss, _ = oc.reference_loss(ref(x_of(obs[idx])), act, target, 1.0)
    loss.backward()
    for i, (p, r) in enumerate(zip(grp.params, orb.trainable(ref), strict=True)):
        want = r.grad.numpy()
        got = grp.view(grads[-1], p).view(p.shape).cpu().numpy()
        record_parity(f"rainbow_grad{edge}/{kind}/grad_{i}", got, want, rtol=2e-4, atol=1e-4 * float(np.abs(want).max()) + 1e-12)
    record_parity(f"rainbow_grad{edge}/{kind}/loss", np.array([stats.loss]), np.array([loss.item()]), rtol=2e-5, atol=2e-6)
    assert len(idx) == B and returns.shape[0] == B, "the update must run on the B sampled rows"


@gpu
@pytest.mark.parametrize("kind", ["mlp", "cnn"])
def test_update_gradient_vs_fp64_autograd(kind):
    """The noisy layers' forward and backward (effective weights, the gradient split, the input gradient through the effective
    weight) and the dueling combine, through a whole update."""
    grad_case(kind)


def _edge_batch(cls):
    if cls == "B1":
        return 1
    if cls in ("splitK_below", "splitK_above"):
        return GEMM_BK + (cls == "splitK_above")
    caps = grid_caps()
    return max(caps["warp_per_row"], caps["block_per_row"]) + 1


@gpu
@pytest.mark.parametrize("cls", ["B1", "splitK_below", "splitK_above", "past_grid"])
def test_update_vs_fp64_autograd_at_batch_edges(cls):
    """B = 1, the largest weight-gradient GEMM at one and at two K chunks, and the smallest batch past C51's kernels' grid caps."""
    B = _edge_batch(cls)
    if cls.startswith("splitK"):
        assert gemm_splits_k(B) == (cls == "splitK_above")
    grad_case("mlp", B=B, edge=f"@{cls}")


@gpu
@pytest.mark.parametrize("order", ["large_then_small", "small_then_large"])
def test_second_batch_size_is_bit_identical_to_a_fresh_instance(order):
    """One batch size, every scratch tensor poisoned with NaN, then another; the second update (the same torch seed, so the same
    noise) must equal a fresh instance's, loaded from the same ``state_dict()``, bit for bit."""
    g = load_golden("rainbow_ref_mlp.npz")
    B1, B2 = (B_LARGE, B_SMALL) if order == "large_then_small" else (B_SMALL, B_LARGE)
    cap, _ = check_second_batch_size(lambda: build_from_golden(g), vector_buffer_from_golden(g, False), B1, B2)
    assert cap["prio"] is not None


# ------------------------------------------------------------------------------------------------------------ RNG parity
@gpu
@pytest.mark.parametrize("variant", ["rainbow_ref_mlp", "rainbow_ref_per"])
def test_noise_draws_match_the_eager_update(variant):
    """Seeded identically, ``RainbowDQN.update()`` and the eager reference-expression update draw bit-identical noise for both
    networks, update after update, and their losses agree."""
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden(f"{variant}.npz")
    algo, buf = build_from_golden(g), vector_buffer_from_golden(g)
    net = orb.net_from_golden(g)
    ods.seeded_params(net, int(g["cfg_init_seed"]))
    net.to(DEV)
    s = orb.RainbowState(net, float(g["cfg_lr"]), int(g["cfg_freq"]), float(g["cfg_v_min"]), float(g["cfg_v_max"]))
    E, cap = int(g["cfg_E"]), int(g["cfg_cap"])
    bufd = dict(obs=g["buf_obs"], obs_next=g["buf_obs_next"], act=g["buf_act"], rew=g["buf_rew"], done=g["buf_done"],
                terminated=g["buf_terminated"], offset=np.arange(E + 1) * cap, last_index=g["meta_last_index"],
                lengths=g["meta_lengths"])
    obs_of = ods.flat_obs(bufd["obs"], DEV)
    U = int(g["cfg_updates"])
    ours, theirs = [], []
    torch.cuda.manual_seed(1234)
    with capture_batches(algo) as capt:
        for u in range(U):
            np.random.seed(500 + u)
            with policy_within_training_step(algo.policy):
                loss = algo.update(buffer=buf, sample_size=int(g["cfg_bs"])).loss
            ours.append((orb.get_noise(algo.policy.model), orb.get_noise(algo.model_old), loss, capt["indices"]))
    torch.cuda.manual_seed(1234)
    for u in range(U):
        loss = orb.rainbow_update_torch(s, obs_of, bufd, ours[u][3], float(g["cfg_gamma"]), int(g["cfg_n_step"]))
        theirs.append((orb.get_noise(s.net), orb.get_noise(s.old), loss))
    for u, (a, b) in enumerate(zip(ours, theirs)):
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]), f"update {u}: the noise draws differ"
        if not bool(g["cfg_per"]):
            record_parity(f"rainbow_rng/{variant}/u{u}/loss", np.array([a[2]]), np.array([b[2]]), rtol=1e-4, atol=1e-6)
    assert not np.array_equal(ours[0][0], ours[1][0])


# ------------------------------------------------------------------------------------------------------------ state_dict
@gpu
@pytest.mark.parametrize("variant", ["rainbow_ref_mlp", "rainbow_ref_cnn"])
def test_state_dict_round_trip_continues_identically(variant):
    """A fresh algorithm loaded from another's ``state_dict()`` continues bit for bit: online, lagged, noise and optimiser state
    (the same torch seed on both runs draws the same noise).  ``_iter`` is a plain attribute, as in the reference."""
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
    assert torch.equal(a._eps.flat, b._eps.flat) and torch.equal(a._eps_old.flat, b._eps_old.flat)
    for algo in (a, b):
        buf = vector_buffer_from_golden(g)
        torch.manual_seed(42)
        for u in range(3):
            np.random.seed(10 + u)
            with policy_within_training_step(algo.policy):
                algo.update(buffer=buf, sample_size=int(g["cfg_bs"]))
    for ga, gb in ((a._group, b._group), (a._g_old, b._g_old)):
        assert torch.equal(ga.flat, gb.flat) and torch.equal(ga.exp_avg, gb.exp_avg) and torch.equal(ga.exp_avg_sq, gb.exp_avg_sq)
    assert torch.equal(a._eps.flat, b._eps.flat) and torch.equal(a._eps_old.flat, b._eps_old.flat)
    assert a._group.step == b._group.step


# ------------------------------------------------------------------------------------------------------------ policy
@gpu
def test_policy_forward_is_noisy_in_train_mode_and_mu_in_eval():
    from tianshou_b200.algorithm import C51Policy
    from tianshou_b200.data import Batch
    torch.manual_seed(0)
    cfg = GRAD_CFG["mlp"]
    model = model_from_cfg(cfg)
    policy = C51Policy(model=model, action_space=Discrete(5), num_atoms=33, v_min=-2.0, v_max=3.0)
    ref = orb.rainbow_net(cfg).to(DEV)
    with torch.no_grad():
        for r, p in zip(ref.parameters(), model.parameters(), strict=True):
            r.copy_(p)
    obs = np.random.default_rng(0).standard_normal((200, 4)).astype(np.float32)
    x = torch.as_tensor(obs, device=DEV)
    for train in (True, False):
        policy.train(train)
        ref.train(train)
        out = policy(Batch(obs=obs, info=Batch()))
        probs = ref(x)
        torch.testing.assert_close(out.logits, probs, rtol=1e-5, atol=1e-6)
        q = (out.logits * policy.support).sum(2)
        assert np.array_equal(out.act, q.argmax(1).cpu().numpy())
    policy.train(True)
    noisy = policy(Batch(obs=obs, info=Batch())).logits
    policy.eval()
    assert not torch.equal(noisy, policy(Batch(obs=obs, info=Batch())).logits)


# ------------------------------------------------------------------------------------------------------------ refusals
@gpu
def test_refusals():
    """Every existing algorithm refuses a network with heads, and C51 a noisy layer; RainbowDQN refuses what C51 refuses."""
    from tianshou_b200.algorithm import AdamOptimizerFactory, C51, C51Policy, QRDQN, QRDQNPolicy, RainbowDQN, UnsupportedModelError
    from tianshou_b200.algorithm.modelfree.dqn import DQN, DiscreteQLearningPolicy
    from tianshou_b200.env.atari import RainbowNet
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.discrete import NoisyLinear
    A, N = 3, 8
    opt = AdamOptimizerFactory(lr=1e-3)
    noisy = lambda x, y: NoisyLinear(x, y, 0.1)
    dueling = lambda n: Net(state_shape=(4,), action_shape=A, hidden_sizes=(16,), softmax=n > 1, num_atoms=n,
                            dueling_param=({"linear_layer": noisy}, {})).to(DEV)
    rainbow = lambda **kw: RainbowNet(c=4, h=44, w=44, action_shape=A, num_atoms=N, **kw).to(DEV)
    for model in (dueling(N), rainbow(), rainbow(is_dueling=False)):
        with pytest.raises(UnsupportedModelError, match="separate Q / V heads"):
            C51(policy=C51Policy(model=model, action_space=Discrete(A), num_atoms=N), optim=opt)
        with pytest.raises(UnsupportedModelError, match="separate Q / V heads"):
            QRDQN(policy=QRDQNPolicy(model=model, action_space=Discrete(A)), optim=opt)
    for model in (dueling(1), rainbow()):
        with pytest.raises(UnsupportedModelError, match="separate Q / V heads"):
            DQN(policy=DiscreteQLearningPolicy(model=model, action_space=Discrete(A)), optim=opt)
    plain_noisy = Net(state_shape=(4,), action_shape=A, hidden_sizes=(16,), softmax=True, num_atoms=N, linear_layer=noisy).to(DEV)
    with pytest.raises(UnsupportedModelError, match="RainbowDQN only"):
        C51(policy=C51Policy(model=plain_noisy, action_space=Discrete(A), num_atoms=N), optim=opt)
    RainbowDQN(policy=C51Policy(model=plain_noisy, action_space=Discrete(A), num_atoms=N), optim=opt)      # a plain noisy chain
    no_softmax = Net(state_shape=(4,), action_shape=A, hidden_sizes=(16,), num_atoms=N, dueling_param=({}, {})).to(DEV)
    with pytest.raises(UnsupportedModelError, match="softmax"):
        RainbowDQN(policy=C51Policy(model=no_softmax, action_space=Discrete(A), num_atoms=N), optim=opt)
    with pytest.raises(UnsupportedModelError, match="outputs, not 3 actions x 7 atoms"):
        RainbowDQN(policy=C51Policy(model=rainbow(), action_space=Discrete(A), num_atoms=7), optim=opt)
    with pytest.raises(UnsupportedModelError, match="no CPU path"):
        RainbowDQN(policy=C51Policy(model=rainbow().cpu(), action_space=Discrete(A), num_atoms=N), optim=opt)
    for kw in (dict(gamma=1.5), dict(n_step_return_horizon=0)):
        with pytest.raises(AssertionError):
            RainbowDQN(policy=C51Policy(model=rainbow(), action_space=Discrete(A), num_atoms=N), optim=opt, **kw)


# ------------------------------------------------------------------------------------------------------------ constructions
@gpu
def test_reference_algorithm_constructions():
    """The construction of test/discrete/test_rainbow.py and examples/atari/atari_rainbow.py (default arguments), and one update
    of each.  ``NoisyLinear`` allocates on the CPU as the reference's does, and there is no CPU path: each network is moved to
    the device before its policy and algorithm are built."""
    from tianshou_b200.algorithm import AdamOptimizerFactory, C51Policy, RainbowDQN
    from tianshou_b200.env.atari import RainbowNet
    from tianshou_b200.utils import policy_within_training_step
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.discrete import NoisyLinear
    def noisy_linear(x: int, y: int) -> NoisyLinear:
        return NoisyLinear(x, y, 0.1)

    net = Net(state_shape=(4,), action_shape=2, hidden_sizes=[128, 128, 128, 128], softmax=True, num_atoms=51,
              dueling_param=({"linear_layer": noisy_linear}, {"linear_layer": noisy_linear})).to(DEV)
    optim = AdamOptimizerFactory(lr=1e-3)
    policy = C51Policy(model=net, action_space=Discrete(2), num_atoms=51, v_min=-10.0, v_max=10.0, eps_training=0.1,
                       eps_inference=0.05)
    mlp = RainbowDQN(policy=policy, optim=optim, gamma=0.99, n_step_return_horizon=3, target_update_freq=320)
    atari_net = RainbowNet(c=4, h=84, w=84, action_shape=6, num_atoms=51, noisy_std=0.1, is_dueling=True, is_noisy=True).to(DEV)
    atari_policy = C51Policy(model=atari_net, action_space=Discrete(6), num_atoms=51, v_min=-10.0, v_max=10.0,
                             eps_training=0.1, eps_inference=0.005)
    atari = RainbowDQN(policy=atari_policy, optim=AdamOptimizerFactory(lr=0.0000625), gamma=0.99, n_step_return_horizon=3,
                       target_update_freq=500).to(DEV)
    rng = np.random.default_rng(0)
    for algo, A in ((mlp, 2), (atari, 6)):
        if algo is atari:
            from tianshou_b200.data import Batch, VectorReplayBuffer
            buf = VectorReplayBuffer(64, 2, device=DEV, stack_num=4, ignore_obs_next=True, save_only_last_obs=True)
            for _ in range(20):
                fr = rng.integers(0, 256, (2, 4, 84, 84), dtype=np.uint8)
                buf.add(Batch(obs=fr, act=rng.integers(0, A, 2), rew=rng.standard_normal(2), terminated=np.zeros(2, bool),
                              truncated=np.zeros(2, bool), obs_next=fr), buffer_ids=np.arange(2))
        else:
            buf = make_buffer("mlp", A, rng)
        with policy_within_training_step(algo.policy):
            loss = algo.update(buffer=buf, sample_size=32).loss
        assert np.isfinite(loss)


# ------------------------------------------------------------------------------------------------------------ resources
def test_kernels_have_no_stack_frame_or_spills(tmp_path):
    report = ptxas_report("rainbow.cu", tmp_path)
    kernels = ("noisy_weight_kernel", "noisy_grad_kernel", "dueling_atoms_kernel", "dueling_atoms_bwd_kernel")
    assert len(report) == 4 and all(any(k in e for k in kernels) for e in report), report
    assert_spill_free(report)
