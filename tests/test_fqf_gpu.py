"""FQF on the GPU: the fraction proposal, target and fraction-loss kernels against the float64 restatement
(oracle/oracle_fqf.py), ``FQF.update()`` against outputs of the imported reference (tests/golden/fqf_ref_*.npz from
oracle/gen_golden_fqf.py), one update's gradients of both parameter groups against float64 autograd, bit-identical repeats,
the ``state_dict()`` round trip, the batch edges, the policy's torch path, the refusals and the kernels' register report."""
import copy

import numpy as np
import pytest
import torch
from torch import nn

from oracle import oracle_discrete_sac as ods
from oracle import oracle_fqf as of
from oracle import oracle_iqn as oi
from offpolicy_testutil import (DEV, EPS, Discrete, assert_spill_free, capture_batches, capture_grads, check_final_state,
                                check_second_batch_size, ptxas_report, sm_count, stream, vector_buffer_from_golden)
from test_iqn_gpu import fp64_quantiles
from test_qrdqn_gpu import make_buffer
from ts_testutil import load_golden, record_parity, sum_length_rel

gpu = pytest.mark.gpu
TINY = 2.0 ** -149                      # fp32's smallest subnormal: the spacing of every result below 2^-126
VARIANTS = ["fqf_ref_mlp", "fqf_ref_relu", "fqf_ref_cnn", "fqf_ref_per"]


def dev(a, dt=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dt, device=DEV)


# ------------------------------------------------------------------------------------------------------------ fractions
def _fractions(z):
    from tianshou_b200._cabi import call, ptr
    B, N = z.shape
    zd = dev(z)
    out = {k: torch.empty(*s, device=DEV) for k, s in (("taus", (B, N + 1)), ("tau_hats", (B, N)), ("inner", (B, N - 1)),
                                                       ("p", (B, N)), ("logp", (B, N)), ("H", (B,)))}
    call("ts_fqf_fractions", ptr(zd), B, N, ptr(out["taus"]), ptr(out["tau_hats"]), ptr(out["inner"]), ptr(out["p"]),
         ptr(out["logp"]), ptr(out["H"]), stream())
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in out.items()}


def _logits(B, N, rng, extreme):
    z = (rng.standard_normal((B, N)) * (30.0 if extreme else 1.5)).astype(np.float32)
    if extreme:
        z[0, 0] = 300.0                  # every other probability of row 0 underflows to exactly 0 in fp32
        z[1, :] = -1e30                  # a row of huge equal logits: uniform
        z[2, 0] = -np.inf                # p = 0 and log p clamped to -FLT_MAX: H stays finite, not NaN
    return z


@gpu
@pytest.mark.parametrize("extreme", [False, True])
@pytest.mark.parametrize("N", [2, 13, 32, 200])
def test_fractions_kernel_vs_fp64(N, extreme):
    """p, log p, H, taus, tau_hats and the inner fractions against float64 of the same fp32 logits.

    Error model (fp32, eps = 2^-23): z_j - m is one rounding, a relative |z_j - m| eps in exp; expf and the division add 3 eps;
    s sums in a fixed order over 128 threads, (N / 128 + 7) eps: p_j is within (|z_j - m| + N / 128 + 12) eps of its value,
    plus 4 units of 2^-149 where expf and the division land among the subnormals.
    log p = z - (m + log s) is within 3 eps (|z| + |m| + 1) + (N / 128 + 10) eps.  H sums the products l p over the block: its
    error is the sum of |dl| p + |l| |dp| plus (N / 128 + 10) eps sum |l p|.  The cumulative sum is in double over the kernel's
    own p, so taus[k] is exactly fl32(sum_{j < k} p_j) of its p (checked bit for bit), and within the sum of the p bounds plus
    one rounding of the float64 value.  tau_hats is exactly (taus[:-1] + taus[1:]) / 2 in fp32, inner exactly taus[:, 1:-1].
    B runs past the block-per-row grid (8 blocks per SM) in one case."""
    rng = np.random.default_rng(N * 10 + extreme)
    B = sm_count() * 8 + 37 if (N, extreme) == (13, False) else 41
    z = _logits(B, N, rng, extreme)
    got = _fractions(z)
    ref = of.fractions(z)
    z64 = z.astype(np.float64)
    m = z64.max(1, keepdims=True)
    k = N / 128 + 12
    pb = (np.where(ref["p"] > 0, np.abs(z64 - m), 0.0) + k) * EPS * ref["p"] + 4 * TINY
    assert np.all(np.abs(got["p"] - ref["p"]) <= pb), f"p off by {float((np.abs(got['p'] - ref['p']) / pb).max()):.2f} x its bound"
    lb = np.where(np.isfinite(z64), 3 * EPS * (np.abs(z64) + np.abs(m) + 1) + (k - 2) * EPS, 0.0)
    assert np.all(np.abs(got["logp"] - ref["logp"]) <= lb)
    hb = (lb * ref["p"] + np.abs(ref["logp"]) * pb).sum(1) + (k - 2) * EPS * np.abs(ref["logp"] * ref["p"]).sum(1) + 1e-30
    assert np.all(np.abs(got["H"] - ref["H"]) <= hb)
    tb = np.concatenate([np.zeros((B, 1)), np.cumsum(pb, 1)], 1) + EPS * ref["taus"]
    assert np.all(np.abs(got["taus"] - ref["taus"]) <= tb)
    tag = f"fqf_fractions/N{N}_x{int(extreme)}"
    record_parity(f"{tag}/p", got["p"], ref["p"], rtol=0.0, atol=float(pb.max()))
    record_parity(f"{tag}/H", got["H"], ref["H"], rtol=0.0, atol=float(hb.max()))
    record_parity(f"{tag}/taus", got["taus"], ref["taus"], rtol=0.0, atol=float(tb.max()))
    assert np.all(got["taus"][:, 0] == 0.0)
    assert np.array_equal(got["taus"][:, 1:], np.cumsum(got["p"].astype(np.float64), 1).astype(np.float32)), "fl32 of the cumsum"
    assert np.array_equal(got["tau_hats"], (got["taus"][:, :-1] + got["taus"][:, 1:]) / np.float32(2))
    assert np.array_equal(got["inner"], got["taus"][:, 1:-1])
    if extreme:
        assert np.all(got["p"][0, 1:] == 0.0) and got["p"][0, 0] == 1.0 and np.isfinite(got["H"]).all() and got["H"][0] == 0.0
        assert np.all(np.isfinite(got["logp"])) and got["logp"][2, 0] == -np.finfo(np.float32).max and got["p"][2, 0] == 0.0
        np.testing.assert_allclose(got["p"][1], 1.0 / N, rtol=4 * EPS)
    again = _fractions(z)
    assert all(np.array_equal(got[k], again[k]) for k in got), "two calls must be bit-identical"


# ------------------------------------------------------------------------------------------------------------ target
@gpu
@pytest.mark.parametrize("N", [2, 13, 32, 200])
@pytest.mark.parametrize("A", [1, 2, 6])
def test_target_kernel_exact(A, N):
    """Exact.  Integer-valued quantiles and dyadic widths make every weighted sum exact in fp32 and float64 alike, so equal sums
    are exact ties: the first action must win, and a NaN sum is the maximum.  The widths decide: an unweighted mean picks other
    actions.  B runs past the one-warp-per-row grid in one case; the same-buffer call is ``target_update_freq == 0``."""
    from tianshou_b200._cabi import call, ptr
    g = torch.Generator().manual_seed(A * 1000 + N)
    B = sm_count() * 16 * 8 + 37 if (A, N) == (6, 13) else 301
    q = torch.randint(-3, 4, (B, N, A), generator=g).float()
    w = torch.randint(1, 8, (B, N), generator=g).double()
    taus = (torch.cumsum(torch.cat([torch.zeros(B, 1), w.float() / 1024], 1), 1)).float()          # dyadic: every width exact
    q_next = torch.randn(B, N, A, generator=g)
    if A > 1:
        q[: B // 3, :, A - 1] = q[: B // 3, :, 0]
        q[B - 1, N - 1, A - 1] = float("nan")
    out, act = torch.empty(B, N, device=DEV), torch.empty(B, dtype=torch.int64, device=DEV)
    qd, td, nd = q.to(DEV), taus.to(DEV), q_next.to(DEV)
    call("ts_fqf_target", ptr(qd), ptr(td), ptr(nd), B, A, N, ptr(out), ptr(act), stream())
    torch.cuda.synchronize()
    ref_a = torch.as_tensor(of.fqf_select(q.numpy(), taus.numpy()))
    if A > 1:
        ref_a[B - 1] = A - 1                             # numpy's argmax also takes the NaN; kept explicit
    assert torch.equal(act.cpu(), ref_a)
    assert torch.equal(out.cpu(), q_next[torch.arange(B), :, ref_a])
    if A > 1 and N > 2:
        lead = ((taus[: B // 3, 1:] - taus[: B // 3, :-1]).unsqueeze(2) * q[: B // 3]).sum(1).argmax(1) == 0
        assert bool(lead.any()) and bool((act.cpu()[: B // 3][lead] == 0).all())
        assert not torch.equal(ref_a, q.mean(1).argmax(1)), "the widths must matter"
    out_same = torch.empty(B, N, device=DEV)
    call("ts_fqf_target", ptr(qd), ptr(td), ptr(qd), B, A, N, ptr(out_same), None, stream())
    torch.cuda.synchronize()
    torch.testing.assert_close(out_same.cpu(), q[torch.arange(B), :, ref_a], rtol=0, atol=0, equal_nan=True)


# ------------------------------------------------------------------------------------------------------------ fraction rows
def _fraction_rows(q_hat, q_tau, act, fr, ent_coef):
    from tianshou_b200._cabi import call, ptr
    B, N, A = q_hat.shape
    dz, rows, losses = torch.empty(B, N, device=DEV), torch.empty(3, B, device=DEV), torch.empty(8, device=DEV).fill_(7.0)
    a = (dev(q_hat), dev(q_tau), dev(act, torch.int64), dev(fr["taus"]), dev(fr["p"]), dev(fr["logp"]), dev(fr["H"]))
    call("ts_fqf_fraction_rows", *(ptr(t) for t in a), B, A, N, float(ent_coef), ptr(dz), ptr(rows), losses.data_ptr() + 16, stream())
    torch.cuda.synchronize()
    l = losses.cpu().numpy()
    assert np.all(l[:4] == 7.0), "only the four floats past the pointer are written"
    return l[4:], dz.cpu().numpy()


@gpu
@pytest.mark.parametrize("ent_coef", [0.0, 10.0])
@pytest.mark.parametrize("extreme", [False, True])
@pytest.mark.parametrize("N", [2, 13, 32, 200])
def test_fraction_rows_kernel_vs_fp64(N, extreme, ent_coef):
    """fraction_loss, entropy_loss, their total and dz against the float64 restatement (pinned to autograd of the reference's
    expressions in test_oracle_fqf) on the kernel's own fractions, with exact ties c_i == c_{i-1}, c_0 == h_0 and
    c_{N-2} == h_{N-1} (the strict tests take the negative branch) and (``extreme``) underflowed probabilities.

    Error model: the sign tests compare the same fp32 values in both, so they agree; v1, v2 and g are three roundings,
    3 eps (|v1| + |v2|) per g_i.  G_j sums those in double: within 3 eps times the suffix sum of |v1| + |v2| plus one rounding;
    S = sum p G over the block adds (N / 128 + 10) eps sum |p G|.  dz_j = (1/B) p_j ((G_j - S) + c (l_j + H)) adds 4 eps of each
    product.  fraction_b sums g_i taus_i over the block, (N / 128 + 10) eps of sum |g tau| plus the g errors; the batch means
    come from row_sums3_kernel, (B / 1024 + 12) eps of the mean magnitude.  B runs past the block-per-row grid in one case."""
    rng = np.random.default_rng(N * 100 + extreme * 10 + int(ent_coef))
    B, A = (sm_count() * 8 + 37 if (N, extreme, ent_coef) == (32, False, 10.0) else 41), 4
    fr = {k: v for k, v in _fractions(_logits(B, N, rng, extreme)).items()}
    q_hat = rng.standard_normal((B, N, A)).astype(np.float32)
    q_tau = rng.standard_normal((B, N - 1, A)).astype(np.float32)
    act = rng.integers(0, A, B)
    r = np.arange(B)
    q_hat[r, :, act] = np.sort(q_hat[r, :, act], 1)
    q_tau[r, :, act] = np.sort(q_tau[r, :, act], 1)
    if N > 3:
        q_tau[2, 0, act[2]] = q_hat[2, 0, act[2]]                          # c_0 == h_0
        q_tau[3, 2, act[3]] = q_tau[3, 1, act[3]]                          # c_2 == c_1: both tests of a pair
        q_tau[4, N - 2, act[4]] = q_hat[4, N - 1, act[4]]                  # c_{N-2} == h_{N-1}
    losses, dz = _fraction_rows(q_hat, q_tau, act, fr, ent_coef)
    f64 = {k: v.astype(np.float64) for k, v in fr.items()}
    ref = of.fraction_rows(q_hat.astype(np.float64), q_tau.astype(np.float64), act, f64, ent_coef)
    h, c = q_hat[r, :, act].astype(np.float64), q_tau[r, :, act].astype(np.float64)
    gmag = 3 * EPS * (np.abs(c - h[:, :-1]) + np.abs(c - h[:, 1:]))               # [B, N - 1]
    Gmag = np.concatenate([np.cumsum(gmag[:, ::-1], 1)[:, ::-1], np.zeros((B, 1))], 1)
    G = np.concatenate([np.cumsum(ref["g"][:, ::-1], 1)[:, ::-1], np.zeros((B, 1))], 1)
    p = f64["p"]
    S = (p * G).sum(1, keepdims=True)
    k = N / 128 + 10
    inner = Gmag + EPS * np.abs(G) + (p * Gmag).sum(1, keepdims=True) + k * EPS * (p * np.abs(G)).sum(1, keepdims=True)
    inner += 4 * EPS * (np.abs(G) + np.abs(S) + ent_coef * (np.abs(f64["logp"]) + np.abs(f64["H"])[:, None]))
    dzb = p * inner / B + 4 * EPS * np.abs(ref["dz"]) + 1e-30
    err = np.abs(dz - ref["dz"])
    assert np.all(err <= dzb), f"dz off by {float((err / dzb).max()):.2f} x its bound"
    tag = f"fqf_fraction_rows/N{N}_x{int(extreme)}_c{int(ent_coef)}"
    record_parity(f"{tag}/dz", dz, ref["dz"], rtol=0.0, atol=float(dzb.max()))
    assert np.all(dz[p == 0.0] == 0.0) and np.isfinite(dz).all()
    fmag = (gmag * f64["taus"][:, 1:-1]).sum(1) + k * EPS * np.abs(ref["g"] * f64["taus"][:, 1:-1]).sum(1)
    mb = (np.ceil(B / 1024) + 12) * EPS
    fb = fmag.mean() + mb * np.abs(ref["frac_b"]).mean() + 1e-30
    eb = mb * np.abs(f64["H"]).mean() + 1e-30
    want = [ref["total"], ref["fraction_loss"], ref["entropy_loss"], 0.0]
    bounds = [fb + ent_coef * (eb + EPS * abs(ref["entropy_loss"])) + 2 * EPS * abs(ref["total"]), fb, eb, 0.0]
    for i, name in enumerate(("total", "fraction", "entropy", "zero")):
        assert abs(losses[i] - want[i]) <= bounds[i], f"{tag}: {name} {losses[i]} vs {want[i]}"
    record_parity(f"{tag}/losses", losses, want, rtol=0.0, atol=float(max(bounds)) + 1e-30)
    again = _fraction_rows(q_hat, q_tau, act, fr, ent_coef)
    assert np.array_equal(losses, again[0]) and np.array_equal(dz, again[1]), "two calls must be bit-identical"


@gpu
def test_kernels_refuse_what_a_block_cannot_hold():
    from tianshou_b200._cabi import call, ptr
    x = torch.zeros(16, device=DEV)
    a = torch.zeros(1, dtype=torch.int64, device=DEV)
    for N in (12289, 1, 0):
        with pytest.raises(RuntimeError, match="ts_fqf_fractions"):
            call("ts_fqf_fractions", ptr(x), 1, N, ptr(x), ptr(x), ptr(x), ptr(x), ptr(x), ptr(x), stream())
        with pytest.raises(RuntimeError, match="ts_fqf_fraction_rows"):
            call("ts_fqf_fraction_rows", ptr(x), ptr(x), ptr(a), ptr(x), ptr(x), ptr(x), ptr(x), 1, 1, N, 0.0, ptr(x), ptr(x),
                 ptr(x), stream())
    with pytest.raises(RuntimeError, match="ent_coef"):
        call("ts_fqf_fraction_rows", ptr(x), ptr(x), ptr(a), ptr(x), ptr(x), ptr(x), ptr(x), 1, 1, 2, float("inf"), ptr(x),
             ptr(x), ptr(x), stream())


# ------------------------------------------------------------------------------------------------------------ vs reference
def model_from_cfg(kind, A, N, C=64, obs=4, hidden=(64,), trunk_out=64, last=(64,), H=44, W=44, scale=True):
    from tianshou_b200.env.atari import DQNet, ScaledObsInputActionReprNet
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.discrete import FractionProposalNetwork, FullQuantileFunction
    if kind == "cnn":
        pre = DQNet(c=4, h=H, w=W, action_shape=A, features_only=True)
        pre = ScaledObsInputActionReprNet(pre) if scale else pre
    else:
        pre = Net(state_shape=(obs,), action_shape=trunk_out, hidden_sizes=hidden)
    model = FullQuantileFunction(preprocess_net=pre, action_shape=A, hidden_sizes=last, num_cosines=C).to(DEV)
    return model, FractionProposalNetwork(N, model.input_dim).to(DEV)


def build_from_golden(g):
    from tianshou_b200.algorithm import FQF, AdamOptimizerFactory, FQFPolicy, RMSpropOptimizerFactory
    kind = str(g["cfg_kind"])
    kw = (dict(H=int(g["cfg_H"]), W=int(g["cfg_W"]), scale=bool(g["cfg_scale"])) if kind == "cnn"
          else dict(obs=int(g["cfg_obs"]), hidden=tuple(int(x) for x in g["cfg_hidden"]), trunk_out=int(g["cfg_trunk_out"])))
    A, N = int(g["cfg_A"]), int(g["cfg_N"])
    model, fm = model_from_cfg(kind, A, N, int(g["cfg_C"]), last=tuple(int(x) for x in g["cfg_last"]), **kw)
    ods.seeded_params(model, int(g["cfg_init_seed"]))
    of.seed_fraction_net(fm.net, int(g["cfg_init_seed"]) + 100)
    policy = FQFPolicy(model=model, fraction_model=fm, action_space=Discrete(A))
    frac = (RMSpropOptimizerFactory if str(g["cfg_frac_opt"]) == "rmsprop" else AdamOptimizerFactory)(lr=float(g["cfg_frac_lr"]))
    return FQF(policy=policy, optim=AdamOptimizerFactory(lr=float(g["cfg_lr"])), fraction_optim=frac, gamma=float(g["cfg_gamma"]),
               num_fractions=N, ent_coef=float(g["cfg_ent_coef"]), n_step_return_horizon=int(g["cfg_n_step"]),
               target_update_freq=int(g["cfg_freq"]))


def check_fraction_state(tag, g, algo):
    """The fraction net's final parameters and optimiser state at the bars of ``check_final_state``."""
    view = ods.golden_view
    lr = float(g["cfg_frac_lr"])
    grp = algo._fgroup
    for i, p in enumerate(grp.params):
        record_parity(f"{tag}/fpf_{i}", view(p), g[f"fpf_{i}"], rtol=1e-3, atol=0.1 * lr)
        sq = view(grp.view(grp.exp_avg_sq, p).view(p.shape))
        if f"fsq_{i}" in g:
            v = g[f"fsq_{i}"]
            record_parity(f"{tag}/fsq_{i}", sq, v, rtol=4e-3, atol=4e-3 * float(np.abs(v).max()) + 1e-20)
        else:
            m, v = g[f"fm_{i}"], g[f"fv_{i}"]
            record_parity(f"{tag}/fm_{i}", view(grp.view(grp.exp_avg, p).view(p.shape)), m, rtol=2e-3,
                          atol=2e-3 * float(np.abs(m).max()) + 1e-12)
            record_parity(f"{tag}/fv_{i}", sq, v, rtol=4e-3, atol=4e-3 * float(np.abs(v).max()) + 1e-20)
    assert grp.sync_step_from_device() == int(g["fstep"])


@gpu
@pytest.mark.parametrize("mirror", [False, True])
@pytest.mark.parametrize("variant", VARIANTS)
def test_update_matches_reference_run(variant, mirror):
    """Update after update against the reference's run: the same sampled indices, n-step returns over N columns, the four
    statistics, the priorities written back (PER: and the sum-tree leaves), then the final state of both parameter groups at
    the QR-DQN bars (DESIGN.md section 4) and the reference's ``state_dict()`` keys and optimiser count.  The per-update bars
    are IQN's.  The device's fractions differ from the reference's in the last bit, and a one-ulp change of a fraction moves
    the third update of ``fqf_ref_mlp`` by up to 7e-6 in the returns (measured on the float64 restatement: the sign tests of
    the fraction loss and the first RMSprop steps amplify it), so that run stops after three updates."""
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden(f"{variant}.npz")
    algo, buf = build_from_golden(g), vector_buffer_from_golden(g, mirror)
    keys = [str(k) for k in g["state_dict_keys"]]
    assert list(algo.state_dict().keys()) == keys and len(algo._optimizers) == int(g["optimizer_count"]) == 2
    assert algo._optimizers == [algo.optim, algo.fraction_optim]
    with capture_batches(algo) as cap:
        for u in range(int(g["cfg_updates"])):
            np.random.seed(500 + u)
            with policy_within_training_step(algo.policy):
                stats = algo.update(buffer=buf, sample_size=int(g["cfg_bs"]))
            tag = f"{variant}_m{int(mirror)}_u{u}"
            assert np.array_equal(cap["indices"], g[f"u{u}_indices"]), "sampled indices differ from the reference's"
            ref_ret = g[f"u{u}_returns"]
            record_parity(f"{tag}/returns", cap["returns"].cpu().numpy(), ref_ret, rtol=1e-5, atol=1e-5 * float(np.abs(ref_ret).max()))
            got = np.array([stats.loss, stats.quantile_loss, stats.fraction_loss, stats.entropy_loss])
            record_parity(f"{tag}/losses", got, g[f"u{u}_losses"], rtol=2e-5, atol=2e-6 * float(np.abs(g[f"u{u}_losses"]).max()))
            record_parity(f"{tag}/prio", cap["prio"].cpu().numpy(), g[f"u{u}_prio"], rtol=2e-5, atol=2e-6)
            if bool(g["cfg_per"]):
                leaves = np.asarray(buf.weight[np.arange(len(buf))])
                record_parity(f"{tag}/tree_leaves", leaves, g[f"u{u}_tree_leaves"], rtol=2e-5, atol=1e-7)
    check_final_state(f"{variant}_m{int(mirror)}", g, algo)
    check_fraction_state(f"{variant}_m{int(mirror)}", g, algo)
    assert list(algo.state_dict().keys()) == keys


# ------------------------------------------------------------------------------------------------------------ gradients
def grad_case(kind, B=64, N=13, ent_coef=10.0, edge=""):
    """One update at batch ``B``: both flat gradients, snapshotted before their optimiser steps, against float64 autograd of the
    reference's losses (fqf.py:200-247) on float64 copies of the two networks with the same weights, batch and returns; the
    fractions, quantiles and sign tests are recomputed in float64.  The quantile network's bars are IQN's (2e-4 relative plus
    1e-4 of the tensor's largest value, the documented sum-length term where it passes 1e-4).  The fraction net's gradient is
    dz^T feat, at the same bars: g_i is a difference of neighbouring quantiles, but the fp32 quantiles' errors stay far below
    them (DESIGN.md section 4)."""
    from tianshou_b200.algorithm import FQF, AdamOptimizerFactory, FQFPolicy, RMSpropOptimizerFactory
    from tianshou_b200.utils import policy_within_training_step
    torch.manual_seed(3)
    rng = np.random.default_rng(4)
    A = 5
    if kind == "cnn":
        model, fm = model_from_cfg("cnn", A, N, C=33, last=(48,))
    else:
        model, fm = model_from_cfg("mlp", A, N, C=33, hidden=(48,), trunk_out=40 if kind == "mlp" else 0, last=(40,))
    of.seed_fraction_net(fm.net, 9)
    policy = FQFPolicy(model=model, fraction_model=fm, action_space=Discrete(A))
    algo = FQF(policy=policy, optim=AdamOptimizerFactory(lr=1e-3), fraction_optim=RMSpropOptimizerFactory(lr=1e-4), gamma=0.9,
               num_fractions=N, ent_coef=ent_coef, n_step_return_horizon=2, target_update_freq=3)
    buf = make_buffer(kind, A, rng)
    grp, fgrp = algo._group, algo._fgroup
    ref = copy.deepcopy(model).to("cpu", torch.float64)
    rfm = copy.deepcopy(fm).to("cpu", torch.float64)
    np.random.seed(7)
    with (capture_batches(algo) as cap, capture_grads(grp) as grads, capture_grads(fgrp, "optimizer_step") as fgrads,
          policy_within_training_step(algo.policy)):
        stats = algo.update(buffer=buf, sample_size=B)
    idx = cap["indices"]
    assert len(idx) == B
    raw = np.asarray(buf.obs)[idx]
    if kind == "cnn":
        x = torch.as_tensor((raw.astype(np.float64) / 255.0).astype(np.float32)).double()
        ref.preprocess = ref.preprocess.module
    else:
        x = torch.as_tensor(raw).double()
    pre_net = ref.preprocess
    feat = (pre_net.net if hasattr(pre_net, "net") else pre_net.model.model)(x)
    z = rfm.net(feat.detach())
    dist = torch.distributions.Categorical(logits=z)
    with torch.no_grad():
        taus = torch.nn.functional.pad(torch.cumsum(dist.probs, 1), (1, 0))
        tau_hats = (taus[:, :-1] + taus[:, 1:]) / 2
    q = fp64_quantiles(ref, x, tau_hats)
    with torch.no_grad():
        q_tau = fp64_quantiles(ref, x, taus[:, 1:-1])
    act = torch.as_tensor(np.asarray(buf.act)[idx].astype(np.int64))
    rows = torch.arange(B)
    loss, _ = oi.reference_loss(q, act, cap["returns"].cpu().double(), tau_hats, 1.0)
    floss, fl, el = of.reference_fraction_loss(z, q[rows, act, :].detach(), q_tau[rows, act, :], ent_coef)
    (loss + floss).backward()
    rel = max(1e-4, sum_length_rel(B * N))
    for i, (p, r) in enumerate(zip(grp.params, ref.parameters(), strict=True)):
        want = r.grad.numpy()
        got = grp.view(grads[-1], p).view(p.shape).cpu().numpy()
        record_parity(f"fqf_grad{edge}/{kind}/grad_{i}", got, want, rtol=2e-4, atol=rel * float(np.abs(want).max()) + 1e-12)
    for i, (p, r) in enumerate(zip(fgrp.params, rfm.parameters(), strict=True)):
        want = r.grad.numpy()
        got = fgrp.view(fgrads[-1], p).view(p.shape).cpu().numpy()
        record_parity(f"fqf_grad{edge}/{kind}/fgrad_{i}", got, want, rtol=2e-4, atol=1e-4 * float(np.abs(want).max()) + 1e-12)
    want = [loss.item() + floss.item(), loss.item(), fl.item(), el.item()]
    got = [stats.loss, stats.quantile_loss, stats.fraction_loss, stats.entropy_loss]
    record_parity(f"fqf_grad{edge}/{kind}/losses", got, want, rtol=2e-5, atol=2e-6 * max(abs(v) for v in want))
    return algo


@gpu
@pytest.mark.parametrize("kind", ["mlp", "relu_trunk", "cnn"])
def test_update_gradients_of_both_groups_vs_fp64_autograd(kind):
    grad_case(kind)


@gpu
@pytest.mark.parametrize("batch", ["one", "odd", "past_grid"])
def test_update_gradients_at_batch_edges(batch):
    """B = 1, an odd B and the smallest B that takes the block-per-row kernels (8 blocks per SM) past their grid."""
    B = {"one": 1, "odd": 17, "past_grid": sm_count() * 8 + 1}[batch]
    grad_case("mlp", B=B, N=32, edge=f"_{batch}")


@gpu
@pytest.mark.parametrize("order", ["large_then_small", "small_then_large"])
def test_second_batch_size_is_bit_identical_to_a_fresh_instance(order):
    """One batch size, every scratch tensor filled with NaN, then another: both groups, the lagged copy, the statistics and the
    priorities equal, bit for bit, the second update of a fresh instance loaded from the same ``state_dict()``."""
    g = load_golden("fqf_ref_relu.npz")         # a uniform buffer: a prioritised one would carry the first update's priorities
    large, small = sm_count() * 8 + 1, 3
    B1, B2 = (large, small) if order == "large_then_small" else (small, large)
    carry_iter = lambda a, b: setattr(b, "_iter", a._iter)
    cap, state = check_second_batch_size(lambda: build_from_golden(g), vector_buffer_from_golden(g), B1, B2, carry=carry_iter)
    assert cap["prio"] is not None and len(state) == 12


# ------------------------------------------------------------------------------------------------------------ repeats, state_dict
def _groups(algo):
    return [algo._group, algo._fgroup] + ([algo._g_old] if algo._g_old is not None else [])


@gpu
def test_two_updates_from_one_state_agree_bit_for_bit():
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden("fqf_ref_mlp.npz")
    algos = [build_from_golden(g), build_from_golden(g)]
    for a in algos:
        buf = vector_buffer_from_golden(g)
        for u in range(2):
            np.random.seed(20 + u)
            with policy_within_training_step(a.policy):
                a.update(buffer=buf, sample_size=int(g["cfg_bs"]))
    for ga, gb in zip(*(_groups(a) for a in algos), strict=True):
        assert torch.equal(ga.flat, gb.flat) and torch.equal(ga.exp_avg, gb.exp_avg) and torch.equal(ga.exp_avg_sq, gb.exp_avg_sq)


@gpu
@pytest.mark.parametrize("variant", ["fqf_ref_mlp", "fqf_ref_relu", "fqf_ref_cnn"])
def test_state_dict_round_trip_continues_identically(variant):
    """A fresh algorithm loaded from another's ``state_dict()`` continues bit for bit: online, lagged, the fraction net and both
    optimisers' state (RMSprop's square_avg, or Adam's moments).  ``_iter`` is a plain attribute, as in the reference."""
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden(f"{variant}.npz")
    a, buf_a = build_from_golden(g), vector_buffer_from_golden(g)
    for u in range(3):
        np.random.seed(u)
        with policy_within_training_step(a.policy):
            a.update(buffer=buf_a, sample_size=int(g["cfg_bs"]))
    sd = copy.deepcopy(a.state_dict())
    fo = sd["_optimizers"][1]["state"]
    assert set(next(iter(fo.values()))) == ({"step", "square_avg"} if str(g["cfg_frac_opt"]) == "rmsprop" else
                                            {"step", "exp_avg", "exp_avg_sq"})
    b = build_from_golden(g)
    with torch.no_grad():
        for p in b.policy.parameters():
            p.add_(0.01)
    b.load_state_dict(sd)
    b._iter = a._iter
    for algo in (a, b):
        buf = vector_buffer_from_golden(g)
        for u in range(3):
            np.random.seed(10 + u)
            with policy_within_training_step(algo.policy):
                algo.update(buffer=buf, sample_size=int(g["cfg_bs"]))
    for ga, gb in zip(_groups(a), _groups(b), strict=True):
        assert torch.equal(ga.flat, gb.flat) and torch.equal(ga.exp_avg, gb.exp_avg) and torch.equal(ga.exp_avg_sq, gb.exp_avg_sq)
        assert ga.sync_step_from_device() == gb.sync_step_from_device()


# ------------------------------------------------------------------------------------------------------------ policy
@gpu
def test_policy_action_and_fractions():
    from tianshou_b200.algorithm import FQFPolicy
    from tianshou_b200.data import Batch
    torch.manual_seed(0)
    model, fm = model_from_cfg("mlp", 5, 11, C=17, hidden=(32,), trunk_out=0, last=(24,))
    of.seed_fraction_net(fm.net, 3)
    policy = FQFPolicy(model=model, fraction_model=fm, action_space=Discrete(5))
    obs = np.random.default_rng(0).standard_normal((300, 4)).astype(np.float32)
    batch = Batch(obs=obs, info=Batch())
    for training in (True, False):
        policy.train(training)
        out = policy(batch)
        assert out.logits.shape == (300, 5, 11) and out.fractions.taus.shape == (300, 12)
        assert (out.quantiles_tau is not None) == training
        w = out.fractions.taus[:, 1:] - out.fractions.taus[:, :-1]
        assert np.array_equal(out.act, (w.unsqueeze(1) * out.logits).sum(2).argmax(1).cpu().numpy())
        assert float(w.detach().std()) > 0.01, "the seeded fraction net proposes non-uniform widths"
    old = copy.deepcopy(model)
    again = policy(batch, model=old, fractions=out.fractions)
    assert again.fractions is out.fractions and torch.equal(again.logits, out.logits)


# ------------------------------------------------------------------------------------------------------------ refusals
@gpu
def test_refusals():
    from tianshou_b200.algorithm import (FQF, IQN, QRDQN, AdamOptimizerFactory, FQFPolicy, RMSpropOptimizerFactory,
                                         UnsupportedModelError)
    from tianshou_b200.algorithm.optim import OptimizerFactory
    from tianshou_b200.utils.net.discrete import FractionProposalNetwork
    A, N = 3, 8

    def make(model=None, fm=None, opt=AdamOptimizerFactory, fopt=RMSpropOptimizerFactory, **kw):
        m, f = model_from_cfg("mlp", A, N, C=8, hidden=(16,), trunk_out=16, last=(16,))
        return FQF(policy=FQFPolicy(model=model or m, fraction_model=fm or f, action_space=Discrete(A)), optim=opt(lr=1e-3),
                   fraction_optim=fopt(lr=1e-4), **kw)

    algo = make()
    assert isinstance(algo, QRDQN) and not isinstance(algo, IQN)
    model, _ = model_from_cfg("mlp", A, N, C=8, hidden=(16,), trunk_out=16, last=(16,))
    with pytest.raises(UnsupportedModelError, match="fraction_model: expected"):
        make(model, FractionProposalNetwork(N, 15).to(DEV))
    with pytest.raises(UnsupportedModelError, match="fraction_model: expected"):
        make(model, nn.Sequential(nn.Linear(16, N)).to(DEV))
    bad = FractionProposalNetwork(N, 16).to(DEV)
    bad.extra = nn.Linear(2, 2).to(DEV)
    with pytest.raises(UnsupportedModelError, match="exactly its Linear"):
        make(model, bad)
    lin = nn.Linear(16, 16).to(DEV)
    model2, _ = model_from_cfg("mlp", A, N, C=8, hidden=(16,), trunk_out=16, last=(16,))
    model2.last.model[0] = lin                            # the head's first layer: Linear(16, 16)
    fm2 = FractionProposalNetwork(16, 16).to(DEV)
    fm2.net = lin
    with pytest.raises(UnsupportedModelError, match="shares parameters"):
        make(model2, fm2)
    with pytest.raises(UnsupportedModelError, match="at least 2"):
        make(model, FractionProposalNetwork(1, 16).to(DEV))
    bad_embed, _ = model_from_cfg("mlp", A, N, C=8, hidden=(16,), trunk_out=16, last=(16,))
    bad_embed.embed_model.net = nn.Sequential(nn.Linear(8, 16)).to(DEV)
    with pytest.raises(UnsupportedModelError, match="embedding must be"):
        make(bad_embed)
    with pytest.raises(UnsupportedModelError, match="Adam"):
        make(opt=RMSpropOptimizerFactory)

    class SGDFactory(OptimizerFactory):
        def _create_optimizer_for_params(self, params):
            return torch.optim.SGD(params, lr=1e-3)

    with pytest.raises(UnsupportedModelError, match="RMSprop"):
        make(fopt=lambda lr: SGDFactory())
    with pytest.raises(UnsupportedModelError, match="no CPU path"):
        m, f = model_from_cfg("mlp", A, N, C=8, hidden=(16,), trunk_out=16, last=(16,))
        make(m.cpu(), f.cpu())
    with pytest.raises(UnsupportedModelError, match="fraction_model lives on"):
        make(model, FractionProposalNetwork(N, 16))
    with pytest.raises(ValueError, match="ent_coef"):
        make(ent_coef=float("nan"))
    for kw in (dict(gamma=1.5), dict(n_step_return_horizon=0), dict(num_fractions=1)):
        with pytest.raises(AssertionError):
            make(**kw)


# ------------------------------------------------------------------------------------------------------------ resources
def test_kernels_have_no_stack_frame_or_spills(tmp_path):
    report = ptxas_report("fqf.cu", tmp_path)
    kernels = ("fqf_fractions_kernel", "fqf_target_kernel", "fqf_fraction_rows_kernel", "row_sums3_kernel")
    assert len(report) == len(kernels) and all(any(k in e for e in report) for k in kernels), report
    assert_spill_free(report)
