"""Pin the restatement of FQF (oracle/oracle_fqf.py: float64 numpy fraction proposal, target, fraction loss rows and their
gradient under plain torch networks) to float64 autograd of the reference's expressions and to outputs of the imported
reference (tests/golden/fqf_ref_*.npz from oracle/gen_golden_fqf.py); ``FractionProposalNetwork`` / ``FullQuantileFunction``
against the reference modules.  CPU only."""
import numpy as np
import pytest
import torch
from torch import nn

from oracle import oracle_discrete_sac as ods
from oracle import oracle_fqf as of
from oracle import oracle_iqn as oi
from oracle_testutil import check_final
from test_oracle_iqn import oracle_setup
from ts_testutil import load_golden

VARIANTS = ["fqf_ref_mlp", "fqf_ref_relu", "fqf_ref_cnn", "fqf_ref_per"]


def fraction_net(g, net) -> nn.Linear:
    """The golden's fraction net ``Linear(D, N)`` with its seeded initial weights."""
    lin = nn.Linear(net.embed.out_features, int(g["cfg_N"]))
    of.seed_fraction_net(lin, int(g["cfg_init_seed"]) + 100)
    return lin


def check_fraction_final(g, lin, opt):
    """The fraction net's final parameters and optimiser state against the golden, at the bars of ``check_final``."""
    view = ods.golden_view
    lr = float(g["cfg_frac_lr"])
    for i, p in enumerate(lin.parameters()):
        np.testing.assert_allclose(view(p), g[f"fpf_{i}"], rtol=1e-3, atol=0.1 * lr, err_msg=f"fraction parameter {i}")
        st = opt.state[p]
        if f"fsq_{i}" in g:
            v = g[f"fsq_{i}"]
            np.testing.assert_allclose(view(st["square_avg"]), v, rtol=2e-3, atol=2e-3 * float(np.abs(v).max()) + 1e-20)
        else:
            m, v = g[f"fm_{i}"], g[f"fv_{i}"]
            np.testing.assert_allclose(view(st["exp_avg"]), m, rtol=1e-3, atol=1e-3 * float(np.abs(m).max()) + 1e-12)
            np.testing.assert_allclose(view(st["exp_avg_sq"]), v, rtol=2e-3, atol=2e-3 * float(np.abs(v).max()) + 1e-20)
        assert int(st["step"]) == int(g["fstep"])


@pytest.mark.parametrize("variant", VARIANTS)
def test_fqf_oracle_matches_reference_run(variant):
    g = load_golden(f"{variant}.npz")
    net, buf, obs_of = oracle_setup(g)
    lin = fraction_net(g, net)
    w = np.diff(g["init_widths"], axis=1)
    assert g["init_widths"].max() > 2.0 * g["init_widths"].min() and np.abs(w).max() > 0, "the proposed widths must be non-uniform"
    freq = int(g["cfg_freq"])
    s = of.FqfState(net, lin, float(g["cfg_lr"]), str(g["cfg_frac_opt"]), float(g["cfg_frac_lr"]), freq)
    w0 = lin.weight.detach().clone()
    for u in range(int(g["cfg_updates"])):
        isw = g[f"u{u}_is_weight"] if bool(g["cfg_per"]) else None
        res = of.fqf_update(s, obs_of, buf, g[f"u{u}_indices"], isw, float(g["cfg_gamma"]), int(g["cfg_n_step"]),
                            float(g["cfg_ent_coef"]))
        ref_ret = g[f"u{u}_returns"]
        assert res["returns"].shape == ref_ret.shape == (int(g["cfg_bs"]), int(g["cfg_N"]))
        np.testing.assert_allclose(res["returns"], ref_ret, rtol=1e-5, atol=1e-5)
        np.testing.assert_allclose(res["losses"], g[f"u{u}_losses"], rtol=1e-5, atol=1e-5)
        np.testing.assert_allclose(res["prio"], g[f"u{u}_prio"], rtol=1e-5, atol=1e-6)
    assert s.iter == int(g["iter"]) and int(g["optimizer_count"]) == 2
    assert float((lin.weight.detach() - w0).abs().max()) > 10 * float(g["cfg_frac_lr"]) * 0.1, "the fraction weights must move"
    check_final(g, list(net.parameters()), s.opt, list(s.old.parameters()) if s.old is not None else [])
    check_fraction_final(g, lin, s.fopt)


# ------------------------------------------------------------------------------------------------------------ vs autograd
def _case(B, N, A, seed, extreme=False):
    rng = np.random.default_rng(seed)
    z = rng.standard_normal((B, N)) * (40.0 if extreme else 1.5)
    if extreme:
        z[0, 0] = 2000.0                 # every other probability of row 0 underflows to 0, in float64 as in fp32
    q_hat = rng.standard_normal((B, N, A))
    q_tau = rng.standard_normal((B, N - 1, A))
    act = rng.integers(0, A, B)
    r = np.arange(B)
    if N > 3:                            # exact ties on both strict sign tests
        q_tau[1, 0, act[1]] = q_hat[1, 0, act[1]]
        q_tau[1, 2, act[1]] = q_tau[1, 1, act[1]]
        q_tau[2, N - 2, act[2]] = q_hat[2, N - 1, act[2]]
    q_hat[r, :, act] = np.sort(q_hat[r, :, act], 1)
    return z, q_hat, q_tau, act


@pytest.mark.parametrize("N,ent_coef,extreme", [(2, 0.0, False), (13, 10.0, False), (32, 0.5, True), (200, 10.0, True)])
def test_fraction_rows_match_autograd_of_reference_expression(N, ent_coef, extreme):
    """fraction_loss, entropy_loss, their total and d total / d z against float64 autograd of discrete.py:242-252 and
    fqf.py:221-247, with exact ties in both sign tests and (``extreme``) a row whose other probabilities underflow to 0."""
    B, A = 9, 4
    z, q_hat, q_tau, act = _case(B, N, A, N * 7 + int(extreme), extreme)
    fr = of.fractions(z)
    r = of.fraction_rows(q_hat, q_tau, act, fr, ent_coef)
    zt = torch.tensor(z, requires_grad=True)
    rows = torch.arange(B)
    total, fl, el = of.reference_fraction_loss(zt, torch.tensor(q_hat)[rows, :, act], torch.tensor(q_tau)[rows, :, act], ent_coef)
    total.backward()
    if extreme:
        assert fr["p"][0, 1:].max() == 0.0 and np.isfinite(r["dz"]).all() and np.isfinite(el.item())
    np.testing.assert_allclose(r["fraction_loss"], fl.item(), rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(r["entropy_loss"], el.item(), rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(r["total"], total.item(), rtol=1e-12, atol=1e-12)
    want = zt.grad.numpy()                  # (G_j - S) and (logp_j + H) cancel: the bar is relative to the largest element
    np.testing.assert_allclose(r["dz"], want, rtol=1e-9, atol=1e-12 * float(np.abs(want).max()))
    dist = torch.distributions.Categorical(logits=torch.tensor(z))
    taus = torch.nn.functional.pad(torch.cumsum(dist.probs, 1), (1, 0))
    np.testing.assert_allclose(fr["taus"], taus.numpy(), rtol=1e-13, atol=1e-15)
    np.testing.assert_allclose(fr["H"], dist.entropy().numpy(), rtol=1e-12, atol=1e-15)


def test_sign_tests_are_strict():
    """A tie on either sign test takes the negative branch (``>`` / ``<``, not ``>=`` / ``<=``)."""
    h = np.array([[0.0, 3.0, 5.0]])
    c = np.array([[1.0, 1.0]])                            # c_0 == c_1: a tie on the second test of i = 0 and the first of i = 1
    g = of.gradient_of_taus(h, c)
    assert g[0, 0] == (1.0 - 0.0) - (1.0 - 3.0)           # c_0 > h_0; c_0 < c_1 is false (<= would give -1)
    assert g[0, 1] == -(1.0 - 3.0) + (1.0 - 5.0)          # c_1 > c_0 is false (>= would give -6); c_1 < h_2


def test_target_takes_first_arg_max_of_the_weighted_mean():
    rng = np.random.default_rng(2)
    B, N, A = 50, 6, 5
    q = rng.integers(-3, 4, (B, N, A)).astype(np.float64)
    q[:10, :, 3] = q[:10, :, 1]
    taus = np.concatenate([np.zeros((B, 1)), np.cumsum(rng.integers(1, 4, (B, N)) / 16.0, 1)], 1)      # dyadic: exact sums
    q_next = rng.standard_normal((B, N, A))
    a = (np.diff(taus, axis=1)[:, :, None] * q).sum(1).argmax(1)
    np.testing.assert_array_equal(of.fqf_target(q, taus, q_next), q_next[np.arange(B), :, a])
    assert not np.any(of.fqf_select(q[:10], taus[:10]) == 3)
    assert not np.array_equal(of.fqf_select(q, taus), oi.iqn_select(q)), "the widths must matter"


# ------------------------------------------------------------------------------------------------------------ reference API
def _reference():
    from oracle.ref_shim import import_reference, reference_available
    if not reference_available():
        pytest.skip("reference tree not present")
    return import_reference()


@pytest.mark.parametrize("kind", ["mlp", "relu_trunk", "cnn"])
@pytest.mark.parametrize("training", [True, False])
def test_full_quantile_function_matches_reference(kind, training):
    """Equal parameter names, initialisation and, for equal weights, equal quantiles, fractions, entropies and (training mode)
    quantiles at taus[:, 1:-1]; given fractions are used as given; the policies pick the same actions."""
    _reference()
    from gymnasium.spaces import Discrete as RDiscrete
    from tianshou.algorithm.modelfree.fqf import FQFPolicy as RFQFPolicy
    from tianshou.data import Batch as RBatch
    from tianshou.env.atari.atari_network import DQNet as RDQNet
    from tianshou.utils.net.common import Net as RNet
    from tianshou.utils.net.discrete import FractionProposalNetwork as RFPN
    from tianshou.utils.net.discrete import FullQuantileFunction as RFQF

    from tianshou_b200.algorithm import FQFPolicy
    from tianshou_b200.data import Batch
    from tianshou_b200.env.atari import DQNet
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.discrete import FractionProposalNetwork, FullQuantileFunction, ImplicitQuantileNetwork
    nets = []
    for net_cls, dq_cls, fqf_cls, fpn_cls in ((RNet, RDQNet, RFQF, RFPN), (Net, DQNet, FullQuantileFunction, FractionProposalNetwork)):
        torch.manual_seed(11)
        if kind == "cnn":
            pre = dq_cls(c=4, h=44, w=44, action_shape=6, features_only=True)
        else:
            pre = net_cls(state_shape=(4,), action_shape=64 if kind == "mlp" else 0, hidden_sizes=(32,))
        m = fqf_cls(preprocess_net=pre, action_shape=6, hidden_sizes=(24,), num_cosines=17)
        nets.append((m, fpn_cls(13, m.input_dim)))
    (ref, rfm), (ours, fm) = nets
    assert isinstance(ours, ImplicitQuantileNetwork)
    assert list(ours.state_dict()) == list(ref.state_dict()) and list(fm.state_dict()) == list(rfm.state_dict()) == ["net.weight", "net.bias"]
    assert torch.equal(fm.net.weight, rfm.net.weight) and torch.equal(fm.net.bias, torch.zeros(13)), "the same initialisation"
    assert fm.num_fractions == 13 and fm.embedding_dim == ours.input_dim
    ours.load_state_dict(ref.state_dict())
    of.seed_fraction_net(rfm.net, 5)
    fm.load_state_dict(rfm.state_dict())
    for m in (ref, ours):
        m.train(training)
    x = torch.rand(5, 4, 44, 44) if kind == "cnn" else torch.randn(5, 4)
    (q_r, fr_r, qt_r), _ = ref(x, propose_model=rfm)
    (q, fr, qt), _ = ours(x, propose_model=fm)
    assert q.shape == (5, 6, 13) and fr.taus.shape == (5, 14) and fr.tau_hats.shape == (5, 13) and fr.entropies.shape == (5,)
    for a, b in ((q, q_r), (fr.taus, fr_r.taus), (fr.tau_hats, fr_r.tau_hats), (fr.entropies, fr_r.entropies)):
        assert torch.equal(a, b)
    if training:
        assert qt.shape == (5, 6, 12) and torch.equal(qt, qt_r) and not qt.requires_grad
    else:
        assert qt is None and qt_r is None
    given = Batch(taus=fr.taus.detach() * 0.5, tau_hats=fr.tau_hats.detach() * 0.5)
    (q2, fr2, _), _ = ours(x, propose_model=fm, fractions=given)
    (q2_r, _, _), _ = ref(x, propose_model=rfm, fractions=RBatch(taus=given.taus, tau_hats=given.tau_hats))
    assert fr2 is given and torch.equal(q2, q2_r)
    pol = FQFPolicy(model=ours, fraction_model=fm, action_space=RDiscrete(6))
    rpol = RFQFPolicy(model=ref, fraction_model=rfm, action_space=RDiscrete(6))
    obs = x.numpy()
    out, rout = pol(Batch(obs=obs, info=Batch())), rpol(RBatch(obs=obs, info=RBatch()))
    np.testing.assert_array_equal(out.act, rout.act)
    assert torch.equal(out.fractions.taus, rout.fractions.taus) and torch.equal(out.logits, rout.logits)
