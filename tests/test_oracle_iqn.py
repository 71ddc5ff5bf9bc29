"""Pin the restatement of IQN (oracle/oracle_iqn.py: float64 numpy cosine embedding, target, loss rows, gradient and priorities
under plain torch networks) to float64 autograd of the reference's loss expression and to outputs of the imported reference
(tests/golden/iqn_ref_*.npz from oracle/gen_golden_iqn.py, replayed with the fractions the reference drew);
``CosineEmbeddingNetwork`` / ``ImplicitQuantileNetwork`` against the reference modules.  CPU only."""
import numpy as np
import pytest
import torch

from oracle import oracle_discrete_sac as ods
from oracle import oracle_iqn as oi
from test_oracle_discrete_bcq import check_final
from ts_testutil import load_golden

VARIANTS = ["iqn_ref_mlp", "iqn_ref_sizes", "iqn_ref_cnn", "iqn_ref_per"]


def oracle_setup(g, device="cpu"):
    """The oracle network with the golden's seeded initial weights, the golden's buffer view and its observation reader."""
    net = oi.net_from_cfg(g)
    ods.seeded_params(net, int(g["cfg_init_seed"]))
    net.to(device)
    E, cap = int(g["cfg_E"]), int(g["cfg_cap"])
    buf = dict(obs=g["buf_obs"], act=g["buf_act"], rew=g["buf_rew"], done=g["buf_done"], terminated=g["buf_terminated"],
               offset=np.arange(E + 1) * cap, last_index=g["meta_last_index"], lengths=g["meta_lengths"])
    if "buf_obs_next" in g:
        buf["obs_next"] = g["buf_obs_next"]
        obs_of = ods.flat_obs(buf["obs"], device)
    else:
        obs_of = ods.frame_obs(buf, 4, 255.0 if bool(g["cfg_scale"]) else 1.0, device)
    return net, buf, obs_of


def golden_taus(g, device="cpu"):
    """Every fraction tensor the reference drew, in call order."""
    n = sum(int(g[f"u{u}_ntaus"]) for u in range(int(g["cfg_updates"])))
    return [torch.as_tensor(g[f"taus_{k}"], device=device) for k in range(n)]


@pytest.mark.parametrize("variant", VARIANTS)
def test_iqn_oracle_matches_reference_run(variant):
    g = load_golden(f"{variant}.npz")
    net, buf, obs_of = oracle_setup(g)
    freq = int(g["cfg_freq"])
    s = oi.IqnState(net, float(g["cfg_lr"]), freq)
    taus = iter(golden_taus(g))
    for u in range(int(g["cfg_updates"])):
        assert int(g[f"u{u}_ntaus"]) == (3 if freq > 0 else 2)      # target online (+ lagged), then the step
        isw = g[f"u{u}_is_weight"] if bool(g["cfg_per"]) else None
        res = oi.iqn_update(s, obs_of, buf, g[f"u{u}_indices"], isw, float(g["cfg_gamma"]), int(g["cfg_n_step"]),
                            int(g["cfg_S_on"]), int(g["cfg_S_t"]), taus)
        ref_ret = g[f"u{u}_returns"]
        assert res["returns"].shape == ref_ret.shape == (int(g["cfg_bs"]), int(g["cfg_S_t"] if freq > 0 else g["cfg_S_on"]))
        np.testing.assert_allclose(res["returns"], ref_ret, rtol=1e-5, atol=1e-5)
        np.testing.assert_allclose(res["loss"], g[f"u{u}_losses"][0], rtol=1e-5, atol=1e-6)
        np.testing.assert_allclose(res["prio"], g[f"u{u}_prio"], rtol=1e-5, atol=1e-6)
    assert next(taus, None) is None, "every recorded draw is used, in order"
    assert s.iter == int(g["iter"])
    check_final(g, list(net.parameters()), s.opt, list(s.old.parameters()) if s.old is not None else [])


@pytest.mark.parametrize("S_on,S_t,weighted", [(2, 3, False), (8, 8, True), (8, 5, True), (6, 4, False)])
def test_rows_match_autograd_of_reference_expression(S_on, S_t, weighted):
    """Loss, priorities and d loss / d q against float64 autograd of iqn.py:163-179, with u_ij exactly 0 (the indicator true)
    and exactly +-1 (the Huber knee) on some pairs and a fraction of exactly 0."""
    rng = np.random.default_rng(S_on * 10 + S_t + weighted)
    B, A = 9, 4
    q = rng.standard_normal((B, S_on, A)) * 2                       # the kernels' [B][S][A]
    act = rng.integers(0, A, B)
    ret = q[np.arange(B), :S_t % S_on + 1, act].mean(1, keepdims=True) + rng.standard_normal((B, S_t)) * 1.5
    ret[0, 0] = q[0, 1, act[0]]                                     # u = 0
    ret[1, 0], ret[1, 1] = q[1, 0, act[1]] + 1.0, q[1, 1, act[1]] - 1.0      # |u| = 1 (exact in float64 for these values)
    taus = rng.random((B, S_on))
    taus[2, 0] = 0.0
    w = rng.uniform(0.2, 1.0, B) if weighted else None
    r = oi.iqn_rows(q, act, ret, taus, w)
    qt = torch.tensor(q.transpose(0, 2, 1).copy(), requires_grad=True)     # the reference's [B, A, S]
    loss, prio = oi.reference_loss(qt, act, torch.tensor(ret), torch.tensor(taus), torch.tensor(w) if weighted else 1.0)
    loss.backward()
    np.testing.assert_allclose(r["loss"], loss.item(), rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(r["prio"], prio.numpy(), rtol=1e-12)
    np.testing.assert_allclose(r["dq"], qt.grad.numpy().transpose(0, 2, 1), rtol=1e-12, atol=1e-15)


def test_target_takes_first_arg_max_of_the_sample_means():
    rng = np.random.default_rng(2)
    q, q_next = rng.integers(-3, 4, (50, 6, 5)).astype(np.float64), rng.standard_normal((50, 4, 5))
    q[:10, :, 3] = q[:10, :, 1]                     # two equal action columns: the first wins where they lead
    a = q.mean(1).argmax(1)
    np.testing.assert_array_equal(oi.iqn_target(q, q_next), q_next[np.arange(50), :, a])
    assert oi.iqn_target(q, q_next).shape == (50, 4)
    assert not np.any(oi.iqn_select(q[:10]) == 3)


def test_mix_backward_matches_autograd():
    rng = np.random.default_rng(3)
    B, S, D = 5, 3, 7
    for act in ("none", "relu", "tanh"):
        pre = torch.tensor(rng.standard_normal((B, D)), requires_grad=True)
        e_pre = torch.tensor(rng.standard_normal((B * S, D)), requires_grad=True)
        feat = {"none": pre, "relu": torch.relu(pre), "tanh": torch.tanh(pre)}[act]
        e = torch.relu(e_pre)
        h = (feat.unsqueeze(1) * e.view(B, S, D)).view(B * S, D)
        dh = rng.standard_normal((B * S, D))
        h.backward(torch.tensor(dh))
        np.testing.assert_allclose(oi.mix(feat.detach().numpy(), e.detach().numpy(), S), h.detach().numpy(), rtol=1e-15)
        dfeat, de_pre = oi.mix_backward(dh, feat.detach().numpy(), e.detach().numpy(), S, act, feat.detach().numpy())
        np.testing.assert_allclose(dfeat, pre.grad.numpy(), rtol=1e-13, atol=1e-15)
        np.testing.assert_allclose(de_pre, e_pre.grad.numpy(), rtol=1e-13, atol=1e-15)


def test_cos_argument_is_the_references_fp32_expression():
    """fl(tau * fl(fl32(pi) * i)), bit for bit as torch forms ``np.pi * arange(fp32)`` times the fractions; a double-precision pi
    or a fused product gives a different argument."""
    taus = torch.rand(300, 8, generator=torch.Generator().manual_seed(0))
    C = 64
    i_pi = np.pi * torch.arange(1, C + 1, dtype=torch.float32)
    want = (taus.view(300, 8, 1) * i_pi).numpy()
    got = oi.cos_argument(taus.numpy(), C)
    assert got.dtype == np.float32 and np.array_equal(got, want)
    double_pi = (taus.numpy().astype(np.float64)[..., None] * (np.pi * np.arange(1, C + 1))).astype(np.float32)
    assert np.count_nonzero(double_pi != want) > 100


# ------------------------------------------------------------------------------------------------------------ reference API
def _reference():
    from oracle.ref_shim import import_reference, reference_available
    if not reference_available():
        pytest.skip("reference tree not present")
    return import_reference()


@pytest.mark.parametrize("kind", ["mlp", "relu_trunk", "cnn"])
def test_implicit_quantile_network_matches_reference(kind):
    """Equal parameter names and, for equal weights and the same torch RNG state, equal outputs and fractions; the oracle's
    ``IqnNet`` gives the same q on those fractions."""
    _reference()
    from tianshou.env.atari.atari_network import DQNet as RDQNet
    from tianshou.utils.net.common import Net as RNet
    from tianshou.utils.net.discrete import ImplicitQuantileNetwork as RIQN

    from tianshou_b200.env.atari import DQNet
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.discrete import CosineEmbeddingNetwork, ImplicitQuantileNetwork
    nets = []
    for net_cls, dq_cls, iqn_cls in ((RNet, RDQNet, RIQN), (Net, DQNet, ImplicitQuantileNetwork)):
        torch.manual_seed(11)
        if kind == "cnn":
            pre = dq_cls(c=4, h=44, w=44, action_shape=6, features_only=True)
        else:
            pre = net_cls(state_shape=(4,), action_shape=64 if kind == "mlp" else 0, hidden_sizes=(32,))
        nets.append(iqn_cls(preprocess_net=pre, action_shape=6, hidden_sizes=(24,), num_cosines=17))
    ref, ours = nets
    assert list(ours.state_dict()) == list(ref.state_dict())
    assert [n for n, _ in ours.named_parameters()][-2:] == ["embed_model.net.0.weight", "embed_model.net.0.bias"]
    assert isinstance(ours.embed_model, CosineEmbeddingNetwork) and ours.embed_model.num_cosines == 17
    ours.load_state_dict(ref.state_dict())
    x = torch.rand(5, 4, 44, 44) if kind == "cnn" else torch.randn(5, 4)
    outs = []
    for m in (ref, ours):
        torch.manual_seed(3)
        outs.append(m(x, sample_size=7))
    (q_ref, t_ref), _ = outs[0]
    (q, t), _ = outs[1]
    assert q.shape == (5, 6, 7) and t.shape == (5, 7)
    assert torch.equal(t, t_ref) and torch.equal(q, q_ref)
    if kind != "cnn":
        g = {"cfg_kind": "mlp", "cfg_obs": 4, "cfg_hidden": [32], "cfg_trunk_out": 64 if kind == "mlp" else 0, "cfg_last": [24],
             "cfg_A": 6, "cfg_C": 17}
        net = oi.net_from_cfg(g)
        with torch.no_grad():
            for p, r in zip(net.parameters(), ref.parameters(), strict=True):
                p.copy_(r)
        torch.testing.assert_close(net(x, t), q, rtol=0, atol=0)
