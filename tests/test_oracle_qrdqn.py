"""Pin the restatement of QR-DQN and discrete CQL (oracle/oracle_qrdqn.py: float64 numpy target, loss rows, gradient and
priorities under plain torch networks) to float64 autograd of the reference's loss expression and to outputs of the imported
reference (tests/golden/{qrdqn,dcql}_ref_*.npz from oracle/gen_golden_qrdqn.py); ``Net(num_atoms)`` and ``QRDQNet`` against the
reference modules.  CPU only."""
import numpy as np
import pytest
import torch

from oracle import oracle_discrete_sac as ods
from oracle import oracle_qrdqn as oq
from oracle_testutil import check_final
from ts_testutil import load_golden

VARIANTS = ["qrdqn_ref_mlp", "qrdqn_ref_cnn", "qrdqn_ref_per", "dcql_ref_mlp", "dcql_ref_cnn"]


def oracle_setup(g, device="cpu"):
    """The oracle network with the golden's seeded initial weights, the golden's buffer view and its observation reader."""
    net = oq.net_from_cfg(g)
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


@pytest.mark.parametrize("variant", VARIANTS)
def test_qrdqn_oracle_matches_reference_run(variant):
    g = load_golden(f"{variant}.npz")
    net, buf, obs_of = oracle_setup(g)
    freq = int(g["cfg_freq"])
    s = oq.QrState(net, float(g["cfg_lr"]), freq)
    mqw = float(g["cfg_min_q_weight"]) if "cfg_min_q_weight" in g else 0.0
    for u in range(int(g["cfg_updates"])):
        isw = g[f"u{u}_is_weight"] if bool(g["cfg_per"]) else None
        res = oq.qrdqn_update(s, obs_of, buf, g[f"u{u}_indices"], isw, float(g["cfg_gamma"]), int(g["cfg_n_step"]), mqw)
        np.testing.assert_allclose(res["returns"], g[f"u{u}_returns"], rtol=1e-5, atol=1e-5)
        ref = g[f"u{u}_losses"]
        np.testing.assert_allclose(res["losses"][: len(ref)], ref, rtol=1e-5, atol=1e-6)
        np.testing.assert_allclose(res["prio"], g[f"u{u}_prio"], rtol=1e-5, atol=1e-6)
    assert s.iter == int(g["iter"])
    check_final(g, list(net.parameters()), s.opt, list(s.old.parameters()) if s.old is not None else [])
    if s.old is not None:      # the last lagged copy precedes the last step
        assert any(not torch.equal(a, b) for a, b in zip(s.old.parameters(), net.parameters()))


@pytest.mark.parametrize("min_q_weight,weighted", [(0.0, False), (0.0, True), (10.0, False), (2.5, True)])
def test_rows_match_autograd_of_reference_expression(min_q_weight, weighted):
    """Losses, priorities and d loss / d q against float64 autograd, with u_ij exactly 0 (the indicator true, zero gradient)
    and exactly +-1 (the Huber knee) on some pairs."""
    rng = np.random.default_rng(int(min_q_weight * 10) + weighted)
    B, A, N = 9, 4, 7
    q = rng.standard_normal((B, A, N)) * 2
    act = rng.integers(0, A, B)
    ret = q[np.arange(B), act, :] + rng.standard_normal((B, N)) * 1.5
    ret[0, 0] = q[0, act[0], 3]                      # u = 0
    ret[1, 1], ret[1, 2] = q[1, act[1], 0] + 1.0, q[1, act[1], 4] - 1.0     # |u| = 1 (exact in float64 for these values)
    w = rng.uniform(0.2, 1.0, B) if weighted else None
    tau = oq.tau_hat(N).astype(np.float64)
    r = oq.qr_rows(q, act, ret, tau, w, min_q_weight)
    qt = torch.tensor(q, requires_grad=True)
    loss, qr, cql, prio = oq.reference_loss(qt, act, torch.tensor(ret), torch.tensor(tau), torch.tensor(w) if weighted else 1.0,
                                         min_q_weight)
    loss.backward()
    want = [loss.item(), qr.item(), cql.item() if min_q_weight else 0.0]
    np.testing.assert_allclose(r["losses"], want, rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(r["prio"], prio.numpy(), rtol=1e-12)
    np.testing.assert_allclose(r["dq"], qt.grad.numpy(), rtol=1e-12, atol=1e-15)


def test_target_takes_first_arg_max_of_the_means():
    rng = np.random.default_rng(2)
    q, q_next = rng.standard_normal((50, 5, 8)), rng.standard_normal((50, 5, 8))
    q[:10, 3] = q[:10, 1]                            # two equal action blocks: the first wins where they lead
    a = q.mean(2).argmax(1)
    np.testing.assert_array_equal(oq.qr_target(q, q_next), q_next[np.arange(50), a])
    assert np.array_equal(oq.qr_select(q), torch.as_tensor(q).mean(2).argmax(1).numpy())
    assert not np.any(oq.qr_select(q[:10]) == 3)


def test_tau_hat_is_the_references_fp32_midpoint():
    """Not (k + 0.5) / N: at N = 5, k = 3 the reference's fp32 midpoint is 0.70000005, (3.5 / 5) rounds to 0.69999999."""
    t = oq.tau_hat(5)
    assert t.dtype == np.float32 and t[3] == np.float32(0.70000005) and t[3] != np.float32(3.5 / 5)


# ------------------------------------------------------------------------------------------------------------ reference API
def _reference():
    from oracle.ref_shim import import_reference, reference_available
    if not reference_available():
        pytest.skip("reference tree not present")
    return import_reference()


@pytest.mark.parametrize("num_atoms", [1, 3])
def test_net_num_atoms_matches_reference(num_atoms):
    _reference()
    from tianshou.utils.net.common import Net as RNet

    from tianshou_b200.utils.net.common import Net
    nets = []
    for cls in (RNet, Net):
        torch.manual_seed(7)
        nets.append(cls(state_shape=(5,), action_shape=4, hidden_sizes=(16, 16), num_atoms=num_atoms))
    ref, ours = nets
    assert list(ours.state_dict()) == list(ref.state_dict())
    x = torch.randn(11, 5)
    y_ref, y = ref(x)[0], ours(x)[0]
    assert y.shape == y_ref.shape == ((11, 4, num_atoms) if num_atoms > 1 else (11, 4))
    assert torch.equal(y, y_ref) and ours.output_dim == ref.output_dim
    torch.manual_seed(7)
    kw = dict(state_shape=(5,), action_shape=4, hidden_sizes=(8,), concat=True, num_atoms=3)
    cat, cat_ref = Net(**kw), RNet(**kw)
    assert cat.model.model[0].in_features == cat_ref.model.model[0].in_features == 5 + 12


def test_qrdqnet_matches_reference():
    _reference()
    from tianshou.env.atari.atari_network import QRDQNet as RQRDQNet

    from tianshou_b200.env.atari import QRDQNet
    nets = []
    for cls in (RQRDQNet, QRDQNet):
        torch.manual_seed(8)
        nets.append(cls(c=4, h=44, w=44, action_shape=6, num_quantiles=9))
    ref, ours = nets
    assert list(ours.state_dict()) == list(ref.state_dict())
    assert ours.action_num == 6 and ours.num_quantiles == 9 and ours.input_shape == (4, 44, 44)
    x = torch.rand(3, 4, 44, 44)
    assert torch.equal(ours(x)[0], ref(x)[0]) and ours(x)[0].shape == (3, 6, 9)


def test_layer_chain_of_quantile_networks():
    """The device path reads either network as a plain chain ending in Linear(., A * N): what describe_q_network and
    compile_sequential see."""
    from tianshou_b200.algorithm.discrete_q import describe_q_network
    from tianshou_b200.algorithm.netgraph import ACT_NONE, compile_sequential, module_layers
    from tianshou_b200.env.atari import QRDQNet, ScaledObsInputActionReprNet
    from tianshou_b200.utils.net.common import Net
    for model, shape, scale in ((Net(state_shape=(4,), action_shape=3, hidden_sizes=(16,), num_atoms=7), (4,), 1.0),
                                (QRDQNet(c=4, h=44, w=44, action_shape=3, num_quantiles=7), (4, 44, 44), 1.0),
                                (ScaledObsInputActionReprNet(QRDQNet(c=4, h=44, w=44, action_shape=3, num_quantiles=7)), (4, 44, 44), 255.0)):
        inner, in_shape, in_scale = describe_q_network(model)
        layers = compile_sequential(module_layers(inner), in_shape)
        assert in_shape == shape and in_scale == scale
        assert layers[-1].kind == "linear" and layers[-1].act == ACT_NONE and layers[-1].out_dim == 21
