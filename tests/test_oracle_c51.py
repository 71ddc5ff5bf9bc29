"""Pin the restatement of C51 (oracle/oracle_c51.py: float64 numpy softmax, expected values, target, projection, cross-entropy,
logit gradient and priorities under plain torch networks) to float64 autograd of the reference's expressions and to outputs
of the imported reference (tests/golden/c51_ref_*.npz from oracle/gen_golden_c51.py); ``C51Net``, ``C51Policy`` and
``LossSequenceTrainingStats`` against the reference's.  CPU only."""
import numpy as np
import pytest
import torch

from oracle import oracle_c51 as oc
from oracle import oracle_discrete_sac as ods
from oracle_testutil import check_final
from ts_testutil import load_golden

VARIANTS = ["c51_ref_mlp", "c51_ref_cnn", "c51_ref_per"]


def oracle_setup(g, device="cpu"):
    """The oracle network with the golden's seeded initial weights, the golden's buffer view and its observation reader."""
    net = oc.net_from_cfg(g)
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
def test_c51_oracle_matches_reference_run(variant):
    g = load_golden(f"{variant}.npz")
    net, buf, obs_of = oracle_setup(g)
    s = oc.C51State(net, float(g["cfg_lr"]), int(g["cfg_freq"]), float(g["cfg_v_min"]), float(g["cfg_v_max"]))
    for u in range(int(g["cfg_updates"])):
        isw = g[f"u{u}_is_weight"] if bool(g["cfg_per"]) else None
        res = oc.c51_update(s, obs_of, buf, g[f"u{u}_indices"], isw, float(g["cfg_gamma"]), int(g["cfg_n_step"]))
        np.testing.assert_allclose(res["returns"], g[f"u{u}_returns"], rtol=1e-5, atol=1e-5)
        np.testing.assert_allclose(res["loss"], g[f"u{u}_losses"][0], rtol=1e-5, atol=1e-6)
        np.testing.assert_allclose(res["prio"], g[f"u{u}_prio"], rtol=1e-5, atol=1e-6)
    assert s.iter == int(g["iter"])
    check_final(g, list(net.parameters()), s.opt, list(s.old.parameters()) if s.old is not None else [])
    assert [int(i) for i in g["opt_param_ids"]] == list(range(len(list(net.parameters())) + 1))
    assert [int(i) for i in g["opt_state_ids"]] == list(range(1, len(list(net.parameters())) + 1))   # support (0) has none


def test_per_golden_clamps_returns_at_both_ends():
    g = load_golden("c51_ref_per.npz")
    ret = np.concatenate([g[f"u{u}_returns"].reshape(-1) for u in range(int(g["cfg_updates"]))])
    assert ret.min() < float(g["cfg_v_min"]) and ret.max() > float(g["cfg_v_max"])
    assert float(g["cfg_v_min"]) != -float(g["cfg_v_max"]) and int(g["cfg_N"]) % 2 == 1


@pytest.mark.parametrize("weighted", [False, True])
def test_rows_match_autograd_of_reference_expression(weighted):
    """Target, cross-entropy, priorities and d loss / d logits against float64 autograd through the module's softmax, with
    returns exactly on an atom, exactly delta_z from one, and clamped at both ends."""
    rng = np.random.default_rng(11 + weighted)
    B, A, N, v_min, v_max = 9, 4, 7, -2.0, 4.0
    dz = (v_max - v_min) / (N - 1)
    z = np.linspace(v_min, v_max, N)
    logits = rng.standard_normal((B, A, N)) * 2
    act = rng.integers(0, A, B)
    ret = rng.uniform(v_min - 3, v_max + 3, (B, N))
    ret[0, :3] = z[2], z[4] + dz, z[0] - dz           # on an atom, delta_z from one (the next atom), below v_min
    ret[1, :2] = v_max + 5.0, v_min - 5.0              # clamped at both ends
    nd = oc.softmax(rng.standard_normal((B, N)))
    w = rng.uniform(0.2, 1.0, B) if weighted else None
    r = oc.c51_rows(logits, act, ret, z, v_min, v_max, dz, nd, w)
    lt = torch.tensor(logits, requires_grad=True)
    target = oc.reference_target(torch.tensor(nd), torch.tensor(ret), torch.tensor(z), v_min, v_max, dz)
    loss, ce = oc.reference_loss(lt.softmax(-1), act, target, torch.tensor(w) if weighted else 1.0)
    loss.backward()
    np.testing.assert_allclose(r["target"], target.numpy(), rtol=1e-12, atol=1e-15)
    np.testing.assert_allclose(r["loss"], loss.item(), rtol=1e-12)
    np.testing.assert_allclose(r["prio"], ce.detach().numpy(), rtol=1e-12)
    np.testing.assert_allclose(r["dlogits"], lt.grad.numpy(), rtol=1e-10, atol=1e-15)
    # a return on atom 2 carrying all of next_dist projects all of it onto atom 2
    one = np.zeros((1, N))
    one[0, 0] = 1.0
    np.testing.assert_array_equal(oc.project(ret[:1], one, z, v_min, v_max, dz)[0], np.eye(N)[2])
    assert np.allclose(target.sum(1).numpy(), 1.0)


def test_target_takes_first_arg_max_of_the_expected_values():
    rng = np.random.default_rng(2)
    z = oc.support(8, -10.0, 10.0)
    lo, ln = rng.standard_normal((50, 5, 8)), rng.standard_normal((50, 5, 8))
    lo[:10, 3] = lo[:10, 1]                          # two equal action blocks: the first wins where they lead
    q = (torch.as_tensor(lo).softmax(-1) * torch.as_tensor(z, dtype=torch.float64)).sum(2)
    a = q.argmax(1).numpy()
    np.testing.assert_array_equal(oc.c51_select(lo, z), a)
    np.testing.assert_allclose(oc.c51_target(lo, ln, z), torch.as_tensor(ln[np.arange(50), a]).softmax(-1).numpy(), rtol=1e-12)
    assert not np.any(oc.c51_select(lo[:10], z) == 3)


# ------------------------------------------------------------------------------------------------------------ reference API
def _reference():
    from oracle.ref_shim import import_reference, reference_available
    if not reference_available():
        pytest.skip("reference tree not present")
    return import_reference()


def test_c51net_matches_reference():
    _reference()
    from tianshou.env.atari.atari_network import C51Net as RC51Net

    from tianshou_b200.env.atari import C51Net
    nets = []
    for cls in (RC51Net, C51Net):
        torch.manual_seed(8)
        nets.append(cls(c=4, h=44, w=44, action_shape=6, num_atoms=9))
    ref, ours = nets
    assert list(ours.state_dict()) == list(ref.state_dict())
    assert ours.action_num == 6 and ours.num_atoms == 9 and ours.input_shape == (4, 44, 44)
    x = torch.rand(3, 4, 44, 44)
    assert torch.equal(ours(x)[0], ref(x)[0]) and ours(x)[0].shape == (3, 6, 9)


def test_policy_support_and_assertions_match_reference():
    _reference()
    from gymnasium.spaces import Discrete
    from tianshou.algorithm.modelfree.c51 import C51Policy as RC51Policy
    from tianshou.utils.net.common import Net as RNet

    from tianshou_b200.algorithm import C51Policy
    from tianshou_b200.utils.net.common import Net
    for kw in (dict(num_atoms=51), dict(num_atoms=21, v_min=-3.0, v_max=7.0)):
        ref = RC51Policy(model=RNet(state_shape=(4,), action_shape=2, softmax=True, num_atoms=kw["num_atoms"]),
                         action_space=Discrete(2), **kw)
        ours = C51Policy(model=Net(state_shape=(4,), action_shape=2, softmax=True, num_atoms=kw["num_atoms"]),
                         action_space=Discrete(2), **kw)
        assert torch.equal(ours.support, ref.support) and not ours.support.requires_grad
        assert list(ours.state_dict()) == list(ref.state_dict())
        assert next(iter(ours.parameters())) is ours.support
    for kw in (dict(num_atoms=1), dict(v_min=1.0, v_max=1.0)):
        with pytest.raises(AssertionError):
            C51Policy(model=Net(state_shape=(4,), action_shape=2), action_space=Discrete(2), **kw)


def test_loss_sequence_training_stats_at_reference_path():
    from tianshou_b200.algorithm.base import TrainingStats
    from tianshou_b200.algorithm.modelfree.reinforce import LossSequenceTrainingStats
    s = LossSequenceTrainingStats(loss=1.5)
    assert isinstance(s, TrainingStats) and s.loss == 1.5


def test_layer_chain_of_categorical_networks():
    """The device path reads either network as a plain chain ending in Linear(., A * N): what atom_chain sees."""
    from tianshou_b200.algorithm.discrete_q import atom_chain, describe_q_network
    from tianshou_b200.algorithm.netgraph import ACT_NONE
    from tianshou_b200.env.atari import C51Net, ScaledObsInputActionReprNet
    from tianshou_b200.utils.net.common import Net
    for model, shape, scale in ((Net(state_shape=(4,), action_shape=3, hidden_sizes=(16,), softmax=True, num_atoms=7), (4,), 1.0),
                                (C51Net(c=4, h=44, w=44, action_shape=3, num_atoms=7), (4, 44, 44), 1.0),
                                (ScaledObsInputActionReprNet(C51Net(c=4, h=44, w=44, action_shape=3, num_atoms=7)), (4, 44, 44), 255.0)):
        inner, in_shape, in_scale = describe_q_network(model)
        layers = atom_chain(inner, in_shape, 3, 7, "categorical", "atoms")
        assert in_shape == shape and in_scale == scale
        assert layers[-1].kind == "linear" and layers[-1].act == ACT_NONE and layers[-1].out_dim == 21
