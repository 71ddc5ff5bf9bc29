"""Pin the restatement of Rainbow DQN (oracle/oracle_rainbow.py: C51's float64 rows under noisy layers and the dueling
categorical heads) to outputs of the imported reference (tests/golden/rainbow_ref_*.npz from oracle/gen_golden_rainbow.py) and
to autograd of the reference's dueling expression; ``NoisyLinear``, the dueling ``Net``, ``RainbowNet`` and the reference's
model and policy constructions against the reference's.  CPU only."""
import numpy as np
import pytest
import torch
from torch import nn

from oracle import oracle_discrete_sac as ods
from oracle import oracle_rainbow as orb
from oracle_testutil import check_final
from ts_testutil import load_golden

VARIANTS = ["rainbow_ref_mlp", "rainbow_ref_cnn", "rainbow_ref_per", "rainbow_ref_nonoisy", "rainbow_ref_nodueling"]


def oracle_setup(g):
    net = orb.net_from_golden(g)
    ods.seeded_params(net, int(g["cfg_init_seed"]))
    E, cap = int(g["cfg_E"]), int(g["cfg_cap"])
    buf = dict(obs=g["buf_obs"], act=g["buf_act"], rew=g["buf_rew"], done=g["buf_done"], terminated=g["buf_terminated"],
               offset=np.arange(E + 1) * cap, last_index=g["meta_last_index"], lengths=g["meta_lengths"])
    if "buf_obs_next" in g:
        buf["obs_next"] = g["buf_obs_next"]
        obs_of = ods.flat_obs(buf["obs"], "cpu")
    else:
        obs_of = ods.frame_obs(buf, 4, 255.0 if bool(g["cfg_scale"]) else 1.0, "cpu")
    return net, buf, obs_of


@pytest.mark.parametrize("variant", VARIANTS)
def test_rainbow_oracle_matches_reference_run(variant):
    """The reference's run replayed with its recorded noise: returns, loss and priorities per update, both networks' noise
    after every update (on a tick the lagged network holds the online network's), and the final state."""
    g = load_golden(f"{variant}.npz")
    net, buf, obs_of = oracle_setup(g)
    s = orb.RainbowState(net, float(g["cfg_lr"]), int(g["cfg_freq"]), float(g["cfg_v_min"]), float(g["cfg_v_max"]))
    freq = int(g["cfg_freq"])
    for u in range(int(g["cfg_updates"])):
        isw = g[f"u{u}_is_weight"] if bool(g["cfg_per"]) else None
        res = orb.rainbow_update(s, obs_of, buf, g[f"u{u}_indices"], isw, float(g["cfg_gamma"]), int(g["cfg_n_step"]),
                                 g[f"u{u}_noise_on"], g[f"u{u}_noise_old"] if freq > 0 else None)
        np.testing.assert_allclose(res["returns"], g[f"u{u}_returns"], rtol=1e-5, atol=1e-5)
        np.testing.assert_allclose(res["loss"], g[f"u{u}_losses"][0], rtol=1e-5, atol=1e-6)
        np.testing.assert_allclose(res["prio"], g[f"u{u}_prio"], rtol=1e-5, atol=1e-6)
        np.testing.assert_array_equal(orb.get_noise(s.net), g[f"u{u}_eps_on"])
        if freq > 0:
            np.testing.assert_array_equal(orb.get_noise(s.old), g[f"u{u}_eps_old"])
            want = g[f"u{u}_noise_on"] if u % freq == 0 else g[f"u{u}_noise_old"]
            np.testing.assert_array_equal(g[f"u{u}_eps_old"], want)
    assert s.iter == int(g["iter"])
    check_final(g, orb.trainable(net), s.opt, orb.trainable(s.old) if s.old is not None else [])
    n_all = len(list(net.parameters()))
    assert [int(i) for i in g["opt_param_ids"]] == list(range(n_all + 1))
    trained = [i + 1 for i, p in enumerate(net.parameters()) if p.requires_grad]
    assert [int(i) for i in g["opt_state_ids"]] == trained          # support (0) and the noise have none
    noisy = bool(g["cfg_noisy"]) if str(g["cfg_kind"]) == "cnn" else True
    assert (len(g["u0_noise_on"]) > 0) == noisy


def test_goldens_cover_ticks_clamps_and_switches():
    g = load_golden("rainbow_ref_mlp.npz")
    assert int(g["cfg_freq"]) == 2 and int(g["cfg_updates"]) > 4 and int(g["cfg_n_step"]) == 3
    assert not np.array_equal(g["u1_noise_on"], g["u1_noise_old"]) and np.array_equal(g["u2_eps_old"], g["u2_noise_on"])
    g = load_golden("rainbow_ref_per.npz")
    ret = np.concatenate([g[f"u{u}_returns"].reshape(-1) for u in range(int(g["cfg_updates"]))])
    assert ret.min() < float(g["cfg_v_min"]) and ret.max() > float(g["cfg_v_max"]) and int(g["cfg_N"]) == 21
    assert bool(g["cfg_trunk_noisy"]) and len(g["cfg_q_hidden"]) == 1 and len(g["cfg_v_hidden"]) == 1


def test_dueling_combine_and_its_gradient_match_autograd():
    rng = np.random.default_rng(3)
    for A, N in ((1, 2), (2, 51), (6, 7), (18, 3)):
        q, v, dl = rng.standard_normal((5, A, N)), rng.standard_normal((5, N)), rng.standard_normal((5, A, N))
        qt, vt = torch.tensor(q, requires_grad=True), torch.tensor(v, requires_grad=True)
        logits = qt - qt.mean(dim=1, keepdim=True) + vt.view(5, 1, N)
        logits.backward(torch.tensor(dl))
        np.testing.assert_allclose(orb.dueling(q, v), logits.detach().numpy(), rtol=1e-13, atol=1e-15)
        dq, dv = orb.dueling_bwd(dl)
        np.testing.assert_allclose(dq, qt.grad.numpy(), rtol=1e-12, atol=1e-14)
        np.testing.assert_allclose(dv, vt.grad.numpy(), rtol=1e-12, atol=1e-14)


# ------------------------------------------------------------------------------------------------------------ reference API
def _reference():
    from oracle.ref_shim import import_reference, reference_available
    if not reference_available():
        pytest.skip("reference tree not present")
    return import_reference()


def _same(ours, ref, x):
    assert list(ours.state_dict()) == list(ref.state_dict())
    for (k, a), b in zip(ours.state_dict().items(), ref.state_dict().values()):
        assert torch.equal(a, b), k
    for train in (True, False):
        ours.train(train)
        ref.train(train)
        a, b = ours(x), ref(x)
        a, b = (a[0], b[0]) if isinstance(a, tuple) else (a, b)
        assert torch.equal(a, b)


def test_noisy_linear_matches_reference():
    """Construction (the same torch draws), forward in train and eval mode, and ``sample()``'s draws."""
    _reference()
    from tianshou.utils.net.discrete import NoisyLinear as RNoisy

    from tianshou_b200.utils.net.discrete import NoisyLinear
    mods = []
    for cls in (RNoisy, NoisyLinear):
        torch.manual_seed(4)
        mods.append(cls(7, 5, 0.3))
    ref, ours = mods
    _same(ours, ref, torch.randn(3, 7))
    assert not ours.eps_p.requires_grad and not ours.eps_q.requires_grad and ours.sigma == 0.3
    for m in (ref, ours):
        torch.manual_seed(9)
        m.sample()
    assert torch.equal(ours.eps_p, ref.eps_p) and torch.equal(ours.eps_q, ref.eps_q)


def _noisy_factory(cls, std):
    return lambda x, y: cls(x, y, std)


def test_dueling_net_matches_reference():
    _reference()
    from tianshou.utils.net.common import Net as RNet
    from tianshou.utils.net.discrete import NoisyLinear as RNoisy

    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.discrete import NoisyLinear
    for kw in (dict(num_atoms=9, softmax=True), dict(num_atoms=1), dict(num_atoms=5, softmax=True, trunk_noisy=True, heads=[6])):
        nets = []
        for net_cls, noisy_cls in ((RNet, RNoisy), (Net, NoisyLinear)):
            torch.manual_seed(5)
            noisy = _noisy_factory(noisy_cls, 0.2)
            heads = kw.get("heads", [])
            nets.append(net_cls(state_shape=(4,), action_shape=3, hidden_sizes=[16, 8], softmax=kw.get("softmax", False),
                                num_atoms=kw["num_atoms"], linear_layer=noisy if kw.get("trunk_noisy") else nn.Linear,
                                dueling_param=({"linear_layer": noisy, "hidden_sizes": heads}, {"hidden_sizes": heads})))
        ref, ours = nets
        assert ours.use_dueling and ours.output_dim == ref.output_dim
        _same(ours, ref, torch.randn(6, 4))


def test_rainbow_net_matches_reference():
    _reference()
    from tianshou.env.atari.atari_network import RainbowNet as RRainbowNet

    from tianshou_b200.env.atari import RainbowNet
    for kw in (dict(), dict(is_noisy=False), dict(is_dueling=False), dict(is_noisy=False, is_dueling=False)):
        nets = []
        for cls in (RRainbowNet, RainbowNet):
            torch.manual_seed(8)
            nets.append(cls(c=4, h=44, w=44, action_shape=3, num_atoms=7, noisy_std=0.4, **kw))
        ref, ours = nets
        assert ours.output_dim == 21 and ours.action_num == 3 and ours.num_atoms == 7 and ours.input_shape == (4, 44, 44)
        _same(ours, ref, torch.rand(2, 4, 44, 44))


def test_rainbow_module_and_stats_at_reference_paths():
    _reference()
    import tianshou.algorithm as ralg
    from tianshou.algorithm.modelfree.rainbow import RainbowTrainingStats as RStats

    import tianshou_b200.algorithm as alg
    from tianshou_b200.algorithm.modelfree.rainbow import RainbowDQN, RainbowTrainingStats
    assert alg.RainbowDQN is RainbowDQN and hasattr(ralg, "RainbowDQN")
    assert RainbowTrainingStats(loss=1.5).loss == RStats(loss=1.5).loss == 1.5
    assert issubclass(RainbowDQN, alg.C51)


def test_reference_model_and_policy_constructions():
    """The model and policy construction of test/discrete/test_rainbow.py and examples/atari/atari_rainbow.py, with their
    default arguments, against the reference's: same modules, same parameters."""
    _reference()
    from gymnasium.spaces import Discrete
    from tianshou.algorithm.modelfree.c51 import C51Policy as RPolicy
    from tianshou.env.atari.atari_network import RainbowNet as RRainbowNet
    from tianshou.utils.net.common import Net as RNet
    from tianshou.utils.net.discrete import NoisyLinear as RNoisy

    from tianshou_b200.algorithm import C51Policy
    from tianshou_b200.env.atari import RainbowNet
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.discrete import NoisyLinear
    built = []
    for net_cls, noisy_cls, rainbow_cls, policy_cls in ((RNet, RNoisy, RRainbowNet, RPolicy), (Net, NoisyLinear, RainbowNet, C51Policy)):
        torch.manual_seed(1626)

        def noisy_linear(x: int, y: int):
            return noisy_cls(x, y, 0.1)

        net = net_cls(state_shape=(4,), action_shape=2, hidden_sizes=[128, 128, 128, 128], softmax=True, num_atoms=51,
                      dueling_param=({"linear_layer": noisy_linear}, {"linear_layer": noisy_linear}))
        policy = policy_cls(model=net, action_space=Discrete(2), num_atoms=51, v_min=-10.0, v_max=10.0, eps_training=0.1,
                            eps_inference=0.05)
        atari = rainbow_cls(c=4, h=84, w=84, action_shape=6, num_atoms=51, noisy_std=0.1, is_dueling=True, is_noisy=True)
        atari_policy = policy_cls(model=atari, action_space=Discrete(6), num_atoms=51, v_min=-10.0, v_max=10.0, eps_training=0.1,
                                  eps_inference=0.005)
        built.append((policy, atari_policy))
    for ref, ours in zip(built[0], built[1]):
        assert list(ours.state_dict()) == list(ref.state_dict())
        assert all(torch.equal(a, b) for a, b in zip(ours.state_dict().values(), ref.state_dict().values()))


def test_layer_chains_of_rainbow_networks():
    """What the device path reads: three chains for a dueling network (noisy layers marked), one for the others; every other
    algorithm's reader refuses a network with heads and a noisy layer."""
    from tianshou_b200.algorithm import UnsupportedModelError
    from tianshou_b200.algorithm.discrete_q import atom_chain, describe_q_network, dueling_atom_chains
    from tianshou_b200.algorithm.netgraph import compile_sequential, layer_params, module_layers, noise_params
    from tianshou_b200.env.atari import RainbowNet, ScaledObsInputActionReprNet
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.discrete import NoisyLinear
    noisy = _noisy_factory(NoisyLinear, 0.1)
    net = Net(state_shape=(4,), action_shape=3, hidden_sizes=[16], softmax=True, num_atoms=7,
              dueling_param=({"linear_layer": noisy}, {"linear_layer": noisy}))
    _, shape, scale, chains = dueling_atom_chains(net, 3, 7)
    assert shape == (4,) and scale == 1.0 and [len(c) for c in chains] == [1, 1, 1]
    assert [c[-1].out_dim for c in chains] == [16, 21, 7] and chains[0][0].noise is None and chains[1][0].noise is not None
    layers = [L for c in chains for L in c]
    assert [id(p) for p in layer_params(layers)] == [id(p) for p in net.parameters() if p.requires_grad]
    assert [id(p) for p in noise_params(layers)] == [id(p) for p in net.parameters() if not p.requires_grad]
    rb = ScaledObsInputActionReprNet(RainbowNet(c=4, h=44, w=44, action_shape=3, num_atoms=7))
    _, shape, scale, chains = dueling_atom_chains(rb, 3, 7)
    assert shape == (4, 44, 44) and scale == 255.0 and [c[-1].out_dim for c in chains] == [256, 21, 7]
    _, _, _, chains = dueling_atom_chains(RainbowNet(c=4, h=44, w=44, action_shape=3, num_atoms=7, is_dueling=False), 3, 7)
    assert len(chains) == 1 and chains[0][-1].out_dim == 21
    for model in (net, rb.module, RainbowNet(c=4, h=44, w=44, action_shape=3, num_atoms=7, is_dueling=False)):
        with pytest.raises(UnsupportedModelError, match="separate Q / V heads"):
            module_layers(model)
    with pytest.raises(UnsupportedModelError, match="separate Q / V heads"):
        describe_q_network(net)
    plain_noisy = Net(state_shape=(4,), action_shape=3, hidden_sizes=[16], softmax=True, num_atoms=7, linear_layer=noisy)
    inner, shape, _ = describe_q_network(plain_noisy)
    with pytest.raises(UnsupportedModelError, match="RainbowDQN only"):
        atom_chain(inner, shape, 3, 7, "categorical", "atoms")
    assert len(atom_chain(inner, shape, 3, 7, "categorical", "atoms", noisy=True)) == 2
    with pytest.raises(UnsupportedModelError, match="RainbowDQN only"):
        compile_sequential([NoisyLinear(4, 3)], (4,))
    empty = Net(state_shape=(4,), action_shape=3, softmax=True, num_atoms=7, dueling_param=({}, {}))
    with pytest.raises(UnsupportedModelError, match="trunk"):
        dueling_atom_chains(empty, 3, 7)
    with pytest.raises(UnsupportedModelError, match="21 outputs, not 3 actions x 6 atoms"):
        dueling_atom_chains(net, 3, 6)
