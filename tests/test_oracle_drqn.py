"""DRQN's float64 restatement (oracle/oracle_drqn.py) against outputs of the imported reference (tests/golden/drqn_ref_*.npz from
oracle/gen_golden_drqn.py), and ``Recurrent``'s construction, ``state_dict()`` keys and torch forward against the reference's.
CPU only."""
import numpy as np
import pytest
import torch

from oracle import oracle_drqn as od
from oracle import oracle_discrete_sac as ods
from oracle_testutil import check_final
from ts_testutil import load_golden

VARIANTS = ["mlp", "per", "s1"]


def _cfg(g, k):
    return g[f"cfg_{k}"].item()


@pytest.mark.parametrize("variant", VARIANTS)
def test_drqn_oracle_matches_reference_run(variant):
    g = load_golden(f"drqn_ref_{variant}.npz")
    from tianshou_b200.utils.net.common import Recurrent
    L, D, A, H = (int(_cfg(g, k)) for k in ("layers", "obs", "A", "hidden"))
    E, cap, freq = int(_cfg(g, "E")), int(_cfg(g, "cap")), int(_cfg(g, "freq"))
    model = Recurrent(layer_num=L, state_shape=D, action_shape=A, hidden_layer_size=H)
    ods.seeded_params(model, int(_cfg(g, "init_seed")))
    net = od.DrqnNet(L, D, A, H)
    od.load_from(net, list(model.parameters()))
    old = od.DrqnNet(L, D, A, H) if freq > 0 else None
    opt = torch.optim.Adam(net.parameters(), lr=float(_cfg(g, "lr")))
    buf = {k: g["buf_" + k] for k in ("obs", "act", "rew", "terminated", "done")}
    obs_next = bool(_cfg(g, "obs_next"))
    if obs_next:
        buf["obs_next"] = g["buf_obs_next"]
    buf.update(offset=np.arange(E + 1) * cap, last_index=g["meta_last_index"], lengths=g["meta_lengths"])
    huber = float(_cfg(g, "huber")) or None
    for u in range(int(_cfg(g, "updates"))):
        sync = freq > 0 and u % freq == 0
        if sync and u == 0:
            old.load_state_dict(net.state_dict())
        w = g[f"u{u}_is_weight"] if bool(_cfg(g, "per")) else None
        r = od.drqn_update(net, old, opt, buf, g[f"u{u}_indices"], w, float(_cfg(g, "gamma")), int(_cfg(g, "n_step")),
                           bool(_cfg(g, "double")), huber, int(_cfg(g, "stack")), obs_next, sync_target=sync and u > 0)
        np.testing.assert_allclose(r["returns"], g[f"u{u}_returns"].reshape(-1), rtol=1e-5, atol=1e-5, err_msg=f"update {u} returns")
        np.testing.assert_allclose(r["td"], g[f"u{u}_prio"].reshape(-1), rtol=1e-4, atol=1e-5, err_msg=f"update {u} priorities")
        np.testing.assert_allclose(r["loss"], g[f"u{u}_losses"][0], rtol=1e-5, atol=1e-6, err_msg=f"update {u} loss")
    check_final(g, list(net.parameters()), opt, list(old.parameters()) if old is not None else [])
    assert int(g["iter"]) == int(_cfg(g, "updates"))


def test_goldens_cross_episode_starts():
    """Every golden's buffer holds finished episodes, so the stacks and n-step chains cross episode starts."""
    for v in VARIANTS:
        g = load_golden(f"drqn_ref_{v}.npz")
        assert g["buf_done"].sum() >= 4, v


def test_state_dict_keys_and_optimiser_ids_of_goldens():
    g = load_golden("drqn_ref_mlp.npz")
    keys = [str(k) for k in g["state_dict_keys"]]
    lstm = [k for k in keys if ".nn." in k]
    assert lstm[:4] == [f"policy.model.nn.{w}_l0" for w in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]
    assert np.array_equal(g["opt_param_ids"], np.arange(len(g["opt_param_ids"])))
    assert np.array_equal(g["opt_state_ids"], g["opt_param_ids"])


# ------------------------------------------------------------------------------------------------------------ reference API
def _reference():
    from oracle.ref_shim import import_reference, reference_available
    if not reference_available():
        pytest.skip("reference tree not present")
    return import_reference()


@pytest.mark.parametrize("layers,hidden,shape", [(2, 128, 4), (1, 64, (3,)), (3, 5, (2, 2))])
def test_recurrent_matches_reference(layers, hidden, shape):
    _reference()
    from tianshou.utils.net.common import Recurrent as RefRecurrent
    from tianshou_b200.utils.net.common import Recurrent
    torch.manual_seed(3)
    ref = RefRecurrent(layer_num=layers, state_shape=shape, action_shape=3, hidden_layer_size=hidden)
    torch.manual_seed(3)
    mine = Recurrent(layer_num=layers, state_shape=shape, action_shape=3, hidden_layer_size=hidden)
    assert list(mine.state_dict().keys()) == list(ref.state_dict().keys())
    for a, b in zip(mine.parameters(), ref.parameters(), strict=True):
        assert torch.equal(a, b)
    assert mine.get_output_dim() == ref.get_output_dim() == 3
    D = int(np.prod(shape))
    rng = np.random.default_rng(0)
    for obs in (rng.standard_normal((5, D)), rng.standard_normal((5, 4, D))):
        qa, sa = mine(obs)
        qb, sb = ref(obs)
        assert torch.equal(qa, qb)
        assert torch.equal(sa["hidden"], sb["hidden"]) and torch.equal(sa["cell"], sb["cell"])
        assert sa["hidden"].shape == (5, layers, hidden)
        qa2, sa2 = mine(obs, state=sa)
        qb2, sb2 = ref(obs, state=sb)
        assert torch.equal(qa2, qb2) and torch.equal(sa2["cell"], sb2["cell"])
    with pytest.raises(ValueError):
        mine(rng.standard_normal((2, D)), state={"hidden": torch.zeros(2, layers, hidden)})


def test_oracle_net_matches_torch_lstm():
    """The explicit LSTM of the restatement against torch's nn.LSTM through Recurrent, in float64."""
    from tianshou_b200.utils.net.common import Recurrent
    torch.manual_seed(1)
    model = Recurrent(layer_num=2, state_shape=3, action_shape=2, hidden_layer_size=7).double()
    net = od.DrqnNet(2, 3, 2, 7)
    od.load_from(net, list(model.parameters()))
    obs = torch.randn(6, 5, 3, dtype=torch.float64)
    y = model.fc1(obs)
    out, _ = model.nn(y)
    torch.testing.assert_close(net(obs), model.fc2(out[:, -1]), rtol=1e-12, atol=1e-12)
