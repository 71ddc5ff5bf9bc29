"""Pin the restatement of discrete BCQ (oracle/oracle_discrete_bcq.py: float64 numpy target, losses and gradients under plain
torch networks) to outputs of the imported reference (tests/golden/dbcq_ref_{mlp,cnn,sep}.npz from
oracle/gen_golden_discrete_bcq.py), and the host logic of ``DiscreteBCQPolicy`` / the two-head network that needs no device.
CPU only."""
import numpy as np
import pytest
import torch

from oracle import oracle_discrete_bcq as odb
from oracle import oracle_discrete_sac as ods
from ts_testutil import load_golden

VARIANTS = ["mlp", "cnn", "sep"]


class _Discrete:
    def __init__(self, n):
        self.n = n
        self.shape = ()


def oracle_setup(g, outs, device="cpu"):
    """Oracle networks with the golden's initial weights, and its buffer view and observation reader."""
    nets = odb.nets_from_cfg(g, outs)
    if bool(g["cfg_compact"]):
        ods.seeded_params(nets, int(g["cfg_init_seed"]))
    else:
        with torch.no_grad():
            for i, p in enumerate(nets.parameters()):
                p.copy_(torch.as_tensor(g[f"p0_{i}"]).reshape(p.shape))
    nets.to(device)
    E, cap = int(g["cfg_E"]), int(g["cfg_cap"])
    buf = dict(obs=g["buf_obs"], act=g["buf_act"], rew=g["buf_rew"], done=g["buf_done"], terminated=g["buf_terminated"],
               offset=np.arange(E + 1) * cap, last_index=g["meta_last_index"], lengths=g["meta_lengths"])
    if "buf_obs_next" in g:
        buf["obs_next"] = g["buf_obs_next"]
        obs_of = ods.flat_obs(buf["obs"], device)
    else:
        obs_of = ods.frame_obs(buf, 4, 255.0, device)
    return nets, buf, obs_of


def check_final(g, params, opt, lagged):
    """Final parameters, Adam moments and lagged parameters against the golden: Adam normalises a step to ~lr per element, so
    the absolute term is stated in units of one step (DESIGN.md section 4)."""
    view = ods.golden_view if bool(g["cfg_compact"]) else (lambda t: t.detach().cpu().numpy())
    lr = float(g["cfg_lr"])
    for i, p in enumerate(params):
        np.testing.assert_allclose(view(p), g[f"pf_{i}"], rtol=1e-3, atol=0.1 * lr, err_msg=f"parameter {i}")
        st = opt.state[p]
        m, v = g[f"m_{i}"], g[f"v_{i}"]
        np.testing.assert_allclose(view(st["exp_avg"]), m, rtol=1e-3, atol=1e-3 * float(np.abs(m).max()) + 1e-12, err_msg=f"exp_avg {i}")
        np.testing.assert_allclose(view(st["exp_avg_sq"]), v, rtol=2e-3, atol=2e-3 * float(np.abs(v).max()) + 1e-20, err_msg=f"exp_avg_sq {i}")
        assert int(st["step"]) == int(g["adam_step"])
    for i, p in enumerate(lagged):
        np.testing.assert_allclose(view(p), g[f"old_{i}"], rtol=1e-3, atol=0.1 * lr, err_msg=f"lagged parameter {i}")


@pytest.mark.parametrize("variant", VARIANTS)
def test_discrete_bcq_oracle_matches_reference_run(variant):
    g = load_golden(f"dbcq_ref_{variant}.npz")
    A = int(g["cfg_A"])
    nets, buf, obs_of = oracle_setup(g, (A, A))
    s = odb.BcqState(nets, float(g["cfg_lr"]))
    tau = float(g["cfg_tau"])
    log_tau = float(np.log(tau)) if tau > 0 else -np.inf
    for u in range(int(g["cfg_updates"])):
        res = odb.discrete_bcq_update(s, obs_of, buf, g[f"u{u}_indices"], float(g["cfg_gamma"]), int(g["cfg_n_step"]),
                                      int(g["cfg_freq"]), log_tau, float(g["cfg_penalty"]))
        np.testing.assert_allclose(res["returns"], g[f"u{u}_returns"].reshape(-1), rtol=1e-5, atol=1e-5)
        np.testing.assert_allclose(res["losses"], g[f"u{u}_losses"], rtol=1e-5, atol=1e-6)
    assert s.iter == int(g["iter"])
    check_final(g, list(nets.parameters()), s.opt, s.old.head_a_parameters())
    # the last lagged copy precedes the last step: the lagged model differs from the online one
    assert any(not torch.equal(a, b) for a, b in zip(s.old.head_a_parameters(), nets.head_a_parameters()))


def test_rows_gradients_match_autograd():
    """The hand-written d loss / d q and d loss / d logits against float64 autograd of the reference expressions, with |td| on
    both sides of the Huber knee and exactly on it."""
    rng = np.random.default_rng(0)
    B, A, penalty = 37, 7, 0.3
    q, z = rng.standard_normal((B, A)) * 2, rng.standard_normal((B, A)) * 3
    act = rng.integers(0, A, B)
    ret = q[np.arange(B), act] + rng.standard_normal(B) * 1.5
    ret[0], ret[1] = q[0, act[0]] - 1.0, q[1, act[1]] + 1.0
    r = odb.bcq_rows(q, z, act, ret, penalty)
    qt, zt = torch.tensor(q, requires_grad=True), torch.tensor(z, requires_grad=True)
    a = torch.as_tensor(act)
    ql = torch.nn.functional.smooth_l1_loss(qt[torch.arange(B), a], torch.tensor(ret))
    il = torch.nn.functional.nll_loss(torch.log_softmax(zt, -1), a)
    reg = zt.pow(2).mean()
    loss = ql + il + penalty * reg
    loss.backward()
    np.testing.assert_allclose(r["losses"], [loss.item(), ql.item(), il.item(), reg.item()], rtol=1e-12)
    np.testing.assert_allclose(r["dq"], qt.grad.numpy(), rtol=1e-12, atol=1e-15)
    np.testing.assert_allclose(r["dlogits"], zt.grad.numpy(), rtol=1e-12, atol=1e-15)


def test_select_matches_torch_expression():
    """Ties under the mask go to the lowest index; with every action but the arg-max-logit one masked that action is taken;
    a threshold of 0 masks nothing."""
    rng = np.random.default_rng(1)
    q = rng.integers(-2, 3, (200, 6)).astype(np.float32)           # many exact ties
    z = rng.standard_normal((200, 6)).astype(np.float32) * 2
    for log_tau in (float(np.log(0.6)), float(np.log(0.05)), -1e-9, -np.inf):
        ratio = torch.as_tensor(z) - torch.as_tensor(z).max(-1, keepdim=True).values
        ref = (torch.as_tensor(q) - torch.finfo(torch.float32).max * (ratio < log_tau).float()).argmax(-1).numpy()
        assert np.array_equal(odb.bcq_select(q, z, log_tau), ref)
    assert np.array_equal(odb.bcq_select(q, z, -1e-9), z.argmax(-1))
    assert np.array_equal(odb.bcq_select(q, z, -np.inf), q.argmax(-1))


# ------------------------------------------------------------------------------------------------------------ host logic
def _heads(shared, trunk=None, A=3, **actor_kw):
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.discrete import DiscreteActor
    mk = trunk or (lambda: Net(state_shape=(4,), hidden_sizes=(16,)))
    t1 = mk()
    t2 = t1 if shared else mk()
    kw = dict(action_shape=A, hidden_sizes=(8,), softmax_output=False)
    return DiscreteActor(preprocess_net=t1, **kw), DiscreteActor(preprocess_net=t2, **{**kw, **actor_kw})


def test_policy_assertions_and_log_tau():
    from tianshou_b200.algorithm import DiscreteBCQPolicy
    model, imitator = _heads(True)
    mk = lambda **kw: DiscreteBCQPolicy(model=model, imitator=imitator, action_space=_Discrete(3), **kw)
    p = mk(unlikely_action_threshold=0.6)
    assert p._log_tau == np.log(0.6) and p.eps_training == 0.0 and p.eps_inference == 0.0
    assert mk(unlikely_action_threshold=0.0)._log_tau == -np.inf
    assert mk(eps_inference=0.1).eps_inference == 0.1
    for kw in (dict(target_update_freq=0), dict(unlikely_action_threshold=1.0), dict(unlikely_action_threshold=-0.1)):
        with pytest.raises(AssertionError):
            mk(**kw)


def test_flat_order_is_the_optimisers_order():
    """Shared parameters once, in the order ``policy.parameters()`` / ``ModuleList([policy, critic]).parameters()`` gives."""
    from tianshou_b200.algorithm.shared_trunk import two_head_parameters
    for shared in (True, False):
        a, b = _heads(shared)
        got = two_head_parameters(a, b)
        ref = list(torch.nn.ModuleList([a, b]).parameters())
        assert [id(p) for p in got] == [id(p) for p in ref]
        assert len(got) == (2 + 4 + 4 if shared else 2 * (2 + 4))


def test_two_head_network_detects_sharing_and_refuses():
    from tianshou_b200.algorithm import UnsupportedModelError
    from tianshou_b200.algorithm.flat_params import FlatGroup
    from tianshou_b200.algorithm.shared_trunk import TwoHeadNetwork, two_head_parameters
    from tianshou_b200.env.atari import DQNet, ScaledObsInputActionReprNet
    from tianshou_b200.utils.net.common import Net
    cpu = torch.device("cpu")
    build = lambda a, b: TwoHeadNetwork(a, b, FlatGroup(two_head_parameters(a, b), cpu), roles=("model", "imitator"))
    assert build(*_heads(True)).shared and not build(*_heads(False)).shared
    cnn = lambda: ScaledObsInputActionReprNet(DQNet(4, 44, 44, 3, features_only=True))
    net = build(*_heads(True, trunk=cnn))
    assert net.shared and net.in_shape == (4, 44, 44) and net.in_scale == 255.0 and net.n_out == (3, 3)
    # one layer of the trunk shared, the rest private
    a, b = _heads(False, trunk=lambda: Net(state_shape=(4,), hidden_sizes=(16, 16)))
    b.preprocess.model.model[0] = a.preprocess.model.model[0]
    with pytest.raises(UnsupportedModelError, match="share some parameters"):
        build(a, b)
    a, b = _heads(False)
    b.preprocess = Net(state_shape=(5,), hidden_sizes=(16,))
    with pytest.raises(UnsupportedModelError, match="must read it the same way"):
        build(a, b)
    a, b = _heads(False)
    b.preprocess = ScaledObsInputActionReprNet(b.preprocess, denom=2.0)
    with pytest.raises(UnsupportedModelError, match="must read it the same way"):
        build(a, b)
    with pytest.raises(UnsupportedModelError, match="softmax preprocess"):
        build(*_heads(True, trunk=lambda: Net(state_shape=(4,), hidden_sizes=(16,), softmax=True)))
    a, b = _heads(True)
    b.last.model.append(torch.nn.ReLU())
    with pytest.raises(UnsupportedModelError, match="imitator: must end in a linear layer"):
        build(a, b)
    a, b = _heads(True)
    b.last.model[-1] = torch.nn.Linear(8, 3, bias=False)
    with pytest.raises(UnsupportedModelError, match="bias"):
        build(a, b)
