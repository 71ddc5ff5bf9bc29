"""The eager BDQN restatement (oracle/oracle_bdqn.py) against outputs of the imported reference (tests/golden/bdqn_ref_*.npz from
oracle/gen_golden_bdqn.py), and BranchingNet / BDQNPolicy / the constructor errors against the reference itself when it is
present.  CPU only."""
import copy

import numpy as np
import pytest
import torch

from offpolicy_testutil import MultiDiscrete, golden_cfg, load_params
from ts_testutil import load_golden, record_parity

VARIANTS = ["pendulum", "bipedal", "per_trunc", "b1"]
PRIO_EPS = float(np.finfo(np.float32).eps)


def _check(tag, mod, g, prefix, lr):
    for i, p in enumerate(mod.parameters()):
        record_parity(f"{tag}/{prefix}{i}", p.detach().numpy(), g[f"{prefix}{i}"], rtol=1e-4, atol=1e-3 * lr)


def branching_net(cfg):
    from tianshou_b200.utils.net.common import BranchingNet
    return BranchingNet(state_shape=(int(cfg["obs"]),), num_branches=int(cfg["nb"]), action_per_branch=int(cfg["A"]),
                        common_hidden_sizes=[int(x) for x in cfg["common"]], value_hidden_sizes=[int(x) for x in cfg["value"]],
                        action_hidden_sizes=[int(x) for x in cfg["action"]],
                        activation=torch.nn.Tanh if str(cfg["act_fn"]) == "tanh" else torch.nn.ReLU)


def end_flags(g):
    """``buffer.done`` with True at every unfinished episode's last slot (bdqn.py:155-156)."""
    end = g["buf_done"].copy()
    end[g["buf_unfinished"]] = True
    return end


@pytest.mark.parametrize("variant", VARIANTS)
def test_oracle_matches_reference(variant):
    from oracle.oracle_bdqn import bdqn_update
    g = load_golden(f"bdqn_ref_{variant}.npz")
    cfg = golden_cfg(g)
    net = branching_net(cfg)
    load_params(net, g, "p0_net_")
    freq = int(cfg["target_update_freq"])
    old = copy.deepcopy(net) if freq > 0 else None
    lr = float(cfg["lr"])
    opt = torch.optim.Adam(net.parameters(), lr=lr)
    buf = {k: g["buf_" + k] for k in ("obs", "act", "rew", "obs_next")}
    end = end_flags(g)
    for u in range(int(cfg["updates"])):
        o, tag = f"u{u}_", f"oracle_bdqn/{variant}/u{u}"
        idx = g[o + "indices"]
        w = g[o + "is_weight"].astype(np.float32) if bool(cfg["per"]) else None
        r = bdqn_update(net, opt, old, buf, end, idx, is_double=bool(cfg["is_double"]), is_weight=w,
                        refresh=freq > 0 and u % freq == 0)
        record_parity(f"{tag}/loss", np.float64(r["loss"]), g[o + "loss"], rtol=1e-5, atol=1e-7)
        _check(tag, net, g, o + "net_", lr)
        if old is not None:
            _check(tag, old, g, o + "old_", lr)
        if bool(cfg["per"]):
            want = (np.abs(r["td_sum"].numpy().astype(np.float64)) + PRIO_EPS) ** float(cfg["per_alpha"])
            record_parity(f"{tag}/priorities", g[o + "priorities"][idx], want, rtol=1e-5, atol=0)


def test_goldens_cover_what_they_claim():
    """pendulum refreshes its lagged network inside the recorded updates; bipedal's buffer has unfinished episodes that end flags
    turn on; per_trunc ends episodes by truncation (which BDQN does not bootstrap) and ran past its capacity."""
    g = load_golden("bdqn_ref_pendulum.npz")
    assert int(golden_cfg(g)["updates"]) > int(golden_cfg(g)["target_update_freq"]) > 0
    assert not np.array_equal(g["u2_old_0"], g["u3_old_0"])
    g = load_golden("bdqn_ref_bipedal.npz")
    assert len(g["buf_unfinished"]) > 0 and not g["buf_done"][g["buf_unfinished"]].any()
    sampled = np.concatenate([g[f"u{u}_indices"] for u in range(int(golden_cfg(g)["updates"]))])
    assert np.isin(sampled, g["buf_unfinished"]).any()
    g = load_golden("bdqn_ref_per_trunc.npz")
    assert (g["buf_truncated"] & ~g["buf_terminated"]).any() and int(golden_cfg(g)["adds"]) > int(golden_cfg(g)["size"])
    assert int(golden_cfg(g)["nb"]) > 8


def test_b1_loss_is_the_usual_loss_plus_the_target_variance():
    """At B = 1 the reference's returns broadcast to [nb, nb, A]: the loss gains the population variance over branches of the
    per-branch targets, the gradient does not change."""
    from oracle.oracle_bdqn import TARGET_GAMMA, bdqn_loss, bdqn_targets, q_values
    g = load_golden("bdqn_ref_b1.npz")
    cfg = golden_cfg(g)
    net = branching_net(cfg)
    load_params(net, g, "p0_net_")
    idx = g["u0_indices"]
    end = end_flags(g)
    obs, obs_next = torch.as_tensor(g["buf_obs"][idx]), torch.as_tensor(g["buf_obs_next"][idx])
    act = torch.as_tensor(g["buf_act"][idx])
    returns = bdqn_targets(net, net, obs_next, g["buf_rew"][idx], end[idx], gamma=TARGET_GAMMA, is_double=True)
    assert returns.shape == (3, 3, 4)
    loss, _ = bdqn_loss(net, obs, act, returns)
    t = returns[:, 0, 0].double()
    q = q_values(net, obs).double()[0].gather(-1, act.long().reshape(-1, 1)).flatten()
    usual = ((t.mean() - q) ** 2).mean()
    assert abs(loss.item() - (usual + t.var(unbiased=False)).item()) < 1e-5
    record_parity("oracle_bdqn/b1/u0_loss", np.float64(loss.item()), g["u0_loss"], rtol=1e-5, atol=1e-7)


# ------------------------------------------------------------------------------------------------------------ reference API
def _reference():
    from oracle.ref_shim import import_reference, reference_available
    if not reference_available():
        pytest.skip("reference tree not present")
    return import_reference()


NET_CASES = [
    dict(state_shape=(3,), num_branches=1, action_per_branch=40, common_hidden_sizes=[64, 64], value_hidden_sizes=[64],
         action_hidden_sizes=[64]),
    dict(state_shape=(4, 6), num_branches=4, action_per_branch=25, common_hidden_sizes=[32, 16], value_hidden_sizes=[8],
         action_hidden_sizes=[8, 8], activation=torch.nn.Tanh),
    dict(state_shape=5, num_branches=9, action_per_branch=3, common_hidden_sizes=[12]),
    dict(state_shape=(5,), num_branches=2, action_per_branch=3, common_hidden_sizes=[12, 6], norm_layer=torch.nn.LayerNorm),
]


@pytest.mark.parametrize("case", range(len(NET_CASES)))
def test_branching_net_matches_reference(case):
    _reference()
    from tianshou.utils.net.common import BranchingNet as RNet

    from tianshou_b200.utils.net.common import BranchingNet
    kw = NET_CASES[case]
    torch.manual_seed(5)
    ref = RNet(**kw)
    torch.manual_seed(5)
    mine = BranchingNet(**kw)
    sr, sm = ref.state_dict(), mine.state_dict()
    assert list(sr.keys()) == list(sm.keys()) and all(torch.equal(sr[k], sm[k]) for k in sr)
    assert (mine.num_branches, mine.action_per_branch) == (ref.num_branches, ref.action_per_branch)
    obs = np.random.default_rng(case).standard_normal((7, *np.atleast_1d(kw["state_shape"]))).astype(np.float32)
    (lr_, sr_), (lm, sm_) = ref(obs, state="s"), mine(obs, state="s")
    assert lm.shape == (7, kw["num_branches"], kw["action_per_branch"]) and sr_ == sm_ == "s"
    assert torch.equal(lr_, lm)


def test_branching_net_keys_and_errors_match_reference():
    _reference()
    from tianshou.utils.net.common import BranchingNet as RNet

    from tianshou_b200.utils.net.common import BranchingNet
    keys = list(BranchingNet(state_shape=3, num_branches=2, common_hidden_sizes=[4], value_hidden_sizes=[4],
                             action_hidden_sizes=[4]).state_dict())
    assert keys[:2] == ["common.model.0.weight", "common.model.0.bias"]
    assert "value.model.2.weight" in keys and "branches.1.model.2.bias" in keys
    for kw in (dict(state_shape=3, num_branches=2), dict(state_shape=3, num_branches=2, common_hidden_sizes=[])):
        with pytest.raises(IndexError) as r:
            RNet(**kw)
        with pytest.raises(IndexError) as m:
            BranchingNet(**kw)
        assert str(r.value) == str(m.value)


def _policies(nb=3, A=5):
    from gymnasium.spaces import MultiDiscrete
    from tianshou.algorithm.modelfree.bdqn import BDQNPolicy as RPolicy
    from tianshou.utils.net.common import BranchingNet as RNet

    from tianshou_b200.algorithm.modelfree.bdqn import BDQNPolicy
    from tianshou_b200.utils.net.common import BranchingNet
    kw = dict(state_shape=(4,), num_branches=nb, action_per_branch=A, common_hidden_sizes=[16], value_hidden_sizes=[8],
              action_hidden_sizes=[8])
    torch.manual_seed(1)
    rp = RPolicy(model=RNet(**kw), action_space=MultiDiscrete([A] * nb), eps_training=0.6, eps_inference=0.3)
    torch.manual_seed(1)
    mp = BDQNPolicy(model=BranchingNet(**kw), action_space=MultiDiscrete([A] * nb), eps_training=0.6, eps_inference=0.3)
    return rp, mp


def test_bdqn_policy_forward_matches_reference():
    _reference()
    from tianshou.data import Batch as RBatch

    from tianshou_b200.data import Batch
    rp, mp = _policies()
    obs = np.random.default_rng(3).standard_normal((6, 4)).astype(np.float32)
    for wrap in (False, True):              # the reference's obs.obs unwrap
        ro = RBatch(obs=obs) if wrap else obs
        mo = Batch(obs=obs) if wrap else obs
        r, m = rp(RBatch(obs=ro, info={})), mp(Batch(obs=mo, info={}))
        assert torch.equal(r.logits, m.logits)
        assert m.act.shape == (6, 3) and np.array_equal(r.act, m.act)


def test_bdqn_exploration_noise_matches_reference():
    """The same draws from numpy's global stream: ``rand(bsz)`` then ``randint(0, action_per_branch, (bsz, nb))``; the mask is
    added; eps 0 draws nothing."""
    _reference()
    from tianshou.data import Batch as RBatch
    from tianshou.utils.torch_utils import policy_within_training_step as r_within

    from tianshou_b200.data import Batch
    from tianshou_b200.utils.torch_utils import policy_within_training_step
    rp, mp = _policies()
    act = np.random.default_rng(4).integers(0, 5, (40, 3))
    mask = np.random.default_rng(5).integers(0, 2, (40, 3))
    for training, with_mask in ((True, False), (False, False), (True, True)):
        obs = Batch(obs=np.zeros((40, 4)), mask=mask) if with_mask else np.zeros((40, 4))
        robs = RBatch(obs=np.zeros((40, 4)), mask=mask) if with_mask else np.zeros((40, 4))
        np.random.seed(11)
        if training:
            with r_within(rp):
                r = rp.add_exploration_noise(act.copy(), RBatch(obs=robs))
        else:
            r = rp.add_exploration_noise(act.copy(), RBatch(obs=robs))
        r_next = np.random.rand()
        np.random.seed(11)
        if training:
            with policy_within_training_step(mp):
                m = mp.add_exploration_noise(act.copy(), Batch(obs=obs))
        else:
            m = mp.add_exploration_noise(act.copy(), Batch(obs=obs))
        assert np.array_equal(r, m) and not np.array_equal(m, act) and np.random.rand() == r_next
    rp.eps_inference = mp.eps_inference = 0.0
    np.random.seed(2)
    assert np.array_equal(mp.add_exploration_noise(act.copy(), Batch(obs=np.zeros((40, 4)))), act)
    assert np.random.rand() == np.random.RandomState(2).rand()


def test_bdqn_constructor_errors():
    from tianshou_b200.algorithm import BDQN, UnsupportedModelError
    from tianshou_b200.algorithm.modelfree.bdqn import BDQNPolicy
    from tianshou_b200.algorithm.optim import AdamOptimizerFactory
    from tianshou_b200.utils.net.common import BranchingNet
    net = BranchingNet(state_shape=3, num_branches=2, action_per_branch=4, common_hidden_sizes=[8])
    policy = BDQNPolicy(model=net, action_space=MultiDiscrete([4, 4]))
    with pytest.raises(UnsupportedModelError, match="no CPU path"):
        BDQN(policy=policy, optim=AdamOptimizerFactory(lr=1e-3))
    with pytest.raises(TypeError):
        BDQN(policy=policy, optim=AdamOptimizerFactory(lr=1e-3), n_step_return_horizon=3)      # 1-step returns only


def test_reference_fails_at_b1_with_a_prioritised_buffer():
    """What the device update refuses up front: the reference steps its optimiser, then ``update_weight`` raises on the
    [nb] td sums of its single row."""
    _reference()
    from gymnasium.spaces import MultiDiscrete
    from tianshou.algorithm import BDQN as RBDQN
    from tianshou.algorithm.modelfree.bdqn import BDQNPolicy as RPolicy
    from tianshou.algorithm.optim import AdamOptimizerFactory
    from tianshou.data import Batch, PrioritizedReplayBuffer
    from tianshou.utils.net.common import BranchingNet as RNet
    from tianshou.utils.torch_utils import policy_within_training_step
    torch.manual_seed(0)
    net = RNet(state_shape=(3,), num_branches=3, action_per_branch=4, common_hidden_sizes=[8])
    algo = RBDQN(policy=RPolicy(model=net, action_space=MultiDiscrete([4] * 3)), optim=AdamOptimizerFactory(lr=1e-3))
    buf = PrioritizedReplayBuffer(10, alpha=0.6, beta=0.4)
    for i in range(5):
        buf.add(Batch(obs=np.ones(3, np.float32) * i, act=np.array([0, 1, 2]), rew=1.0, terminated=False, truncated=False,
                      obs_next=np.ones(3, np.float32), info={}))
    before = [p.detach().clone() for p in net.parameters()]
    with policy_within_training_step(algo.policy), pytest.raises(ValueError):
        algo.update(buf, 1)
    assert any(not torch.equal(a, b) for a, b in zip(before, net.parameters()))
