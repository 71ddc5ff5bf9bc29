"""The eager REDQ restatement (oracle/oracle_redq.py) against outputs of the imported reference (tests/golden/redq_ref_*.npz from
oracle/gen_golden_redq.py), and EnsembleLinear / REDQPolicy / the REDQ constructor against the reference itself when it is
present.  CPU only."""
import numpy as np
import pytest
import torch

from offpolicy_testutil import golden_cfg, load_params, oracle_buffer
from ts_testutil import load_golden, record_parity

VARIANTS = ["mujoco", "per_mean", "full"]


def _check(tag, mod, g, prefix, lr):
    for i, p in enumerate(mod.parameters()):
        record_parity(f"{tag}/{prefix}{i}", p.detach().numpy(), g[f"{prefix}{i}"], rtol=1e-4, atol=1e-3 * lr)


def cpu_noise(shape):
    """``Normal.rsample``'s draw on torch's CPU generator."""
    return torch.empty(shape).normal_()


def build_oracle(g):
    from oracle.oracle_redq import AutoAlpha, FixedAlpha, RedqNets
    cfg = golden_cfg(g)
    O, A, H, E = int(cfg["obs"]), int(cfg["act"]), tuple(int(x) for x in cfg["hidden"]), int(cfg["E"])
    nets = RedqNets(O, A, H, E)
    load_params(nets.actor, g, "p0_actor_"); load_params(nets.critic, g, "p0_critic_")
    nets.critic_old.load_state_dict(nets.critic.state_dict())
    opts = [torch.optim.Adam(nets.actor.parameters(), lr=float(cfg["actor_lr"])),
            torch.optim.Adam(nets.critic.parameters(), lr=float(cfg["critic_lr"]))]
    alpha = AutoAlpha(-A, 0.0, float(cfg["alpha_lr"])) if bool(cfg["auto_alpha"]) else FixedAlpha(float(cfg["alpha"]))
    return cfg, nets, opts, alpha


@pytest.mark.parametrize("variant", VARIANTS)
def test_oracle_matches_reference(variant):
    from oracle.oracle_redq import redq_update
    g = load_golden(f"redq_ref_{variant}.npz")
    cfg, nets, opts, alpha = build_oracle(g)
    buf = oracle_buffer(g)
    last, actor_steps = 0.0, 0
    for u in range(int(cfg["updates"])):
        o, tag = f"u{u}_", f"oracle_redq/{variant}/u{u}"
        w = torch.as_tensor(g[o + "is_weight"]).float() if bool(cfg["per"]) else None
        torch.manual_seed(100 + u)
        step = (u + 1) % int(cfg["delay"]) == 0
        r = redq_update(nets, opts, alpha, buf, g[o + "indices"], cpu_noise, g[o + "subset"], gamma=float(cfg["gamma"]),
                        n_step=int(cfg["n_step"]), tau=float(cfg["tau"]), target_mode=str(cfg["target_mode"]), actor_step=step,
                        is_weight=w)
        if step:
            last, actor_steps = r["actor_loss"], actor_steps + 1
        record_parity(f"{tag}/losses", np.array([last, r["critic_loss"]]), g[o + "losses"], rtol=1e-5, atol=1e-6)
        record_parity(f"{tag}/alpha", np.float64(alpha.value), g[o + "alpha"], rtol=1e-6, atol=0)
        assert (r["alpha_loss"] is None) == bool(np.isnan(g[o + "alpha_loss"]))
        assert len(set(g[o + "subset"].tolist())) == int(cfg["M"])
        _check(tag, nets.actor, g, o + "actor_", float(cfg["actor_lr"]))
        _check(tag, nets.critic, g, o + "critic_", float(cfg["critic_lr"]))
        _check(tag, nets.critic_old, g, o + "cold_", float(cfg["critic_lr"]))
        if not step:            # critic-only update: the actor does not move
            prev = "p0_actor_" if u == 0 else f"u{u - 1}_actor_"
            assert all(np.array_equal(g[f"{o}actor_{i}"], g[f"{prev}{i}"]) for i in range(len(list(nets.actor.parameters()))))
    assert actor_steps == int(cfg["updates"]) // int(cfg["delay"]) and actor_steps > 0


# ------------------------------------------------------------------------------------------------------------ reference API
class _Box:
    def __init__(self, low, high, shape):
        self.shape = shape
        self.low = np.full(shape, low, np.float32)
        self.high = np.full(shape, high, np.float32)


def _reference():
    from oracle.ref_shim import import_reference, reference_available
    if not reference_available():
        pytest.skip("reference tree not present")
    return import_reference()


def test_ensemble_linear_matches_reference():
    _reference()
    from tianshou.utils.net.common import EnsembleLinear as REL

    from tianshou_b200.utils.net.common import EnsembleLinear
    for bias in (True, False):
        torch.manual_seed(7)
        ref = REL(4, 6, 5, bias=bias)
        torch.manual_seed(7)
        mine = EnsembleLinear(4, 6, 5, bias=bias)
        sr, sm = ref.state_dict(), mine.state_dict()
        assert list(sr.keys()) == list(sm.keys()) and all(torch.equal(sr[k], sm[k]) for k in sr)
        for x in (torch.randn(3, 6), torch.randn(4, 3, 6)):
            y = mine(x)
            assert y.shape == (4, 3, 5) and torch.equal(ref(x), y)


def test_ensemble_critic_construction_matches_reference():
    """test/continuous/test_redq.py:95-109 builds here unchanged and gives [E, B, 1] with the reference's keys and weights."""
    _reference()
    from tianshou.utils.net.common import EnsembleLinear as REL
    from tianshou.utils.net.common import Net as RNet
    from tianshou.utils.net.continuous import ContinuousCritic as RCritic

    from tianshou_b200.utils.net.common import EnsembleLinear, Net
    from tianshou_b200.utils.net.continuous import ContinuousCritic

    def make(NetC, CriticC, EL):
        torch.manual_seed(3)
        net_c = NetC(state_shape=(5,), action_shape=(2,), hidden_sizes=[16, 16], concat=True, linear_layer=lambda x, y: EL(4, x, y))
        return CriticC(preprocess_net=net_c, linear_layer=lambda x, y: EL(4, x, y), flatten_input=False)

    ref, mine = make(RNet, RCritic, REL), make(Net, ContinuousCritic, EnsembleLinear)
    sr, sm = ref.state_dict(), mine.state_dict()
    assert list(sr.keys()) == list(sm.keys()) and all(torch.equal(sr[k], sm[k]) for k in sr)
    obs, act = torch.randn(7, 5), torch.randn(7, 2)
    q = mine(obs, act)
    assert q.shape == (4, 7, 1) and torch.allclose(q, ref(obs, act), rtol=1e-6, atol=1e-6)


def test_redq_policy_forward_matches_reference():
    _reference()
    from gymnasium.spaces import Box as RBox
    from tianshou.algorithm.modelfree.redq import REDQPolicy as RPolicy
    from tianshou.data import Batch as RBatch
    from tianshou.utils.net.common import Net as RNet
    from tianshou.utils.net.continuous import ContinuousActorProbabilistic as RActor
    from tianshou.utils.torch_utils import policy_within_training_step as r_within

    from tianshou_b200.algorithm.modelfree.redq import REDQPolicy
    from tianshou_b200.data import Batch
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.continuous import ContinuousActorProbabilistic
    from tianshou_b200.utils.torch_utils import policy_within_training_step

    def actor(NetC, ActorC):
        torch.manual_seed(2)
        return ActorC(preprocess_net=NetC(state_shape=(5,), hidden_sizes=(8,)), action_shape=(2,), unbounded=True,
                      conditioned_sigma=True)

    rp = RPolicy(actor=actor(RNet, RActor), action_space=RBox(-2.0, 3.0, (2,)))
    mp = REDQPolicy(actor=actor(Net, ContinuousActorProbabilistic), action_space=_Box(-2.0, 3.0, (2,)))
    obs = np.random.default_rng(0).standard_normal((6, 5)).astype(np.float32)
    r, m = rp(RBatch(obs=obs, info={})), mp(Batch(obs=obs, info={}))          # deterministic eval: the mode
    assert torch.equal(r.act, m.act) and torch.equal(r.log_prob, m.log_prob)
    torch.manual_seed(9)
    with r_within(rp):
        r = rp(RBatch(obs=obs, info={}))
    torch.manual_seed(9)
    with policy_within_training_step(mp):
        m = mp(Batch(obs=obs, info={}))
    assert torch.equal(r.act, m.act) and torch.equal(r.log_prob, m.log_prob)
    raw = np.array([[-1.7, 0.2], [0.9, 1.4]], dtype=np.float32)
    np.testing.assert_array_equal(rp.map_action(raw), mp.map_action(raw))


def test_redq_constructor_errors():
    from tianshou_b200.algorithm import REDQ
    with pytest.raises(ValueError, match="target_mode"):
        REDQ(policy=None, policy_optim=None, critic=None, critic_optim=None, target_mode="max")
    for e, m in ((4, 0), (4, 5)):
        with pytest.raises(ValueError, match="subset_size"):
            REDQ(policy=None, policy_optim=None, critic=None, critic_optim=None, ensemble_size=e, subset_size=m)
