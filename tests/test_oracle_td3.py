"""The eager TD3 / TD3+BC restatement (oracle/oracle_td3.py) against outputs of the imported reference (tests/golden/td3_ref_*.npz
from oracle/gen_golden_td3.py), and the deterministic actor, policy and exploration noise against the reference itself when it
is present.  CPU only."""
import numpy as np
import pytest
import torch

from ts_testutil import load_golden, record_parity

VARIANTS = ["mujoco", "per_nstep", "bc", "bc_freq1"]


def _cfg(g):
    return {k[4:]: g[k] for k in g.files if k.startswith("cfg_")}


def _load(mod, g, prefix):
    with torch.no_grad():
        for i, p in enumerate(mod.parameters()):
            p.copy_(torch.as_tensor(g[f"{prefix}{i}"]).reshape(p.shape))


def _check(tag, mod, g, prefix, lr):
    for i, p in enumerate(mod.parameters()):
        record_parity(f"{tag}/{prefix}{i}", p.detach().numpy(), g[f"{prefix}{i}"], rtol=1e-4, atol=1e-3 * lr)


def oracle_buffer(g):
    """The arrays ``oracle_td3.nstep_targets`` reads, for the single buffer of a golden."""
    d = {k: g["buf_" + k] for k in ("obs", "act", "rew", "done", "terminated", "obs_next")}
    size, n = len(g["buf_obs"]), int(g["buf_len"])
    last = (int(g["buf_insertion_idx"]) - 1) % n
    d.update(offset=np.array([0, size]), last_index=g["buf_last_index"], lengths=np.array([n]),
             unfinished=[last] if not d["done"][last] else [])
    return d


@pytest.mark.parametrize("variant", VARIANTS)
def test_oracle_matches_reference(variant):
    from oracle.oracle_td3 import Td3Nets, td3_update
    g = load_golden(f"td3_ref_{variant}.npz")
    cfg = _cfg(g)
    O, A, H = int(cfg["obs"]), int(cfg["act"]), tuple(int(x) for x in cfg["hidden"])
    nets = Td3Nets(O, A, H, float(cfg["max_action"]))
    _load(nets.a, g, "p0_actor_"); _load(nets.c[0], g, "p0_c1_"); _load(nets.c[1], g, "p0_c2_")
    nets.a_old.load_state_dict(nets.a.state_dict())
    for k in range(2):
        nets.c_old[k].load_state_dict(nets.c[k].state_dict())
    lr, c2_lr = float(cfg["critic_lr"]), float(cfg["critic2_lr"]) if bool(cfg["critic2"]) else float(cfg["critic_lr"])
    opts = [torch.optim.Adam(nets.a.parameters(), lr=float(cfg["actor_lr"])), torch.optim.Adam(nets.c[0].parameters(), lr=lr),
            torch.optim.Adam(nets.c[1].parameters(), lr=c2_lr)]
    buf = oracle_buffer(g)
    bc = float(cfg["alpha"]) if str(cfg["algo"]) == "bc" else None
    last = 0.0
    actor_steps = 0
    for u in range(int(cfg["updates"])):
        o, tag = f"u{u}_", f"oracle_td3/{variant}/u{u}"
        w = torch.as_tensor(g[o + "is_weight"]).float() if bool(cfg["per"]) else None
        torch.manual_seed(100 + u)
        step = u % int(cfg["freq"]) == 0
        r = td3_update(nets, opts, buf, g[o + "indices"], lambda shape: torch.randn(shape), gamma=float(cfg["gamma"]),
                       n_step=int(cfg["n_step"]), tau=float(cfg["tau"]), policy_noise=float(cfg["policy_noise"]),
                       noise_clip=float(cfg["noise_clip"]), actor_step=step, is_weight=w, bc_alpha=bc)
        if step:
            last, actor_steps = r["actor_loss"], actor_steps + 1
        record_parity(f"{tag}/losses", np.array([last, r["critic1_loss"], r["critic2_loss"]]), g[o + "losses"], rtol=1e-5, atol=1e-6)
        assert np.array_equal(torch.get_rng_state().numpy(), g[o + "torch_rng"]), "CPU generator differs from the reference's"
        _check(tag, nets.a, g, o + "actor_", float(cfg["actor_lr"]))
        _check(tag, nets.c[0], g, o + "c1_", lr); _check(tag, nets.c[1], g, o + "c2_", c2_lr)
        _check(tag, nets.c_old[0], g, o + "c1old_", lr); _check(tag, nets.c_old[1], g, o + "c2old_", c2_lr)
        _check(tag, nets.a_old, g, o + "aold_", float(cfg["actor_lr"]))
        if u > 0 and not step:       # critic-only update: the lagged networks do not move
            for k in ("c1old_", "c2old_", "aold_"):
                assert all(np.array_equal(g[f"{o}{k}{i}"], g[f"u{u - 1}_{k}{i}"]) for i in range(len(list(nets.a.parameters()))))
    assert 0 < actor_steps < int(cfg["updates"]) or int(cfg["freq"]) == 1


def test_per_nstep_target_actions_leave_the_action_bounds():
    """With noise_clip=0 and max_action=2 the smoothed target actions are not clamped: some leave [-2, 2], as in the reference."""
    from oracle.oracle_td3 import Td3Nets
    g = load_golden("td3_ref_per_nstep.npz")
    cfg = _cfg(g)
    nets = Td3Nets(int(cfg["obs"]), int(cfg["act"]), tuple(int(x) for x in cfg["hidden"]), float(cfg["max_action"]))
    _load(nets.a, g, "p0_actor_")
    torch.manual_seed(100)
    with torch.no_grad():
        a = nets.pi(torch.as_tensor(g["buf_obs_next"])) + torch.randn(len(g["buf_obs_next"]), int(cfg["act"])) * float(cfg["policy_noise"])
    assert float(cfg["noise_clip"]) == 0.0 and float(a.abs().max()) > float(cfg["max_action"])


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


def test_deterministic_actor_matches_reference():
    _reference()
    from tianshou.utils.net.common import Net as RNet
    from tianshou.utils.net.continuous import ContinuousActorDeterministic as RActor

    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.continuous import ContinuousActorDeterministic
    for hidden, m in (((), 1.0), ((12,), 2.5)):
        torch.manual_seed(4)
        ref = RActor(preprocess_net=RNet(state_shape=(7,), hidden_sizes=(16, 16)), action_shape=(3,), hidden_sizes=hidden, max_action=m)
        torch.manual_seed(4)
        mine = ContinuousActorDeterministic(preprocess_net=Net(state_shape=(7,), hidden_sizes=(16, 16)), action_shape=(3,),
                                            hidden_sizes=hidden, max_action=m)
        sr, sm = ref.state_dict(), mine.state_dict()
        assert list(sr.keys()) == list(sm.keys())
        assert all(torch.equal(sr[k], sm[k]) for k in sr)
        obs = torch.randn(5, 7)
        (a_r, _), (a_m, _) = ref(obs), mine(obs)
        assert torch.equal(a_r, a_m) and mine.get_output_dim() == 3 and float(a_m.abs().max()) <= m


def test_deterministic_policy_matches_reference():
    _reference()
    from gymnasium.spaces import Box as RBox
    from tianshou.algorithm.modelfree.ddpg import ContinuousDeterministicPolicy as RPolicy
    from tianshou.data import Batch as RBatch
    from tianshou.exploration import GaussianNoise as RGauss
    from tianshou.utils.net.common import Net as RNet
    from tianshou.utils.net.continuous import ContinuousActorDeterministic as RActor

    from tianshou_b200.algorithm.modelfree.ddpg import ContinuousDeterministicPolicy
    from tianshou_b200.data import Batch
    from tianshou_b200.exploration import GaussianNoise
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.continuous import ContinuousActorDeterministic
    torch.manual_seed(1)
    ra = RActor(preprocess_net=RNet(state_shape=(5,), hidden_sizes=(8,)), action_shape=(2,), max_action=1.0)
    torch.manual_seed(1)
    ma = ContinuousActorDeterministic(preprocess_net=Net(state_shape=(5,), hidden_sizes=(8,)), action_shape=(2,), max_action=1.0)
    rp = RPolicy(actor=ra, exploration_noise="default", action_space=RBox(-2.0, 3.0, (2,)))
    mp = ContinuousDeterministicPolicy(actor=ma, exploration_noise="default", action_space=_Box(-2.0, 3.0, (2,)))
    assert isinstance(rp.exploration_noise, RGauss) and isinstance(mp.exploration_noise, GaussianNoise)
    obs = np.random.default_rng(0).standard_normal((6, 5)).astype(np.float32)
    r_act, m_act = rp(RBatch(obs=obs, info={})).act, mp(Batch(obs=obs, info={})).act
    assert torch.equal(r_act, m_act)
    with torch.no_grad():
        r_old, m_old = rp(RBatch(obs=obs, info={}), model=ra).act, mp(Batch(obs=obs, info={}), model=ma).act
    assert torch.equal(r_old, m_old)
    raw = np.array([[-1.7, 0.2], [0.9, 1.4]], dtype=np.float32)             # map_action clips to [-1, 1], then scales
    np.testing.assert_array_equal(rp.map_action(raw), mp.map_action(raw))
    np.random.seed(3)
    r_noisy = rp.add_exploration_noise(raw.copy(), None)
    np.random.seed(3)
    m_noisy = mp.add_exploration_noise(raw.copy(), None)
    np.testing.assert_array_equal(r_noisy, m_noisy)
    mp.set_exploration_noise(None)
    assert mp.add_exploration_noise(raw, None) is raw
    with pytest.warns(UserWarning, match="max_action"):
        ContinuousDeterministicPolicy(actor=ContinuousActorDeterministic(preprocess_net=Net(state_shape=(5,), hidden_sizes=(8,)),
                                                                         action_shape=(2,), max_action=2.0),
                                      action_space=_Box(-2.0, 2.0, (2,)))


def test_exploration_noise_matches_reference():
    _reference()
    from tianshou.exploration import GaussianNoise as RGauss
    from tianshou.exploration import OUNoise as ROU

    from tianshou_b200.exploration import BaseNoise, GaussianNoise, OUNoise
    for make_r, make_m in ((lambda: RGauss(0.3, 0.7), lambda: GaussianNoise(0.3, 0.7)),
                           (lambda: ROU(), lambda: OUNoise()), (lambda: ROU(0.1, 0.5, 0.3, 0.05, x0=0.2), lambda: OUNoise(0.1, 0.5, 0.3, 0.05, x0=0.2))):
        r, m = make_r(), make_m()
        assert isinstance(m, BaseNoise)
        for seed in (0, 1):
            np.random.seed(seed)
            a = [r((4, 3)) for _ in range(3)] + [r((2,))]
            np.random.seed(seed)
            b = [m((4, 3)) for _ in range(3)] + [m((2,))]
            for x, y in zip(a, b, strict=True):
                np.testing.assert_array_equal(x, y)
            r.reset(); m.reset()
    with pytest.raises(AssertionError):
        GaussianNoise(sigma=-1.0)
