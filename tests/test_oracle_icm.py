"""Pin the float64 restatement of the intrinsic curiosity module (oracle/oracle_icm.py) to outputs of the imported reference
(tests/golden/icm_ref_*.npz from oracle/gen_golden_icm.py), its hand-written gradients to float64 autograd of the reference's
loss, and show that the goldens tell apart the two easy misreadings of the reference: a detached phi2, and lr_scale applied to
the learning rate.  CPU only."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from offpolicy_testutil import Discrete
from oracle import oracle_discrete_sac as ods
from oracle import oracle_icm as oic
from ts_testutil import load_golden

VARIANTS = ["dqn_mlp", "dqn_per", "dqn_cnn", "ppo_shared", "a2c_sep"]


def _cfg(g):
    return {k[4:]: (g[k].item() if g[k].ndim == 0 else tuple(g[k].tolist())) for k in g.files if k.startswith("cfg_")}


def icm_module(cfg):
    """The golden's ICM module from tianshou_b200's classes, with its seeded initial weights (float32, on the host)."""
    from tianshou_b200.env.atari.atari_network import DQNet
    from tianshou_b200.utils.net.common import MLP
    from tianshou_b200.utils.net.discrete import IntrinsicCuriosityModule
    A = int(cfg["A"])
    if cfg["kind"] == "cnn":
        fm = DQNet(c=4, h=int(cfg["H"]), w=int(cfg["H"]), action_shape=A, features_only=True)
        feat, F_ = fm.net, int(fm.output_dim)
    else:
        F_ = int(cfg["F"])
        feat = MLP(input_dim=int(cfg["obs"]), output_dim=F_, hidden_sizes=tuple(cfg["feat_hidden"]))
    icm = IntrinsicCuriosityModule(feature_net=feat, feature_dim=F_, action_dim=A, hidden_sizes=tuple(cfg["icm_hidden"]))
    ods.seeded_params(icm, int(cfg["icm_seed"]))
    return icm


def replay(g, **kw):
    cfg = _cfg(g)
    s = oic.ICMState(icm_module(cfg), float(cfg["lr"]))
    on_policy = cfg["algo"] in ("ppo", "a2c")
    res = []
    for u in range(int(cfg["updates"])):
        if u > 0:       # the ICM optimiser's lr of this update (a scheduler steps after each update)
            for pg in s.opt.param_groups:
                pg["lr"] = float(g[f"u{u - 1}_icm_lr"])
        obs, nxt = (g["u0_obs"], g["u0_obs_next"]) if on_policy else (g[f"u{u}_obs"], g[f"u{u}_obs_next"])
        res.append(oic.icm_update(s, obs, g[f"u{u}_act"], nxt, float(cfg["lr_scale"]), float(cfg["reward_scale"]), float(cfg["w"]),
                                  **kw))
    return s, res


def final_error(g, s):
    """The largest deviation of the final ICM parameters from the golden, in units of the bar ``check_final`` uses."""
    lr = float(g["cfg_lr"])
    worst = 0.0
    for i, p in enumerate(s.params):
        got, want = ods.golden_view(p), g[f"icm_pf_{i}"]
        worst = max(worst, float(np.max(np.abs(got - want) / (0.1 * lr + 1e-3 * np.abs(want)))))
    return worst


@pytest.mark.parametrize("variant", VARIANTS)
def test_icm_oracle_matches_reference_run(variant):
    g = load_golden(f"icm_ref_{variant}.npz")
    s, res = replay(g)
    for u, r in enumerate(res):
        for k, key in (("loss", "icm_loss"), ("forward", "icm_forward_loss"), ("inverse", "icm_inverse_loss")):
            np.testing.assert_allclose(r[k], float(g[f"u{u}_{key}"]), rtol=2e-5, atol=1e-7, err_msg=f"update {u} {key}")
        want = g[f"u{u}_intrinsic"]
        np.testing.assert_allclose(r["intrinsic"], want, rtol=2e-5, atol=1e-6 * float(np.abs(want).max()) + 1e-12)
    assert final_error(g, s) <= 1.0
    lr = float(g["cfg_lr"])
    for i, p in enumerate(s.params):
        st = s.opt.state[p]
        m, v = g[f"icm_m_{i}"], g[f"icm_v_{i}"]
        np.testing.assert_allclose(ods.golden_view(st["exp_avg"]), m, rtol=1e-3, atol=1e-3 * float(np.abs(m).max()) + 1e-12)
        np.testing.assert_allclose(ods.golden_view(st["exp_avg_sq"]), v, rtol=2e-3, atol=2e-3 * float(np.abs(v).max()) + 1e-20)
        assert int(st["step"]) == int(g["icm_adam_step"])
    assert lr > 0


def test_scheduler_moves_only_the_icm_lr():
    """a2c_sep puts a linear schedule on the ICM optimiser: its lr falls update by update, the wrapped optimiser's stays."""
    g = load_golden("icm_ref_a2c_sep.npz")
    n = int(g["cfg_updates"])
    icm_lr = [float(g[f"u{u}_icm_lr"]) for u in range(n)]
    assert all(b < a for a, b in zip(icm_lr, icm_lr[1:]))
    assert {float(g[f"u{u}_wrapped_lr"]) for u in range(n)} == {float(g["cfg_lr"])}


@pytest.mark.parametrize("A", [1, 2, 6, 33, 70])
def test_icm_loss_gradients_match_autograd(A):
    """The hand-written gradients at phi2_hat, act_hat and phi2 against float64 autograd of the reference's loss expression."""
    rng = np.random.default_rng(A)
    B, F_, lr_scale, w = 37, 45, 0.7, 0.3
    ph, p2, ah = rng.standard_normal((B, F_)), rng.standard_normal((B, F_)), rng.standard_normal((B, A)) * 3
    act = rng.integers(0, A, B)
    t = [torch.tensor(x, requires_grad=True) for x in (ph, p2, ah)]
    mse = 0.5 * F.mse_loss(t[0], t[1], reduction="none").sum(1)
    inv = F.cross_entropy(t[2], torch.as_tensor(act)).mean()
    loss = ((1 - w) * inv + w * mse.mean()) * lr_scale
    loss.backward()
    r = oic.icm_rows(ph, p2, ah, act, lr_scale, w)
    np.testing.assert_allclose(r["loss"], loss.item(), rtol=1e-13)
    np.testing.assert_allclose(r["mse"], mse.detach().numpy(), rtol=1e-13)
    for got, tt in ((r["d_phi2_hat"], t[0]), (r["d_phi2"], t[1]), (r["d_act_hat"], t[2])):
        np.testing.assert_allclose(got, tt.grad.numpy(), rtol=1e-11, atol=1e-16)


@pytest.mark.parametrize("misreading", ["detach_phi2", "lr_scale_as_lr"])
def test_golden_pins_the_misreadings(misreading):
    """Detaching phi2, or scaling the learning rate instead of the loss, moves dqn_per's final ICM parameters by well over the
    tolerance the oracle meets against the golden."""
    g = load_golden("icm_ref_dqn_per.npz")
    s, _ = replay(g, **{misreading: True})
    assert final_error(g, s) > 5.0


def test_torch_forward_is_the_references():
    """``IntrinsicCuriosityModule.forward`` on the host equals the oracle's rows on the golden's first batch."""
    g = load_golden("icm_ref_dqn_mlp.npz")
    icm = icm_module(_cfg(g))
    with torch.no_grad():
        mse, act_hat = icm(g["u0_obs"], g["u0_act"], g["u0_obs_next"])
    want = g["u0_intrinsic"] / float(g["cfg_reward_scale"])
    np.testing.assert_allclose(mse.numpy(), want, rtol=1e-5, atol=1e-7)
    assert act_hat.shape == (len(g["u0_act"]), int(g["cfg_A"]))
    assert Discrete(3).n == 3
