"""Pin the float64 restatement of imitation learning (oracle/oracle_imitation.py) to outputs of the imported reference
(tests/golden/il_ref_*.npz from oracle/gen_golden_imitation.py), its hand-written gradients to float64 autograd of the reference
expressions, the goldens' ``state_dict()`` keys and optimiser ids to the tianshou_b200 construction, and ``ImitationPolicy.forward``
on the CPU.  CPU only."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import oracle_discrete_sac as ods
from oracle import oracle_imitation as oim
from offpolicy_testutil import Box, Discrete
from oracle_testutil import check_final
from ts_testutil import load_golden

VARIANTS = ["cont", "d4rl", "disc_sm", "disc_logits", "cnn", "per"]


def _cfg(g):
    return {k[4:]: (g[k].item() if g[k].ndim == 0 else tuple(g[k].tolist())) for k in g.files if k.startswith("cfg_")}


def b200_actor(g):
    """The golden's actor built from tianshou_b200's modules, with the golden's initial weights (float32)."""
    from tianshou_b200.env.atari.atari_network import DQNet
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.continuous import ContinuousActorDeterministic
    from tianshou_b200.utils.net.discrete import DiscreteActor
    cfg = _cfg(g)
    actor = oim.make_actor(cfg, (Net, ContinuousActorDeterministic, DiscreteActor, DQNet))
    if cfg["compact"]:
        ods.seeded_params(actor, int(cfg["init_seed"]))
    else:
        with torch.no_grad():
            for i, p in enumerate(actor.parameters()):
                p.copy_(torch.as_tensor(g[f"p0_{i}"]).reshape(p.shape))
    return actor


def b200_policy(g, actor):
    from tianshou_b200.algorithm.imitation import ImitationPolicy
    if str(g["cfg_kind"]) == "cont":
        m = float(g["cfg_max_action"])
        return ImitationPolicy(actor=actor, action_space=Box(int(g["cfg_A"]), m), action_scaling=True)
    return ImitationPolicy(actor=actor, action_space=Discrete(int(g["cfg_A"])))


@pytest.mark.parametrize("variant", VARIANTS)
def test_imitation_oracle_matches_reference_run(variant):
    g = load_golden(f"il_ref_{variant}.npz")
    kind = str(g["cfg_kind"])
    actor = b200_actor(g)
    policy = b200_policy(g, actor)
    # the construction's module names are the reference's: policy.*, then the one optimiser over every policy parameter
    assert ["policy." + k for k in policy.state_dict()] + ["_optimizers"] == [str(k) for k in g["state_dict_keys"]]
    assert g["optim_param_ids"].tolist() == list(range(len(list(policy.parameters()))))
    s = oim.ImitationState(actor, float(g["cfg_lr"]))
    softmax = bool(g["cfg_softmax"]) if "cfg_softmax" in g.files else False
    outside = False
    for u in range(int(g["cfg_updates"])):
        r = oim.imitation_update(s, g[f"u{u}_obs"], g[f"u{u}_act"], kind, float(g["cfg_max_action"]) if kind == "cont" else 1.0,
                                 softmax)
        np.testing.assert_allclose(r["loss"], float(g[f"u{u}_loss"]), rtol=1e-5, atol=1e-7)
        if kind == "cont":
            outside |= bool((np.abs(g[f"u{u}_act"]) > float(g["cfg_max_action"])).any())
    if variant == "cont":
        assert outside, "the cont golden must hold actions outside +-max_action"
    check_final(g, s.params, s.opt, [])
    if variant == "per":        # the tree holds (|w| + eps) ** alpha of the last weights written back
        u = int(g["cfg_updates"]) - 1
        idx, w = g[f"u{u}_indices"], g[f"u{u}_prio"]
        last = {int(i): k for k, i in enumerate(idx)}
        k = np.array(list(last.values()))
        want = (np.abs(w[k]) + np.finfo(np.float32).eps) ** float(g["cfg_alpha"])
        np.testing.assert_allclose(g["prio_leaves"][list(last)], want, rtol=1e-12)


def test_double_softmax_is_pinned():
    """Without the reference's log_softmax of probabilities, disc_sm's loss moves by 100 times the tolerance the oracle meets
    against the golden: the golden pins the double softmax."""
    g = load_golden("il_ref_disc_sm.npz")
    s = oim.ImitationState(b200_actor(g), float(g["cfg_lr"]))
    r = oim.imitation_update(s, g["u0_obs"], g["u0_act"], "disc", softmax_output=False)
    assert abs(r["loss"] - float(g["u0_loss"])) > 100 * 1e-5 * float(g["u0_loss"])


@pytest.mark.parametrize("A", [1, 2, 6, 33, 70])
def test_rows_gradients_match_autograd(A):
    rng = np.random.default_rng(A)
    B, m = 37, 2.0
    z = rng.standard_normal((B, A)) * 3
    z[:4] *= 40.0
    act = rng.standard_normal((B, A)) * 3
    zt = torch.tensor(z, requires_grad=True)
    loss = F.mse_loss(m * torch.tanh(zt), torch.tensor(act))
    loss.backward()
    got, dz = oim.mse_rows(z, act, m)
    np.testing.assert_allclose(got, loss.item(), rtol=1e-13)
    np.testing.assert_allclose(dz, zt.grad.numpy(), rtol=1e-11, atol=1e-15)   # saturated tanh: 1 - t^2 is 0 or a few ulps
    a = rng.integers(0, A, B)
    for softmax in (False, True):
        zt = torch.tensor(z, requires_grad=True)
        y = F.softmax(zt, -1) if softmax else zt
        loss = F.nll_loss(F.log_softmax(y, -1), torch.as_tensor(a))
        loss.backward()
        got, dz, rows = oim.nll_rows(z, a, softmax)
        np.testing.assert_allclose(got, loss.item(), rtol=1e-12)
        np.testing.assert_allclose(dz, zt.grad.numpy(), rtol=1e-10, atol=1e-16)
        assert rows.shape == (B,)


def test_policy_forward_on_the_host():
    """``ImitationPolicy.forward``: discrete, (logits, arg-max); continuous, the actor's output as both."""
    from tianshou_b200.data import Batch
    g = load_golden("il_ref_disc_logits.npz")
    policy = b200_policy(g, b200_actor(g))
    obs = g["u0_obs"][:5]
    with torch.no_grad():
        out = policy(Batch(obs=obs, info=Batch()))
        logits, _ = policy.actor(obs)
    assert torch.equal(out.logits, logits) and torch.equal(out.act, logits.argmax(1))
    g = load_golden("il_ref_d4rl.npz")
    policy = b200_policy(g, b200_actor(g))
    with torch.no_grad():
        out = policy(Batch(obs=g["u0_obs"][:5], info=Batch()))
    assert torch.equal(out.act, out.logits) and out.act.shape == (5, 6) and float(out.act.abs().max()) <= 1.0
