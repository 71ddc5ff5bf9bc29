"""Pin the restatement of discrete CRR (oracle/oracle_discrete_crr.py: float64 numpy target, losses and gradients under plain
torch networks) to outputs of the imported reference (tests/golden/dcrr_ref_{mlp,cnn,sep}.npz from
oracle/gen_golden_discrete_crr.py), its hand-written gradients to float64 autograd of the reference expressions, and the host
logic of ``DiscreteCRR`` that needs no device.  CPU only."""
import numpy as np
import pytest
import torch
from torch.distributions import Categorical

from oracle import oracle_discrete_crr as odc
from offpolicy_testutil import Discrete
from oracle_testutil import check_final, oracle_setup
from ts_testutil import load_golden

VARIANTS = ["mlp", "cnn", "sep"]


@pytest.mark.parametrize("variant", VARIANTS)
def test_discrete_crr_oracle_matches_reference_run(variant):
    g = load_golden(f"dcrr_ref_{variant}.npz")
    A, freq = int(g["cfg_A"]), int(g["cfg_freq"])
    nets, buf, obs_of = oracle_setup(g, (A, A))
    s = odc.CrrState(nets, float(g["cfg_lr"]), freq)
    saturated = False
    for u in range(int(g["cfg_updates"])):
        r = odc.discrete_crr_update(s, obs_of, buf, g[f"u{u}_indices"], float(g["cfg_gamma"]), str(g["cfg_mode"]), float(g["cfg_beta"]),
                                    float(g["cfg_bound"]), float(g["cfg_min_q_weight"]))
        np.testing.assert_allclose(r["losses"], g[f"u{u}_losses"], rtol=1e-5, atol=1e-6)
        saturated |= bool((r["coef"] == float(g["cfg_bound"])).any() and (r["coef"] < float(g["cfg_bound"])).any())
    assert s.iter == int(g["iter"])
    if variant == "mlp":
        assert saturated, "the exp golden must have rows on both sides of the clamp"
    # actor_old's parameters (trunk, last) then critic_old's (its own copy of the trunk, last)
    lagged = [*s.old.head_a_parameters(), *s.old.head_b_parameters()] if freq > 0 else []
    check_final(g, list(nets.parameters()), s.opt, lagged)
    if freq > 0:
        assert any(not torch.equal(a, b) for a, b in zip(s.old.parameters(), nets.parameters()))


def _reference_loss(q, z, act, qo, zo, rew, done, gamma, mode, beta, bound, w):
    """discrete_crr.py:131-158 on float64 tensors."""
    qa = q.gather(1, act.unsqueeze(1))
    with torch.no_grad():
        eq = (qo * Categorical(logits=zo).probs).sum(-1, keepdim=True)
        eq[done > 0] = 0.0
        target = rew.unsqueeze(1) + gamma * eq
    critic = 0.5 * torch.nn.functional.mse_loss(qa, target)
    dist = Categorical(logits=z)
    adv = qa - (q * dist.probs).sum(-1, keepdim=True)
    if mode == "binary":
        coef = (adv > 0).double()
    elif mode == "exp":
        coef = (adv / beta).exp().clamp(0, bound)
    else:
        coef = 1.0
    actor = (-dist.log_prob(act) * coef).mean()          # [B] * [B, 1]: the reference's [B, B] broadcast
    cql = (q.logsumexp(1) - qa.squeeze(-1)).mean()
    return actor + critic + w * cql, actor, critic, cql


@pytest.mark.parametrize("mode", ["exp", "binary", "all"])
def test_rows_gradients_match_autograd(mode):
    """The gradient is autograd's, not the paper's: in exp mode the coefficient carries gradient where the clamp passes."""
    rng = np.random.default_rng(3)
    B, A, gamma, beta, bound, w = 41, 6, 0.9, 0.7, 2.0, 3.0
    q, z = rng.standard_normal((B, A)) * 2, rng.standard_normal((B, A)) * 3
    qo, zo = rng.standard_normal((B, A)) * 2, rng.standard_normal((B, A)) * 3
    act = rng.integers(0, A, B)
    rew, done = rng.standard_normal(B), (rng.random(B) < 0.3).astype(np.float64)
    r = odc.crr_rows(q, z, act, qo, zo, rew, done, gamma, mode, beta, bound, w)
    qt, zt = torch.tensor(q, requires_grad=True), torch.tensor(z, requires_grad=True)
    loss, actor, critic, cql = _reference_loss(qt, zt, torch.as_tensor(act), torch.tensor(qo), torch.tensor(zo), torch.tensor(rew),
                                               torch.tensor(done), gamma, mode, beta, bound, w)
    loss.backward()
    np.testing.assert_allclose(r["losses"], [loss.item(), actor.item(), critic.item(), cql.item()], rtol=1e-12)
    np.testing.assert_allclose(r["dq"], qt.grad.numpy(), rtol=1e-11, atol=1e-14)
    np.testing.assert_allclose(r["dlogits"], zt.grad.numpy(), rtol=1e-11, atol=1e-14)
    if mode == "exp":
        assert (r["coef"] == bound).any() and (r["coef"] < bound).any() and (r["adv"] > 0).any() and (r["adv"] < 0).any()


def test_mode_and_gamma_are_checked_on_the_host():
    """Checked before any network is looked at, so no device is needed."""
    from tianshou_b200.algorithm import AdamOptimizerFactory, DiscreteActorPolicy, DiscreteCRR
    from tianshou_b200.algorithm.imitation.discrete_crr import DiscountedReturnComputation
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.discrete import DiscreteActor, DiscreteCritic

    trunk = Net(state_shape=(4,), hidden_sizes=(16,))
    policy = DiscreteActorPolicy(actor=DiscreteActor(preprocess_net=trunk, action_shape=3, softmax_output=False), action_space=Discrete(3))
    critic = DiscreteCritic(preprocess_net=trunk, last_size=3)
    with pytest.raises(ValueError, match="policy_improvement_mode"):
        DiscreteCRR(policy=policy, critic=critic, optim=AdamOptimizerFactory(lr=1e-3), policy_improvement_mode="softmax")
    with pytest.raises(AssertionError):
        DiscreteCRR(policy=policy, critic=critic, optim=AdamOptimizerFactory(lr=1e-3), gamma=1.5)
    d = DiscountedReturnComputation(gamma=0.9, return_standardization=True)
    assert d.gamma == 0.9 and d.return_standardization
