"""Pin the eager restatement of discrete SAC (oracle/oracle_discrete_sac.py) to outputs of the imported reference
(tests/golden/dsac_ref_{mlp,auto,cnn}.npz from oracle/gen_golden_discrete_sac.py), and the host-side draw order: the
uniform buffer's index streams and the two discarded Categorical draws per update.  CPU only."""
import copy

import numpy as np
import pytest
import torch

from oracle import oracle_discrete_sac as ods
from offpolicy_testutil import load_params
from ts_testutil import load_golden

VARIANTS = ["mlp", "auto", "cnn"]


def _init(mods, g):
    """The golden's initial weights: stored tensors, or (compact goldens) the seeded recipe it names."""
    for k, (m, pfx) in enumerate(zip(mods, ("p0_actor_", "p0_c1_", "p0_c2_"), strict=True)):
        if bool(g["cfg_compact"]):
            ods.seeded_params(m, int(g["cfg_init_seed"]) + k)
        else:
            load_params(m, g, pfx)


def _close(mod, g, prefix, lr, what):
    view = ods.golden_view if bool(g["cfg_compact"]) else (lambda t: t.detach().numpy())
    for i, p in enumerate(mod.parameters()):
        np.testing.assert_allclose(view(p), g[f"{prefix}{i}"], rtol=1e-3, atol=0.1 * lr, err_msg=f"{what} {prefix}{i}")


def build_oracle(g, device="cpu"):
    """Oracle networks, optimisers, alpha and buffer view of a golden file, with its initial weights."""
    A = int(g["cfg_A"])
    if str(g["cfg_kind"]) == "mlp":
        O, H = int(g["cfg_obs"]), tuple(int(x) for x in g["cfg_hidden"])
        mk = lambda: ods.mlp_head_net(O, H, A)
    else:
        mk = lambda: ods.cnn_head_net(4, int(g["cfg_H"]), int(g["cfg_W"]), int(g["cfg_feat"]), A)
    actor, c1, c2 = mk(), mk(), mk()
    _init((actor, c1, c2), g)
    actor, c1, c2 = (m.to(device) for m in (actor, c1, c2))
    critics = [c1, c2]
    olds = [copy.deepcopy(c) for c in critics]
    alr, clr = float(g["cfg_actor_lr"]), float(g["cfg_critic_lr"])
    opts = [torch.optim.Adam(actor.parameters(), lr=alr)] + [torch.optim.Adam(c.parameters(), lr=clr) for c in critics]
    if bool(g["cfg_auto"]):
        la = torch.nn.Parameter(torch.tensor(0.0, device=device))
        alpha = ods.AutoAlphaState(la, float(0.98 * np.log(A)), torch.optim.Adam([la], lr=float(g["cfg_alpha_lr"])))
    else:
        alpha = float(g["cfg_alpha"])
    E, cap = int(g["cfg_E"]), int(g["cfg_cap"])
    buf = dict(obs=g["buf_obs"], act=g["buf_act"], rew=g["buf_rew"], done=g["buf_done"], terminated=g["buf_terminated"],
               offset=np.arange(E + 1) * cap, last_index=g["meta_last_index"], lengths=g["meta_lengths"])
    stored_next = "buf_obs_next" in g
    if stored_next:
        buf["obs_next"] = g["buf_obs_next"]
        obs_of = ods.flat_obs(buf["obs"], device)
    else:
        obs_of = ods.frame_obs(buf, 4, 255.0, device)
    return actor, critics, olds, opts, alpha, buf, obs_of, stored_next


@pytest.mark.parametrize("variant", VARIANTS)
def test_discrete_sac_oracle_matches_reference_run(variant):
    g = load_golden(f"dsac_ref_{variant}.npz")
    actor, critics, olds, opts, alpha, buf, obs_of, stored_next = build_oracle(g)
    per = bool(g["cfg_per"])
    alr, clr = float(g["cfg_actor_lr"]), float(g["cfg_critic_lr"])
    for u in range(int(g["cfg_updates"])):
        o = f"u{u}_"
        torch.manual_seed(100 + u)
        res = ods.discrete_sac_update(actor, critics, olds, opts, obs_of, buf, g[o + "indices"], g[o + "is_weight"] if per else None,
                                      float(g["cfg_gamma"]), int(g["cfg_n_step"]), alpha, float(g["cfg_tau"]), stored_next)
        # the reference drew exactly two Categorical samples of the same shapes from the same generator
        assert torch.equal(torch.get_rng_state(), torch.from_numpy(g[o + "torch_rng"])), "torch generator out of step"
        np.testing.assert_allclose(res["returns"], g[o + "returns"].reshape(-1), rtol=1e-5, atol=1e-5)
        np.testing.assert_allclose(res["weight"], g[o + "weight"], rtol=1e-4, atol=1e-5)
        np.testing.assert_allclose(res["losses"], g[o + "losses"], rtol=1e-5, atol=1e-6)
        np.testing.assert_allclose(res["alpha"], float(g[o + "alpha"]), rtol=1e-6)
        if bool(g["cfg_auto"]):
            np.testing.assert_allclose(res["alpha_loss"], float(g[o + "alpha_loss"]), rtol=1e-5, atol=1e-7)
            np.testing.assert_allclose(alpha.log_alpha.item(), float(g[o + "log_alpha"]), rtol=0, atol=1e-7)
        else:
            assert res["alpha_loss"] is None and np.isnan(g[o + "alpha_loss"])
        if o + "actor_0" not in g:
            continue
        _close(actor, g, o + "actor_", alr, "actor")
        for k in range(2):
            _close(critics[k], g, o + f"c{k + 1}_", clr, "critic")
            _close(olds[k], g, o + f"c{k + 1}old_", clr, "lagged critic")


def test_uniform_index_draws_match_reference():
    """The uniform buffer's per-environment RandomState streams: tianshou_b200's VectorReplayBuffer, filled with the same
    rollout, draws the reference's indices update after update."""
    from tianshou_b200.data import Batch, VectorReplayBuffer
    g = load_golden("dsac_ref_auto.npz")
    E, cap = int(g["cfg_E"]), int(g["cfg_cap"])
    buf = VectorReplayBuffer(E * cap, E)
    for i in range(int(g["cfg_steps"])):
        buf.add(Batch(**{k: g[f"roll{i}_{k}"] for k in ("obs", "act", "rew", "terminated", "truncated", "obs_next")}),
                buffer_ids=np.arange(E))
    for u in range(int(g["cfg_updates"])):
        np.random.seed(500 + u)
        assert np.array_equal(buf.sample_indices(int(g["cfg_bs"])), g[f"u{u}_indices"])


def test_discarded_draws_are_two_categorical_samples():
    """The restatement's only generator use per update is two ``Categorical(logits).sample()`` calls of [B, A] probabilities:
    replaying them as ``torch.multinomial(p, 1, True)`` (what ``Categorical.sample`` runs, and what the device update draws)
    from the same seed leaves the generator in the golden state."""
    for variant in VARIANTS:
        g = load_golden(f"dsac_ref_{variant}.npz")
        B, A = int(g["cfg_bs"]), int(g["cfg_A"])
        for u in range(int(g["cfg_updates"])):
            torch.manual_seed(100 + u)
            p = torch.full((B, A), 1.0 / A)
            torch.multinomial(p, 1, True)
            torch.multinomial(p, 1, True)
            assert torch.equal(torch.get_rng_state(), torch.from_numpy(g[f"u{u}_torch_rng"])), (variant, u)
