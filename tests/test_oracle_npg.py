"""Pin the eager-PyTorch restatement of NPG / TRPO (oracle/oracle_npg.py) to outputs of the imported reference
(tests/golden/npg_ref_*.npz, trpo_ref_*.npz).  CPU only.  The preprocessing (returns, advantages, logp_old) is taken from the
goldens: the update loop is what the restatement covers."""
import numpy as np
import pytest
import torch

from oracle import oracle_npg as on
from ts_testutil import load_golden

VARIANTS = ["npg_ref_gauss", "trpo_ref_gauss", "npg_ref_mb", "trpo_ref_mb", "npg_ref_cat", "trpo_ref_cat", "trpo_ref_backtrack",
            "trpo_ref_fail", "trpo_ref_nobt"]


@pytest.mark.parametrize("variant", VARIANTS)
def test_npg_trpo_oracle_matches_reference_run(variant):
    g = load_golden(f"{variant}.npz")
    cat, O, A = bool(g["cfg_categorical"]), int(g["cfg_obs"]), int(g["cfg_act"])
    act_fn = torch.nn.ReLU if cat else torch.nn.Tanh
    actor = on.Actor(O, A, (64, 64), act_fn, cat)
    critic = on.critic_net(O, (64, 64), act_fn)
    with torch.no_grad():
        for mod, tag in ((actor, "actor"), (critic, "critic")):
            for i, p in enumerate(mod.parameters()):
                p.copy_(torch.as_tensor(g[f"p0_{tag}_{i}"]).reshape(p.shape))
    opt = torch.optim.Adam(critic.parameters(), lr=float(g["cfg_lr"]))
    kw = {k[3:]: g[k].item() for k in g.files if k.startswith("kw_") and k[3:] not in ("return_scaling", "advantage_normalization")}
    for k in ("optim_critic_iters", "max_backtracks"):
        if k in kw:
            kw[k] = int(kw[k])
    kw.setdefault("optim_critic_iters", 5)
    trpo = bool(g["cfg_trpo"])
    bs = int(g["cfg_bs"])
    for u in range(2):
        o = f"u{u}_"
        N = g[o + "adv"].shape[0]
        data = {"obs": torch.as_tensor(g[o + "buf_obs"][:N], dtype=torch.float32),
                "act": torch.as_tensor(g[o + "buf_act"][:N]).long() if cat else torch.as_tensor(g[o + "buf_act"][:N], dtype=torch.float32),
                **{k: torch.as_tensor(g[o + k]) for k in ("adv", "returns", "logp_old")}}
        with torch.no_grad():      # logp_old at the restatement's own parameters (npg.py:131-133), as the reference does
            data["logp_old"] = actor.dist(data["obs"]).log_prob(data["act"])
        np.random.seed(int(g[o + "np_seed"]))
        perms = [np.random.permutation(N) for _ in range(int(g["cfg_repeat"]))]
        res = on.update(actor, critic, opt, data, perms, None if bs < 0 else bs, trpo=trpo, **kw)
        assert res["warnings"] == list(g[o + "warnings"])
        assert res["cg_iters"] == list(g[o + "cg_iters"])
        # fp32 conjugate gradients whose vector updates round differently: the step size and the log-std after a TRPO step
        # (up to 1.5 along the natural direction) differ from the reference at the 1e-4 .. 4e-3 level
        for k in ("actor_loss", "vf_loss", "kl") + (("step_size",) if trpo else ()):
            np.testing.assert_allclose(res[k], g[o + k], rtol=1e-3, atol=1e-6, err_msg=f"{variant} u{u} {k}")
        for mod, tag in ((actor, "actor"), (critic, "critic")):
            for i, p in enumerate(mod.parameters()):
                ref = g[f"{o}{tag}_{i}"]
                np.testing.assert_allclose(p.detach().numpy(), ref.reshape(p.shape), rtol=2e-3, atol=1e-4 + 1e-3 * np.abs(ref).max(),
                                           err_msg=f"{variant} u{u} {tag}_{i}")
