"""The eager CQL restatement (oracle/oracle_cql.py) against outputs of the imported reference (tests/golden/cql_ref_*.npz from
oracle/gen_golden_cql.py), on the CPU: the positional calibration store, and three updates per golden -- losses, the Lagrange
multiplier, alpha, every parameter and the torch CPU generator after each update."""
import numpy as np
import pytest
import torch

from ts_testutil import load_golden, record_parity

VARIANTS = ["d4rl", "nolag", "wrap"]


def _load(mods, g, prefix):
    params = [p for m in mods for p in m.parameters()]
    with torch.no_grad():
        for i, p in enumerate(params):
            p.copy_(torch.as_tensor(g[f"{prefix}{i}"]).reshape(p.shape))


def _check(tag, mods, g, prefix, lr):
    params = [p for m in mods for p in m.parameters()]
    for i, p in enumerate(params):
        record_parity(f"{tag}/{prefix}{i}", p.detach().numpy(), g[f"{prefix}{i}"], rtol=1e-4, atol=1e-3 * lr)


@pytest.mark.parametrize("variant", VARIANTS)
def test_calibration_returns_are_stored_positionally(variant):
    from oracle.oracle_cql import calibration_returns, sample_all_order
    g = load_golden(f"cql_ref_{variant}.npz")
    if not bool(g["cfg_calibrated"]):
        pytest.skip("uncalibrated: process_buffer adds no key")
    size, ins = int(g["buf_size"]), int(g["buf_insertion_idx"])
    got = calibration_returns(g["buf_rew"], g["buf_terminated"], g["buf_truncated"], g["buf_done"], size, ins, float(g["cfg_gamma"]))
    np.testing.assert_allclose(got, g["calibration_returns"], rtol=1e-12, atol=1e-12)
    order = sample_all_order(size, ins)
    if variant == "wrap":
        # the wrapped buffer: slot i holds the return of the i-th OLDEST transition, not of slot i itself
        assert ins > 0 and not np.array_equal(order, np.arange(size))
        per_slot = np.empty(size)
        per_slot[order] = got
        assert not np.allclose(per_slot, got)
    else:
        assert np.array_equal(order, np.arange(size))


@pytest.mark.parametrize("variant", VARIANTS)
def test_oracle_matches_reference(variant):
    from oracle.oracle_cql import cql_nets, cql_update
    from oracle.oracle_discrete_sac import AutoAlphaState
    g = load_golden(f"cql_ref_{variant}.npz")
    cfg = {k[4:]: g[k] for k in g.files if k.startswith("cfg_")}
    O, A, H = int(cfg["obs"]), int(cfg["act"]), tuple(int(x) for x in cfg["hidden"])
    nets = cql_nets(O, A, H)
    actor_mods = (nets.a_trunk, nets.a_mu, nets.a_sigma)
    _load(actor_mods, g, "p0_actor_"); _load([nets.c[0]], g, "p0_c1_"); _load([nets.c[1]], g, "p0_c2_")
    for k in range(2):
        nets.c_old[k].load_state_dict(nets.c[k].state_dict())
    c2_lr = float(cfg["critic2_lr"]) if bool(cfg["critic2"]) else float(cfg["critic_lr"])
    opts = [torch.optim.Adam(nets.actor_params(), lr=float(cfg["actor_lr"])),
            torch.optim.Adam(nets.c[0].parameters(), lr=float(cfg["critic_lr"])), torch.optim.Adam(nets.c[1].parameters(), lr=c2_lr)]
    if bool(cfg["auto"]):
        la = torch.nn.Parameter(torch.tensor(0.0))
        alpha = AutoAlphaState(la, -float(A), torch.optim.Adam([la], lr=float(cfg["alpha_lr"])))
    else:
        alpha = float(cfg["alpha"])
    cql_log_alpha = torch.tensor([0.0], requires_grad=True)
    mult = (cql_log_alpha, torch.optim.Adam([cql_log_alpha], lr=float(cfg["cql_alpha_lr"]))) if bool(cfg["with_lagrange"]) else None
    kw = dict(gamma=float(cfg["gamma"]), tau=float(cfg["tau"]), temperature=float(cfg["temperature"]), cql_weight=float(cfg["cql_weight"]),
              num_repeat_actions=int(cfg["R"]), lagrange_threshold=float(cfg["lagrange_threshold"]), min_action=float(cfg["min_action"]),
              max_action=float(cfg["max_action"]), alpha_min=float(cfg["alpha_min"]), alpha_max=float(cfg["alpha_max"]),
              max_grad_norm=float(cfg["max_grad_norm"]))
    noise = lambda shape: torch.normal(torch.zeros(shape), torch.ones(shape))
    for u in range(int(cfg["updates"])):
        o, tag = f"u{u}_", f"oracle_cql/{variant}/u{u}"
        idx = g[o + "indices"]
        f32 = lambda k: torch.as_tensor(np.asarray(g["buf_" + k])[idx]).to(torch.float32)
        batch = dict(obs=f32("obs"), act=f32("act"), rew=f32("rew"), done=f32("done"), obs_next=f32("obs_next"),
                     calibration_returns=torch.as_tensor(g["calibration_returns"][idx]).float() if bool(cfg["calibrated"]) else None)
        torch.manual_seed(100 + u)
        r = cql_update(nets, opts, alpha, mult, batch, noise, **kw)
        got = np.array([r["actor_loss"], r["critic1_loss"], r["critic2_loss"]])
        record_parity(f"{tag}/losses", got, g[o + "losses"], rtol=1e-5, atol=1e-6)
        if mult is not None:
            record_parity(f"{tag}/cql_alpha", np.array([r["cql_alpha"], r["cql_alpha_loss"], cql_log_alpha.item()]),
                          np.array([g[o + "cql_alpha"], g[o + "cql_alpha_loss"], g[o + "cql_log_alpha"]]), rtol=1e-5, atol=1e-7)
        else:
            assert np.isnan(g[o + "cql_alpha"]) and r["cql_alpha"] is None
        if bool(cfg["auto"]):
            record_parity(f"{tag}/log_alpha", np.array([alpha.log_alpha.item()]), np.array([g[o + "log_alpha"]]), rtol=1e-5, atol=1e-7)
        assert np.array_equal(torch.get_rng_state().numpy(), g[o + "torch_rng"]), "CPU generator differs from the reference's"
        lr = float(cfg["critic_lr"])
        _check(tag, actor_mods, g, o + "actor_", float(cfg["actor_lr"]))
        _check(tag, [nets.c[0]], g, o + "c1_", lr); _check(tag, [nets.c[1]], g, o + "c2_", c2_lr)
        _check(tag, [nets.c_old[0]], g, o + "c1old_", lr); _check(tag, [nets.c_old[1]], g, o + "c2old_", c2_lr)


def test_random_actions_of_the_defaults_are_all_one():
    """cql.py:303-307 with min_action = -1, max_action = 1 draws uniform_(1, 1): every random action is exactly 1.0, and the
    CPU generator still advances."""
    torch.manual_seed(0)
    before = torch.get_rng_state()
    x = torch.FloatTensor(40, 3).uniform_(1.0, 1.0)
    assert bool((x == 1.0).all()) and not torch.equal(before, torch.get_rng_state())
