"""The eager BCQ restatement (oracle/oracle_bcq.py) against outputs of the imported reference (tests/golden/bcq_ref_*.npz from
oracle/gen_golden_bcq.py), and ``Perturbation``, ``VAE`` and the policy's torch path against the reference itself when it is
present.  CPU only."""
import copy

import numpy as np
import pytest
import torch

from offpolicy_testutil import golden_cfg
from ts_testutil import load_golden, record_parity

VARIANTS = ["d4rl", "net", "small"]


def oracle_nets(cfg):
    """BcqNets with the recipe's seeded initial weights (critic 2 a copy of critic 1 unless the golden has its own)."""
    from oracle.oracle_bcq import BcqNets
    from oracle.oracle_discrete_sac import seeded_params
    O, A, L = int(cfg["obs"]), int(cfg["act"]), int(cfg["latent"])
    nets = BcqNets(O, A, tuple(int(x) for x in cfg["hidden"]), tuple(int(x) for x in cfg["vae_hidden"]), L,
                   float(cfg["max_action"]), float(cfg["phi"]), bool(cfg["per_row"]))
    s = int(cfg["init_seed"])
    seeded_params(nets.p, s)
    seeded_params(nets.c[0], s + 1)
    if bool(cfg["critic2"]):
        seeded_params(nets.c[1], s + 2)
    else:
        nets.c[1].load_state_dict(nets.c[0].state_dict())
    seeded_params(torch.nn.ModuleList(nets.vae_modules()), s + 3)
    nets.p_old.load_state_dict(nets.p.state_dict())
    for k in range(2):
        nets.c_old[k].load_state_dict(nets.c[k].state_dict())
    return nets


def oracle_batch(g, idx, dtype=torch.float32):
    f = lambda k: torch.as_tensor(g["buf_" + k][idx]).to(dtype)
    return dict(obs=f("obs"), act=f("act"), obs_next=f("obs_next"), rew=torch.as_tensor(g["buf_rew"][idx]).float().to(dtype),
                done=torch.as_tensor(g["buf_done"][idx]))


def check_net_params(tag, mods, g, prefix, rtol, atol):
    from oracle.oracle_discrete_sac import golden_view
    compact = bool(golden_cfg(g)["compact"])
    params = [p for m in mods for p in m.parameters()]
    for i, p in enumerate(params):
        got = golden_view(p) if compact else p.detach().cpu().numpy()
        record_parity(f"{tag}/{prefix}{i}", got, g[f"{prefix}{i}"].reshape(got.shape), rtol=rtol, atol=atol)


@pytest.mark.parametrize("variant", VARIANTS)
def test_oracle_matches_reference(variant):
    from oracle.oracle_bcq import bcq_policy, bcq_update
    g = load_golden(f"bcq_ref_{variant}.npz")
    cfg = golden_cfg(g)
    nets = oracle_nets(cfg)
    opts = [torch.optim.Adam(nets.p.parameters(), lr=float(cfg["actor_lr"])), torch.optim.Adam(nets.c[0].parameters(), lr=float(cfg["critic_lr"])),
            torch.optim.Adam(nets.c[1].parameters(), lr=float(cfg["critic2_lr"] if bool(cfg["critic2"]) else cfg["critic_lr"])),
            torch.optim.Adam(nets.vae_parameters(), lr=float(cfg["vae_lr"]))]
    U = int(cfg["updates"])
    for u in range(U):
        o, tag = f"u{u}_", f"oracle_bcq/{variant}/u{u}"
        torch.manual_seed(100 + u)
        r = bcq_update(nets, opts, oracle_batch(g, g[o + "indices"]), lambda shape: torch.randn(shape), gamma=float(cfg["gamma"]),
                       tau=float(cfg["tau"]), lmbda=float(cfg["lmbda"]), N=int(cfg["N"]))
        record_parity(f"{tag}/losses", np.array([r["actor_loss"], r["critic1_loss"], r["critic2_loss"], r["vae_loss"]]), g[o + "losses"],
                      rtol=1e-5, atol=1e-6)
        assert np.array_equal(torch.get_rng_state().numpy(), g[o + "torch_rng"]), "CPU generator differs from the reference's"
        if bool(cfg["compact"]) and u < U - 1:
            continue
        for prefix, mods in (("pert_", [nets.p]), ("c1_", [nets.c[0]]), ("c2_", [nets.c[1]]), ("vae_", nets.vae_modules()),
                             ("pold_", [nets.p_old]), ("c1old_", [nets.c_old[0]]), ("c2old_", [nets.c_old[1]])):
            check_net_params(tag, mods, g, o + prefix, rtol=1e-4, atol=1e-6)
    if "policy_obs" in g.files:
        torch.manual_seed(900)
        act = bcq_policy(nets, torch.as_tensor(g["policy_obs"]), int(cfg["S"]))
        record_parity(f"oracle_bcq/{variant}/policy_act", act, g["policy_act"], rtol=1e-5, atol=1e-6)
        assert np.array_equal(torch.get_rng_state().numpy(), g["policy_torch_rng"])


def test_net_golden_binds_the_clamp_and_has_done_rows():
    """The ``net`` case exercises what it is there for: perturbed actions at +-max_action, many done rows, N = 1."""
    g = load_golden("bcq_ref_net.npz")
    cfg = golden_cfg(g)
    nets = oracle_nets(cfg)
    b = oracle_batch(g, g["u0_indices"])
    torch.manual_seed(7)
    with torch.no_grad():
        a = nets.perturb(b["obs"], nets.decode(b["obs"]))
    m = float(cfg["max_action"])
    assert int((a.abs() == m).sum()) > 0 and int(cfg["N"]) == 1 and float(cfg["lmbda"]) == 0.5
    assert b["done"].float().mean() > 0.2


# ------------------------------------------------------------------------------------------------------------ reference API
def _reference():
    from oracle.ref_shim import import_reference, reference_available
    if not reference_available():
        pytest.skip("reference tree not present")
    return import_reference()


def _pair(per_row, O=5, A=3, m=2.0, phi=0.3, seed=3):
    """(reference, tianshou_b200) Perturbation, critic and VAE built under the same seed."""
    _reference()
    from tianshou.utils.net.common import MLP as RMLP
    from tianshou.utils.net.common import Net as RNet
    from tianshou.utils.net.continuous import VAE as RVAE
    from tianshou.utils.net.continuous import ContinuousCritic as RCritic
    from tianshou.utils.net.continuous import Perturbation as RPert

    from tianshou_b200.utils.net.common import MLP, Net
    from tianshou_b200.utils.net.continuous import VAE, ContinuousCritic, Perturbation
    out = []
    for mlp_cls, net_cls, pert_cls, crit_cls, vae_cls in ((RMLP, RNet, RPert, RCritic, RVAE), (MLP, Net, Perturbation, ContinuousCritic, VAE)):
        torch.manual_seed(seed)
        pre = (net_cls(state_shape=(O + A,), action_shape=(A,), hidden_sizes=(16,)) if per_row
               else mlp_cls(input_dim=O + A, output_dim=A, hidden_sizes=(16,)))
        pert = pert_cls(preprocess_net=pre, max_action=m, phi=phi)
        crit = crit_cls(preprocess_net=net_cls(state_shape=(O,), action_shape=(A,), hidden_sizes=(16,), concat=True))
        vae = vae_cls(encoder=mlp_cls(input_dim=O + A, hidden_sizes=(12, 12)), decoder=mlp_cls(input_dim=O + 4, output_dim=A, hidden_sizes=(12, 12)),
                      hidden_dim=12, latent_dim=4, max_action=m)
        out.append((pert, crit, vae))
    return out


@pytest.mark.parametrize("per_row", [False, True], ids=["mlp", "net"])
def test_perturbation_and_vae_match_reference(per_row):
    (rp, _, rv), (mp, _, mv) = _pair(per_row)
    for r, m in ((rp, mp), (rv, mv)):
        sr, sm = r.state_dict(), m.state_dict()
        assert list(sr.keys()) == list(sm.keys())
        assert all(torch.equal(sr[k], sm[k]) for k in sr)
    assert (mv.latent_dim, mv.max_action, mp.phi, mp.max_action) == (4, 2.0, 0.3, 2.0)
    s, a = torch.randn(4, 5), torch.randn(4, 3)
    out_r, out_m = rp(s, a), mp(s, a)
    assert torch.equal(out_r, out_m)
    noise = out_m - a
    if not per_row:      # row 0's perturbation on every row (until the clamp)
        inside = (out_m.abs() < 2.0).all(dim=0)
        assert torch.allclose(noise[:, inside], noise[:1, inside].expand(4, -1), atol=1e-6)
    torch.manual_seed(5)
    rr = rv(s, a)
    torch.manual_seed(5)
    mm = mv(s, a)
    assert all(torch.equal(x, y) for x, y in zip(rr, mm, strict=True))
    torch.manual_seed(6)
    dr = rv.decode(s)
    torch.manual_seed(6)
    assert torch.equal(dr, mv.decode(s))


@pytest.mark.parametrize("per_row", [False, True], ids=["mlp", "net"])
def test_policy_torch_path_matches_reference(per_row):
    _reference()
    from gymnasium.spaces import Box as RBox
    from tianshou.algorithm.imitation.bcq import BCQPolicy as RPolicy
    from tianshou.data import Batch as RBatch

    from tianshou_b200.algorithm import BCQPolicy
    from tianshou_b200.data import Batch
    (rp, rc, rv), (mp, mc, mv) = _pair(per_row)
    mc.load_state_dict(rc.state_dict())
    ref = RPolicy(actor_perturbation=rp, critic=rc, vae=rv, action_space=RBox(-2.0, 2.0, (3,)), forward_sampled_times=7)
    mine = BCQPolicy(actor_perturbation=mp, critic=mc, vae=mv, action_space=RBox(-2.0, 2.0, (3,)), forward_sampled_times=7)
    obs = np.random.default_rng(1).standard_normal((6, 5)).astype(np.float32)
    torch.manual_seed(11)
    with torch.no_grad():
        a_r = ref(RBatch(obs=obs, info={})).act
    st_r = torch.get_rng_state()
    torch.manual_seed(11)
    with torch.no_grad():
        a_m = mine(Batch(obs=copy.deepcopy(obs), info={})).act
    assert isinstance(a_m, np.ndarray) and a_m.shape == (6, 3)
    np.testing.assert_array_equal(a_r, a_m)
    assert torch.equal(st_r, torch.get_rng_state())
