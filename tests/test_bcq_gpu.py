"""BCQ on the GPU: the bcq.cu kernels against float64 references, ``update()`` against outputs of the imported reference
(tests/golden/bcq_ref_*.npz from oracle/gen_golden_bcq.py) with the buffer mirror on and off, the gradients of all four optimiser
steps against float64 autograd of the eager restatement, the lagged perturbation network, the absence of host synchronisation
inside the update, ``state_dict()`` round trips, the refusals, the device policy path against the reference loop and the kernels'
register report."""
import copy
import re

import numpy as np
import pytest
import torch

from offpolicy_testutil import DEV, Box, Discrete, assert_spill_free, golden_cfg, ptxas_report, stream
from test_oracle_bcq import check_net_params, oracle_batch, oracle_nets
from ts_testutil import load_golden, record_parity

gpu = pytest.mark.gpu
BIG = 300000                 # rows past the grid cap of every grid-stride kernel


def _call(name, *args):
    from tianshou_b200._cabi import call, ptr
    call(name, *[ptr(a) if isinstance(a, torch.Tensor) else a for a in args], stream())
    torch.cuda.synchronize()


def _d(t):
    return t.to(DEV).contiguous()


# ------------------------------------------------------------------------------------------------------------ kernels
VAE_CASES = [(7, 5, 3, 4, 1.0), (256, 17, 6, 12, 1.0), (BIG, 3, 2, 2, 2.0)]


@gpu
@pytest.mark.parametrize("B,O,A,L,m", VAE_CASES, ids=[f"B{c[0]}-O{c[1]}-A{c[2]}-L{c[3]}" for c in VAE_CASES])
def test_vae_kernels_vs_fp64_autograd(B, O, A, L, m):
    """Reparameterisation, loss and head backward against float64 autograd of the reference's VAE arithmetic, with log_std
    exactly at -4 and 15 and beyond both bounds; every row written; two runs bit-identical."""
    g = torch.Generator().manual_seed(B + L)
    head = torch.randn(B, 2 * L, generator=g) * 3
    head[0, L], head[1 % B, L + 1 % L], head[2 % B, L], head[3 % B, L + 1 % L] = -4.0, 15.0, -9.0, 17.0
    eps, s = torch.randn(B, L, generator=g), torch.randn(B, O, generator=g)
    y, act, dz = torch.randn(B, A, generator=g), m * torch.tanh(torch.randn(B, A, generator=g)), torch.randn(B, L, generator=g) / B

    def run():
        std, x = torch.full((B, L), float("nan"), device=DEV), torch.full((B, O + L), float("nan"), device=DEV)
        _call("ts_bcq_vae_reparam", _d(head), _d(eps), B, L, _d(s), O, std, x)
        dy, loss = torch.full((B, A), float("nan"), device=DEV), torch.full((1,), float("nan"), device=DEV)
        _call("ts_bcq_vae_loss", _d(y), _d(act), _d(head), std, B, A, L, m, dy, loss)
        dhead = torch.full((B, 2 * L), float("nan"), device=DEV)
        _call("ts_bcq_vae_head_bwd", _d(head), std, _d(eps), _d(dz), B, L, dhead)
        return std, x, dy, loss, dhead

    std, x, dy, loss, dhead = run()
    hh, yy = head.double().requires_grad_(True), y.double().requires_grad_(True)
    mean, sd = hh[:, :L], torch.exp(hh[:, L:].clamp(-4, 15))
    z = mean + sd * eps.double()
    recon = m * torch.tanh(yy)
    ref = torch.nn.functional.mse_loss(act.double(), recon) + (-torch.log(sd) + (sd.pow(2) + mean.pow(2) - 1) / 2).mean() / 2
    (ref + (z * dz.double()).sum()).backward()
    tag = f"bcq_vae/B{B}_A{A}_L{L}"
    record_parity(f"{tag}/std", std.cpu().numpy(), sd.detach().numpy(), rtol=2e-6, atol=0)
    record_parity(f"{tag}/x", x.cpu().numpy(), torch.cat([s.double(), z.detach()], 1).numpy(), rtol=1e-5, atol=1e-5)
    record_parity(f"{tag}/loss", loss.cpu().numpy(), np.array([ref.item()]), rtol=2e-5, atol=1e-6)
    record_parity(f"{tag}/dy", dy.cpu().numpy(), yy.grad.numpy(), rtol=1e-5, atol=1e-6 * float(yy.grad.abs().max()))
    record_parity(f"{tag}/dhead", dhead.cpu().numpy(), hh.grad.numpy(), rtol=1e-4, atol=1e-5 * float(hh.grad.abs().max()))
    assert float(dhead[0, L]) != 0.0 and float(dhead[1 % B, L + 1 % L]) != 0.0, "the clamp passes the gradient at its bounds"
    assert float(dhead[2 % B, L]) == 0.0 and float(dhead[3 % B, L + 1 % L]) == 0.0
    for a, b in zip((std, x, dy, loss, dhead), run(), strict=True):
        assert torch.equal(a, b)


ROW_CASES = [(5, 1, 3, 4, 2), (70, 33, 17, 6, 3), (BIG // 10, 10, 4, 2, 2)]


@gpu
@pytest.mark.parametrize("B,N,O,A,L", ROW_CASES, ids=[f"B{c[0]}-N{c[1]}" for c in ROW_CASES])
def test_decode_and_target_kernels(B, N, O, A, L):
    """[s repeated N | clamp(z, +-0.5)], [s | m tanh(y)] (also one row per group), and the lmbda-mixed group max with exact ties
    and NaN, done-masked, against float64."""
    g = torch.Generator().manual_seed(B * N)
    s, z = torch.randn(B, O, generator=g), torch.randn(B * N, L, generator=g)
    x = torch.full((B * N, O + L), float("nan"), device=DEV)
    _call("ts_bcq_decode_input", _d(s), B, N, O, _d(z), L, 0.5, x)
    assert torch.equal(x.cpu(), torch.cat([s.repeat_interleave(N, 0), z.clamp(-0.5, 0.5)], 1))
    y, m = torch.randn(B * N, A, generator=g) * 2, 1.5
    xc = torch.full((B * N, O + A), float("nan"), device=DEV)
    _call("ts_bcq_act_rows", x, O + L, _d(y), 1, B * N, O, A, m, xc)
    want = torch.cat([s.repeat_interleave(N, 0).double(), m * torch.tanh(y.double())], 1)
    record_parity(f"bcq_act_rows/B{B}_N{N}", xc.cpu().numpy(), want.numpy(), rtol=1e-6, atol=1e-6)
    xg = torch.full((B, O + A), float("nan"), device=DEV)
    _call("ts_bcq_act_rows", x, O + L, _d(y), N, B, O, A, m, xg)
    assert torch.equal(xg.cpu(), xc.cpu()[::N])
    q1, q2 = torch.randn(B * N, generator=g), torch.randn(B * N, generator=g)
    q1[N:2 * N] = 0.25                         # group 1: exact ties
    q2[N:2 * N] = 0.25
    q1[2 * N + N // 2] = float("nan")          # group 2: a NaN
    rew, done = torch.randn(B, generator=g), (torch.rand(B, generator=g) < 0.3).float()
    lm = 0.75
    out = torch.full((B,), float("nan"), device=DEV)
    _call("ts_bcq_target", _d(q1), _d(q2), B, N, lm, 1 - lm, _d(rew), _d(done), 0.99, out)
    v = lm * torch.min(q1, q2) + (1 - lm) * torch.max(q1, q2)
    ref = rew + torch.logical_not(done.bool()) * 0.99 * v.reshape(B, N).max(1)[0]
    got = out.cpu()
    assert bool(torch.isnan(got[2])) and bool(torch.isnan(ref[2])), "NaN propagates through the group max (and 0 * NaN)"
    mask = ~torch.isnan(ref)
    record_parity(f"bcq_target/B{B}_N{N}", got[mask].numpy(), ref[mask].double().numpy(), rtol=1e-6, atol=1e-6)
    again = torch.empty_like(out)
    _call("ts_bcq_target", _d(q1), _d(q2), B, N, lm, 1 - lm, _d(rew), _d(done), 0.99, again)
    assert torch.equal(out.nan_to_num(7.0), again.nan_to_num(7.0))


PERT_CASES = [(256, 256, 6, 17, 1.0, 0.05), (64, 1, 3, 5, 2.0, 3.0), (BIG, 1, 2, 3, 1.0, 0.5), (20000, 100, 4, 3, 2.0, 3.0)]


@gpu
@pytest.mark.parametrize("rows,S,A,O,m,phi", PERT_CASES, ids=[f"R{c[0]}-S{c[1]}-phi{c[5]}" for c in PERT_CASES])
def test_perturb_and_backward_vs_fp64_autograd(rows, S, A, O, m, phi):
    """Perturbed actions per row (S = 1) and per group (S rows share one logits row), with actions exactly at +-max_action
    (the clamp's gradient passes there) and beyond; dlogits against float64 autograd; two runs bit-identical."""
    G = rows // S
    g = torch.Generator().manual_seed(rows + S)
    logits, y, s = torch.randn(G, A, generator=g), torch.randn(rows, A, generator=g) * 2, torch.randn(rows, O, generator=g)
    vae_m = m
    logits[0, 0], y[0, 0] = 0.0, 30.0              # tanh(30) == 1 in fp32: a = m exactly, noise 0 -> exactly at the bound
    dact = torch.randn(rows, A, generator=g) / rows
    pm = float(np.float32(phi * m))

    def run():
        x = torch.full((rows, O + A), float("nan"), device=DEV)
        _call("ts_bcq_perturb", _d(logits), S, _d(y), rows, A, vae_m, m, phi * m, _d(s), O, O, x)
        dl = torch.full((G, A), float("nan"), device=DEV)
        _call("ts_bcq_perturb_bwd", _d(logits), S, G, _d(y), _d(dact), A, vae_m, m, phi * m, dl)
        return x, dl

    x, dl = run()
    ll = logits.double().requires_grad_(True)
    a = vae_m * torch.tanh(y.double())
    pert = (pm * torch.tanh(ll).repeat_interleave(S, 0) + a).clamp(-m, m)
    (pert * dact.double()).sum().backward()
    tag = f"bcq_perturb/R{rows}_S{S}_phi{phi}"
    record_parity(f"{tag}/x", x[:, O:].cpu().numpy(), pert.detach().numpy(), rtol=1e-6, atol=1e-6)
    assert torch.equal(x[:, :O].cpu(), s) and float(x[0, O]) == m
    if phi > 1:
        assert int((x[:, O:].abs() == m).sum()) > rows // 10
    record_parity(f"{tag}/dlogits", dl.cpu().numpy(), ll.grad.numpy(), rtol=1e-4, atol=1e-5 * float(ll.grad.abs().max()) + 1e-12)
    for u, v in zip((x, dl), run(), strict=True):
        assert torch.equal(u, v)


SEL_CASES = [(10, 100, 3), (BIG, 1, 2), (3000, 33, 4)]


@gpu
@pytest.mark.parametrize("G,S,A", SEL_CASES, ids=[f"G{c[0]}-S{c[1]}" for c in SEL_CASES])
def test_select_kernel_first_argmax_with_nan(G, S, A):
    g = torch.Generator().manual_seed(G + S)
    q = torch.randn(G * S, generator=g)
    if S > 2:
        q[0:S] = 1.0                               # group 0: every value tied -> index 0
        q[S + 1], q[S + 2] = 9.0, 9.0              # group 1: a tie at the max -> the first
        q[2 * S + 2], q[2 * S + 1] = float("nan"), 50.0     # group 2: NaN is the maximum
    O = 3
    x = torch.randn(G * S, O + A, generator=g)
    act, idx = torch.full((G, A), float("nan"), device=DEV), torch.full((G,), -1, dtype=torch.int64, device=DEV)
    _call("ts_bcq_select", _d(q), G, S, _d(x), O + A, O, A, act, idx)
    ref = q.reshape(G, S).argmax(1)
    assert torch.equal(idx.cpu(), ref)
    assert torch.equal(act.cpu(), x.reshape(G, S, O + A)[torch.arange(G), ref, O:])


# ------------------------------------------------------------------------------------------------------------ goldens
def build_from_cfg(cfg, **over):
    """tianshou_b200's BCQ with the recipe's seeded initial weights, on the GPU."""
    from oracle.oracle_discrete_sac import seeded_params

    from tianshou_b200.algorithm import BCQ, AdamOptimizerFactory, BCQPolicy
    from tianshou_b200.utils.net.common import MLP, Net
    from tianshou_b200.utils.net.continuous import VAE, ContinuousCritic, Perturbation
    O, A, L, m = int(cfg["obs"]), int(cfg["act"]), int(cfg["latent"]), float(cfg["max_action"])
    H, VH = tuple(int(x) for x in cfg["hidden"]), tuple(int(x) for x in cfg["vae_hidden"])
    net_a = (Net(state_shape=(O + A,), action_shape=(A,), hidden_sizes=H) if bool(cfg["per_row"])
             else MLP(input_dim=O + A, output_dim=A, hidden_sizes=H))
    pert = Perturbation(preprocess_net=net_a, max_action=m, phi=float(cfg["phi"]))
    crit = lambda: ContinuousCritic(preprocess_net=Net(state_shape=(O,), action_shape=(A,), hidden_sizes=H, concat=True))
    c1 = crit()
    c2 = crit() if bool(cfg["critic2"]) else None
    vae = VAE(encoder=MLP(input_dim=O + A, hidden_sizes=VH), decoder=MLP(input_dim=O + L, output_dim=A, hidden_sizes=VH),
              hidden_dim=VH[-1], latent_dim=L, max_action=m)
    for k, mod in enumerate((pert, c1, c2, vae)):
        if mod is not None:
            seeded_params(mod, int(cfg["init_seed"]) + k)
    policy = BCQPolicy(actor_perturbation=pert.to(DEV), critic=c1.to(DEV), vae=vae.to(DEV), action_space=Box(A, m),
                       forward_sampled_times=int(cfg["S"]))
    kw = dict(policy=policy, actor_perturbation_optim=AdamOptimizerFactory(lr=float(cfg["actor_lr"])),
              critic_optim=AdamOptimizerFactory(lr=float(cfg["critic_lr"])), vae_optim=AdamOptimizerFactory(lr=float(cfg["vae_lr"])),
              critic2=c2.to(DEV) if c2 is not None else None,
              critic2_optim=AdamOptimizerFactory(lr=float(cfg["critic2_lr"])) if c2 is not None else None, gamma=float(cfg["gamma"]),
              tau=float(cfg["tau"]), lmbda=float(cfg["lmbda"]), num_sampled_action=int(cfg["N"]))
    kw.update(over)
    return BCQ(**kw)


def buffer_from_golden(g, mirror):
    from tianshou_b200.data import ReplayBuffer
    buf = ReplayBuffer.from_data(*(g["buf_" + k].copy() for k in ("obs", "act", "rew", "terminated", "truncated", "done", "obs_next")))
    if mirror:
        buf.enable_device_mirror()
        buf.sync_device_mirror()
        assert buf.device_columns() is not None
    return buf


def _cpu_noise(shape):
    """The reference ran on the CPU: eps is torch.randn on the CPU generator, uploaded."""
    return torch.randn(shape).to(DEV)


def _modules(algo):
    return (("pert_", [algo.policy.actor_perturbation]), ("c1_", [algo.policy.critic]), ("c2_", [algo.critic2]), ("vae_", [algo.policy.vae]),
            ("pold_", [algo.actor_perturbation_target]), ("c1old_", [algo.critic_target]), ("c2old_", [algo.critic2_target]))


@gpu
@pytest.mark.parametrize("mirror", [False, True])
@pytest.mark.parametrize("variant", ["d4rl", "net", "small"])
def test_update_matches_reference(variant, mirror):
    from tianshou_b200.data import Batch
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden(f"bcq_ref_{variant}.npz")
    cfg = golden_cfg(g)
    algo = build_from_cfg(cfg)
    assert sorted(algo.state_dict().keys()) == list(g["state_dict_keys"]), "state_dict() keys differ from the reference's"
    buf = buffer_from_golden(g, mirror)
    algo._noise_fn = _cpu_noise
    captured = {}
    orig = algo._preprocess_batch
    algo._preprocess_batch = lambda b, buffer, idx: (captured.update(indices=np.asarray(idx).copy()), orig(b, buffer, idx))[1]
    U = int(cfg["updates"])
    for u in range(U):
        np.random.seed(500 + u)
        torch.manual_seed(100 + u)
        with policy_within_training_step(algo.policy):
            stats = algo.update(buf, int(cfg["bs"]))
        o, tag = f"u{u}_", f"bcq/{variant}_m{int(mirror)}_u{u}"
        assert np.array_equal(captured["indices"], g[o + "indices"]), "sampled indices differ from the reference's"
        assert np.array_equal(torch.get_rng_state().numpy(), g[o + "torch_rng"]), "CPU generator differs from the reference's"
        record_parity(f"{tag}/losses", np.array([stats.actor_loss, stats.critic1_loss, stats.critic2_loss, stats.vae_loss]), g[o + "losses"],
                      rtol=1e-4, atol=2e-5)
        if bool(cfg["compact"]) and u < U - 1:
            continue
        for prefix, mods in _modules(algo):
            check_net_params(tag, mods, g, o + prefix, rtol=1e-3, atol=0.1 * float(cfg["critic_lr"]))
    if "policy_obs" in g.files:
        torch.manual_seed(900)
        with torch.no_grad():
            act = algo.policy(Batch(obs=g["policy_obs"], info={})).act
        assert np.array_equal(torch.get_rng_state().numpy(), g["policy_torch_rng"])
        record_parity(f"bcq/{variant}_m{int(mirror)}/policy_act", act, g["policy_act"], rtol=1e-3, atol=1e-4)


@gpu
def test_lagged_perturbation_moves_by_polyak_only():
    """The target never uses the lagged perturbation network: after an update it is exactly Polyak of its old value toward the
    updated perturbation network, whatever it held before."""
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden("bcq_ref_net.npz")
    cfg = golden_cfg(g)
    a, b = build_from_cfg(cfg), build_from_cfg(cfg)
    with torch.no_grad():
        for p in b.actor_perturbation_target.parameters():
            p.add_(5.0)                             # a different lagged perturbation network ...
    for algo in (a, b):
        algo._noise_fn = _cpu_noise
        np.random.seed(1)
        torch.manual_seed(2)
        old = algo._g_at.flat.clone()
        with policy_within_training_step(algo.policy):
            algo.update(buffer_from_golden(g, mirror=True), int(cfg["bs"]))
        tau = float(cfg["tau"])
        want = old * (1 - tau) + algo._g_actor.flat * tau
        torch.testing.assert_close(algo._g_at.flat, want, rtol=1e-6, atol=1e-6)
    for ga, gb in zip([a._g_actor, *a._g_c, a._g_vae], [b._g_actor, *b._g_c, b._g_vae], strict=True):
        assert torch.equal(ga.flat, gb.flat)        # ... changes nothing else


# ------------------------------------------------------------------------------------------------------------ gradients
class _Recorder(torch.optim.Adam):
    """Adam that keeps the gradient it is about to apply."""

    def step(self, closure=None):
        self.seen = [p.grad.detach().clone() for g in self.param_groups for p in g["params"]]
        return super().step(closure)


def _random_buffer(O, A, n, seed, m=1.0):
    from tianshou_b200.data import ReplayBuffer
    rng = np.random.default_rng(seed)
    term = rng.random(n) < 0.1
    term[[0, -1]] = True
    trunc = (rng.random(n) < 0.03) & ~term
    return ReplayBuffer.from_data(rng.standard_normal((n, O)).astype(np.float32), (m * np.tanh(rng.standard_normal((n, A)))).astype(np.float32),
                                  rng.standard_normal(n), term, trunc, term | trunc, rng.standard_normal((n, O)).astype(np.float32))


def _copy_into(nets, algo):
    """The algorithm's current networks into the restatement's modules."""
    pairs = ((nets.p, algo.policy.actor_perturbation), (nets.c[0], algo.policy.critic), (nets.c[1], algo.critic2),
             (torch.nn.ModuleList(nets.vae_modules()), algo.policy.vae), (nets.p_old, algo.actor_perturbation_target),
             (nets.c_old[0], algo.critic_target), (nets.c_old[1], algo.critic2_target))
    with torch.no_grad():
        for dst, src in pairs:
            for p, q in zip(dst.parameters(), src.parameters(), strict=True):
                p.copy_(q.detach().cpu())


GRAD_CASES = [(17, 6, (256, 256), (512, 512), 12, False), (17, 6, (256, 256), (512, 512), 12, True),
              (376, 17, (64, 64), (128, 128), 34, False), (376, 17, (64, 64), (128, 128), 34, True)]


@gpu
@pytest.mark.parametrize("O,A,H,VH,L,per_row", GRAD_CASES, ids=[f"O{c[0]}-A{c[1]}-{'net' if c[5] else 'mlp'}" for c in GRAD_CASES])
def test_update_gradients_vs_fp64_autograd(O, A, H, VH, L, per_row):
    grad_case(O, A, H, VH, L, per_row)


def grad_case(O, A, H, VH, L, per_row, B=256, edge=""):
    """One update at batch ``B`` (256 in the suite's own cases) with N = 10, max_action 2 and phi 0.5: the VAE's and both
    critics' gradients, taken before their
    Adam steps, against float64 autograd of the eager restatement on copies of the modules with the same eps and latents; the
    perturbation step's against float64 autograd of the actor loss on the pre-update perturbation network with the VAE and
    critic 1 the update stepped (an Adam step is about lr * sign(g), so a float64 re-run of those steps could move a weight by
    2 lr where a tiny gradient's sign differs)."""
    from oracle.oracle_bcq import BcqNets, bcq_update
    from tianshou_b200.algorithm.flat_params import FlatGroup
    from tianshou_b200.utils import policy_within_training_step
    m, N, phi = 2.0, 10, 0.5
    cfg = dict(obs=O, act=A, hidden=H, vae_hidden=VH, latent=L, max_action=m, phi=phi, per_row=per_row, critic2=True, actor_lr=1e-3,
               critic_lr=1e-3, critic2_lr=3e-4, vae_lr=1e-3, gamma=0.99, tau=0.005, lmbda=0.75, N=N, S=10, init_seed=O + A)
    algo = build_from_cfg(cfg)
    buf = _random_buffer(O, A, 900, seed=O, m=m)
    eps_seen = []
    algo._noise_fn = lambda shape: (eps_seen.append(torch.randn(shape, device=DEV)), eps_seen[-1])[1]
    names = {id(algo._g_actor): "pert", id(algo._g_c[0]): "c1", id(algo._g_c[1]): "c2", id(algo._g_vae): "vae"}
    cap = {}

    def adam(group, optimizer, mgn):
        cap[names[id(group)]] = group.grad[:group.n].detach().cpu().double().clone()
        FlatGroup.adam_step(group, optimizer, mgn)

    algo._adam = adam
    orig = algo._preprocess_batch
    algo._preprocess_batch = lambda b, buffer, idx: (cap.update(indices=np.asarray(idx).copy()), orig(b, buffer, idx))[1]
    nets = BcqNets(O, A, H, VH, L, m, phi, per_row)
    _copy_into(nets, algo)
    for mod in nets.modules():
        mod.double()
    pert_before = [p.detach().clone() for p in nets.p.parameters()]
    torch.manual_seed(31)
    with policy_within_training_step(algo.policy):
        stats = algo.update(buf, B)
    torch.cuda.synchronize()
    assert set(cap) == {"indices", "pert", "c1", "c2", "vae"}
    g = {("buf_" + k): np.asarray(buf._meta[k]) for k in ("obs", "act", "obs_next", "rew", "done")}
    batch = oracle_batch(g, cap["indices"], torch.float64)
    opts = [_Recorder(nets.p.parameters(), lr=1e-3), _Recorder(nets.c[0].parameters(), lr=1e-3), _Recorder(nets.c[1].parameters(), lr=3e-4),
            _Recorder([*nets.enc.parameters(), nets.mean.weight, nets.log_std.weight, nets.mean.bias, nets.log_std.bias,
                       *nets.dec.parameters()], lr=1e-3)]           # the VAE group's flat order: the two heads' rows adjacent
    torch.manual_seed(31)
    ref = bcq_update(nets, opts, batch, lambda shape: eps_seen[0].double().cpu(), gamma=0.99, tau=0.005, lmbda=0.75, N=N)
    tag = f"bcq_grad{edge}/O{O}_A{A}_{'net' if per_row else 'mlp'}"
    for name, opt in (("vae", opts[3]), ("c1", opts[1]), ("c2", opts[2])):
        want = torch.cat([x.reshape(-1) for x in opt.seen]).numpy()
        record_parity(f"{tag}/grad_{name}", cap[name].numpy(), want, rtol=2e-4, atol=1e-4 * float(np.abs(want).max()) + 1e-12)
    record_parity(f"{tag}/losses", np.array([stats.critic1_loss, stats.critic2_loss, stats.vae_loss]),
                  np.array([ref["critic1_loss"], ref["critic2_loss"], ref["vae_loss"]]), rtol=2e-5, atol=1e-5)
    # the perturbation step: float64 autograd on the pre-update perturbation network and the stepped VAE / critic 1, with the
    # actor latents the update drew (after the B * N target latents)
    anets = BcqNets(O, A, H, VH, L, m, phi, per_row)
    _copy_into(anets, algo)
    for mod in anets.modules():
        mod.double()
    with torch.no_grad():
        for p, q in zip(anets.p.parameters(), pert_before, strict=True):
            p.copy_(q)
    torch.manual_seed(31)
    torch.randn((B * N, L))
    obs = batch["obs"]
    loss = -anets.c[0](torch.cat([obs, anets.perturb(obs, anets.decode(obs))], -1)).mean()
    want = torch.cat([x.reshape(-1) for x in torch.autograd.grad(loss, list(anets.p.parameters()))]).numpy()
    # the MLP form's one logits row takes the sum over the batch of d loss / d action, which cancels: its absolute error is
    # bounded relative to the largest entry rather than to each
    scale = (1e-3 if not per_row else 1e-4) * float(np.abs(want).max())
    record_parity(f"{tag}/grad_pert", cap["pert"].numpy(), want, rtol=2e-4, atol=scale + 1e-12)
    record_parity(f"{tag}/actor_loss", np.array([stats.actor_loss]), np.array([loss.item()]), rtol=2e-5, atol=1e-5)
    assert len(cap["indices"]) == B and eps_seen[0].shape[0] == B, "the update must run on the B sampled rows"
    assert algo._scratch["t_xc"].shape[0] == B * N, "the target's sampled-action rows must be B x N"


# ------------------------------------------------------------------------------------------------------------ host sync
@gpu
@pytest.mark.parametrize("variant", ["d4rl", "net"])
def test_device_update_has_no_torch_host_sync(variant):
    """The VAE step, the target with its CPU draws, both critic steps, the perturbation step and Polyak run under
    torch.cuda.set_sync_debug_mode("error")."""
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden(f"bcq_ref_{variant}.npz")
    cfg = golden_cfg(g)
    algo = build_from_cfg(cfg)
    buf = buffer_from_golden(g, mirror=True)
    with policy_within_training_step(algo.policy):
        algo.update(buf, int(cfg["bs"]))                 # first update: scratch buffers exist afterwards
        batch, _ = algo._sample(buf, int(cfg["bs"]))
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            losses = algo._device_update(batch)
        finally:
            torch.cuda.set_sync_debug_mode("default")
    assert bool(torch.isfinite(losses).all())


# ------------------------------------------------------------------------------------------------------------ state_dict
@gpu
@pytest.mark.parametrize("variant", ["small", "net"])
def test_state_dict_round_trip_continues_identically(variant):
    """A fresh algorithm loaded from another's ``state_dict()`` after two updates continues bit for bit."""
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden(f"bcq_ref_{variant}.npz")
    cfg = golden_cfg(g)
    a = build_from_cfg(cfg)
    a._noise_fn = _cpu_noise
    for u in range(2):
        torch.manual_seed(1 + u)
        with policy_within_training_step(a.policy):
            a.update(buffer_from_golden(g, False), int(cfg["bs"]))
    b = build_from_cfg(cfg)
    b._noise_fn = _cpu_noise
    with torch.no_grad():
        for p in b.parameters():
            p.add_(0.01)
    b.load_state_dict(copy.deepcopy(a.state_dict()))
    for algo in (a, b):
        buf = buffer_from_golden(g, mirror=False)
        np.random.seed(3)
        for u in range(3):
            torch.manual_seed(10 + u)
            with policy_within_training_step(algo.policy):
                algo.update(buf, int(cfg["bs"]))
    groups = lambda x: [x._g_actor, *x._g_c, *x._g_ct, x._g_at, x._g_vae]
    for ga, gb in zip(groups(a), groups(b), strict=True):
        assert torch.equal(ga.flat, gb.flat) and torch.equal(ga.exp_avg, gb.exp_avg) and torch.equal(ga.exp_avg_sq, gb.exp_avg_sq)


# ------------------------------------------------------------------------------------------------------------ policy
@gpu
@pytest.mark.parametrize("per_row", [False, True], ids=["mlp", "net"])
def test_device_policy_matches_reference_loop(per_row):
    """BCQPolicy.forward on the device against the reference's loop (the torch path, grad enabled) on the same draws: the same
    action except where the top two Q values lie within the GEMM tolerance; the same generator state afterwards."""
    from tianshou_b200.data import Batch
    cfg = dict(obs=11, act=3, hidden=(64, 64), vae_hidden=(64, 64), latent=6, max_action=1.0, phi=0.5, per_row=per_row, critic2=False,
               actor_lr=1e-3, critic_lr=1e-3, critic2_lr=1e-3, vae_lr=1e-3, gamma=0.99, tau=0.005, lmbda=0.75, N=10, S=100, init_seed=8)
    algo = build_from_cfg(cfg)
    obs = np.random.default_rng(4).standard_normal((10, 11)).astype(np.float32)
    torch.manual_seed(77)
    with torch.no_grad():
        dev_act = algo.policy(Batch(obs=obs, info={})).act
    st_dev = torch.get_rng_state()
    torch.manual_seed(77)
    ref_act = algo.policy(Batch(obs=obs, info={})).act       # grad enabled: the reference loop
    assert torch.equal(st_dev, torch.get_rng_state())
    assert dev_act.shape == ref_act.shape == (10, 3)
    # where the choice differs, the two candidates' Q values must be within tolerance of each other
    from oracle.oracle_bcq import BcqNets
    nets = BcqNets(11, 3, (64, 64), (64, 64), 6, 1.0, 0.5, per_row)
    _copy_into(nets, algo)
    same = np.all(np.abs(dev_act - ref_act) <= 1e-4 + 1e-4 * np.abs(ref_act), axis=1)
    for i in np.nonzero(~same)[0]:
        s = torch.as_tensor(obs[i:i + 1]).repeat(2, 1)
        q = nets.c[0](torch.cat([s, torch.as_tensor(np.stack([dev_act[i], ref_act[i]]))], -1)).detach()
        assert abs(float(q[0] - q[1])) <= 1e-4 * max(1.0, float(q.abs().max()))
    assert same.mean() >= 0.8


# ------------------------------------------------------------------------------------------------------------ refusals
@gpu
def test_refusals():
    from torch import nn

    from tianshou_b200.algorithm import BCQ, AdamOptimizerFactory, BCQPolicy, RMSpropOptimizerFactory, UnsupportedModelError
    from tianshou_b200.data import PrioritizedReplayBuffer
    from tianshou_b200.utils import policy_within_training_step
    from tianshou_b200.utils.net.common import MLP, Net
    from tianshou_b200.utils.net.continuous import VAE, ContinuousCritic, Perturbation
    O, A, L = 4, 2, 3

    def make(dev=DEV, space=None, pert=None, critic=None, vae=None, vae_optim=None, **kw):
        pert = pert or Perturbation(preprocess_net=MLP(input_dim=O + A, output_dim=A, hidden_sizes=(8,)), max_action=1.0)
        critic = critic or ContinuousCritic(preprocess_net=Net(state_shape=(O,), action_shape=(A,), hidden_sizes=(8,), concat=True))
        vae = vae or VAE(encoder=MLP(input_dim=O + A, hidden_sizes=(8,)), decoder=MLP(input_dim=O + L, output_dim=A, hidden_sizes=(8,)),
                         hidden_dim=8, latent_dim=L, max_action=1.0)
        pol = BCQPolicy(actor_perturbation=pert.to(dev), critic=critic.to(dev), vae=vae.to(dev), action_space=space or Box(A))
        return BCQ(policy=pol, actor_perturbation_optim=AdamOptimizerFactory(lr=1e-3), critic_optim=AdamOptimizerFactory(lr=1e-3),
                   vae_optim=vae_optim or AdamOptimizerFactory(lr=1e-3), **kw)

    make()
    make(pert=Perturbation(preprocess_net=Net(state_shape=(O + A,), action_shape=(A,), hidden_sizes=(8,)), max_action=1.0))
    with pytest.raises(UnsupportedModelError, match="Box"):
        make(space=Discrete(3))
    with pytest.raises(UnsupportedModelError, match="no CPU path"):
        make(dev="cpu")
    with pytest.raises(UnsupportedModelError, match="no CPU path"):
        _vae_on_cpu(O, A, L)
    with pytest.raises(UnsupportedModelError, match="outside the fused"):
        make(pert=Perturbation(preprocess_net=MLP(input_dim=O + A, output_dim=A, hidden_sizes=(8,), norm_layer=nn.LayerNorm), max_action=1.0))
    with pytest.raises(UnsupportedModelError, match="softmax"):
        make(pert=Perturbation(preprocess_net=Net(state_shape=(O + A,), action_shape=(A,), hidden_sizes=(8,), softmax=True), max_action=1.0))
    with pytest.raises(UnsupportedModelError, match="apply_preprocess_net_to_obs_only"):
        make(critic=ContinuousCritic(preprocess_net=Net(state_shape=(O,), hidden_sizes=(8,)), apply_preprocess_net_to_obs_only=True))
    with pytest.raises(UnsupportedModelError, match="hidden_dim"):
        make(vae=VAE(encoder=MLP(input_dim=O + A, hidden_sizes=(8, 6)), decoder=MLP(input_dim=O + L, output_dim=A, hidden_sizes=(8,)),
                     hidden_dim=8, latent_dim=L, max_action=1.0))
    with pytest.raises(UnsupportedModelError, match="latent"):
        make(vae=VAE(encoder=MLP(input_dim=O + A, hidden_sizes=(8,)), decoder=MLP(input_dim=O + L + 1, output_dim=A, hidden_sizes=(8,)),
                     hidden_dim=8, latent_dim=L, max_action=1.0))
    with pytest.raises(UnsupportedModelError, match="Adam"):
        make(vae_optim=RMSpropOptimizerFactory(lr=1e-3))
    algo = make()
    buf = PrioritizedReplayBuffer(40, alpha=0.6, beta=0.4)
    with pytest.raises(UnsupportedModelError, match="prioritised"):
        with policy_within_training_step(algo.policy):
            algo.update(buf, 8)
    for pert in (None, Perturbation(preprocess_net=Net(state_shape=(O + A,), action_shape=(A,), hidden_sizes=(8,)), max_action=1.0)):
        algo = make(pert=pert)
        with policy_within_training_step(algo.policy):
            stats = algo.update(_random_buffer(O, A, 40, seed=2), 8)
        assert np.isfinite([stats.actor_loss, stats.critic1_loss, stats.critic2_loss, stats.vae_loss]).all()


def _vae_on_cpu(O, A, L):
    """BCQ with every network on the GPU but the VAE."""
    from tianshou_b200.algorithm import BCQ, AdamOptimizerFactory, BCQPolicy
    from tianshou_b200.utils.net.common import MLP, Net
    from tianshou_b200.utils.net.continuous import VAE, ContinuousCritic, Perturbation
    vae = VAE(encoder=MLP(input_dim=O + A, hidden_sizes=(8,)), decoder=MLP(input_dim=O + L, output_dim=A, hidden_sizes=(8,)),
              hidden_dim=8, latent_dim=L, max_action=1.0)
    pert = Perturbation(preprocess_net=MLP(input_dim=O + A, output_dim=A, hidden_sizes=(8,)), max_action=1.0).to(DEV)
    critic = ContinuousCritic(preprocess_net=Net(state_shape=(O,), action_shape=(A,), hidden_sizes=(8,), concat=True)).to(DEV)
    pol = BCQPolicy(actor_perturbation=pert, critic=critic, vae=vae, action_space=Box(A))
    return BCQ(policy=pol, actor_perturbation_optim=AdamOptimizerFactory(lr=1e-3), critic_optim=AdamOptimizerFactory(lr=1e-3),
               vae_optim=AdamOptimizerFactory(lr=1e-3))


# ------------------------------------------------------------------------------------------------------------ resources
def test_bcq_kernels_have_no_stack_frame_or_spills(tmp_path):
    report = ptxas_report("bcq.cu", tmp_path)
    names = sorted(re.search(r"\d+bcq_(\w+?)_kernelE", e).group(1) for e in report)
    assert names == sorted(["vae_reparam", "vae_loss", "vae_head_bwd", "decode_input", "act_rows", "perturb", "perturb_bwd", "target",
                            "select"]), report
    assert_spill_free(report)
