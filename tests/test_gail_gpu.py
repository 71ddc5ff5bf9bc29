"""GAIL on the device (algorithm/imitation/gail.py; csrc/gail.cu).

Yardsticks:
  * ``ts_gail_reward_rows`` against float64 -logsigmoid(-x): 8 x torch fp32's own error + 1e-7 x max, every row written past
    the grid cap;
  * ``ts_gail_disc_rows`` against float64 autograd of the reference's two losses: loss 2e-5 relative, d loss / d logit 1e-6,
    counts exact, two calls bit-identical;
  * one discriminator step's weight gradient against float64 autograd on the module: 2e-4 relative + 1e-4 x max, the bar of
    the three-product weight-gradient MMAs;
  * ``update()`` against the reference's own outputs (tests/golden/gail_ref_*.npz): rewards and PPO's preprocessing at 1e-5,
    the per-step losses at the per-row bars, accuracies exactly, parameters at 1e-3 + 0.1 lr, generator states identical.
"""
import copy

import numpy as np
import pytest
import torch

from offpolicy_testutil import DEV, ptxas_report, sm_count, stream
from ts_testutil import Box, load_golden, record_parity, restore_vector_buffer

VARIANTS = ["gail_ref_tc", "gail_ref_merge", "gail_ref_steps", "gail_ref_layered"]
gpu = pytest.mark.gpu


def _gaussian_dist(loc_scale):
    loc, scale = loc_scale
    return torch.distributions.Independent(torch.distributions.Normal(loc, scale), 1)


def _disc(O, A, hidden, act):
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.continuous import ContinuousCritic
    return ContinuousCritic(preprocess_net=Net(state_shape=(O,), action_shape=(A,), hidden_sizes=hidden, activation=act,
                                               concat=True)).to(DEV)


def _nets(O, A, hidden=(64, 64), disc_act=torch.nn.Tanh):
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.continuous import ContinuousActorProbabilistic, ContinuousCritic
    actor = ContinuousActorProbabilistic(preprocess_net=Net(state_shape=(O,), hidden_sizes=hidden, activation=torch.nn.Tanh),
                                         action_shape=(A,), unbounded=True).to(DEV)
    critic = ContinuousCritic(preprocess_net=Net(state_shape=(O,), hidden_sizes=hidden, activation=torch.nn.Tanh)).to(DEV)
    return actor, critic, _disc(O, A, hidden, disc_act)


def _gail(actor, critic, disc, expert, A, lr=3e-4, disc_lr=5e-4, disc_optim=None, policy=None, **kw):
    from tianshou_b200.algorithm import GAIL, AdamOptimizerFactory, ProbabilisticActorPolicy
    policy = policy or ProbabilisticActorPolicy(actor=actor, dist_fn=_gaussian_dist, action_scaling=True, action_bound_method="clip",
                                                action_space=Box(A))
    return GAIL(policy=policy, critic=critic, optim=AdamOptimizerFactory(lr=lr), expert_buffer=expert, disc_net=disc,
                disc_optim=disc_optim or AdamOptimizerFactory(lr=disc_lr), **kw)


def _expert(g):
    from tianshou_b200.data import ReplayBuffer
    if int(g["cfg_vector_expert"]):
        return restore_vector_buffer(g, "exp_", 4, 50, device=DEV)
    return ReplayBuffer.from_data(*(g["exp_" + k] for k in ("obs", "act", "rew", "terminated", "truncated")),
                                  g["exp_terminated"] | g["exp_truncated"], g["exp_obs_next"])


def _golden_algo(g, expert=None):
    from tianshou_b200.algorithm import AdamOptimizerFactory, LRSchedulerFactoryLinear
    O, A = int(g["cfg_obs"]), int(g["cfg_act"])
    hidden = tuple(int(h) for h in g["cfg_hidden"])
    actor, critic, disc = _nets(O, A, hidden, torch.nn.ReLU if int(g["cfg_disc_relu"]) else torch.nn.Tanh)
    with torch.no_grad():
        for mod, tag in ((actor, "actor"), (critic, "critic"), (disc, "disc")):
            for i, p in enumerate(mod.parameters()):
                p.copy_(torch.as_tensor(g[f"p0_{tag}_{i}"]).reshape(p.shape))
    kw = {k[3:]: g[k].item() for k in g.files if k.startswith("kw_")}
    for k in ("return_scaling", "value_clip", "advantage_normalization", "recompute_advantage"):
        if k in kw:
            kw[k] = bool(kw[k])
    disc_optim = AdamOptimizerFactory(lr=float(g["cfg_disc_lr"]))
    if int(g["cfg_sched"]):
        disc_optim.with_lr_scheduler_factory(LRSchedulerFactoryLinear(max_epochs=2, epoch_num_steps=8, collection_step_num_env_steps=4))
    algo = _gail(actor, critic, disc, expert if expert is not None else _expert(g), A, lr=float(g["cfg_lr"]), disc_optim=disc_optim,
                 disc_update_num=int(g["cfg_dun"]), **kw)
    return algo, actor, critic, disc


# ---------------------------------------------------------------------------------------------------------- kernels
@gpu
@pytest.mark.parametrize("n", [1, 17, 1000, None])
def test_reward_rows_vs_fp64(n):
    """-logsigmoid(-x) per row; None: 2 grid caps + 7 rows, every row must be written."""
    from tianshou_b200._cabi import call, ptr
    if n is None:
        n = sm_count() * 16 * 256 * 2 + 7
    special = np.array([0.0, 1e-30, -1e-30, 20.0, -20.0, 88.0, -88.0, 100.0, -100.0, 1e4, -1e4], dtype=np.float32)
    x = (np.random.default_rng(n).standard_normal(n) * 5.0).astype(np.float32)
    x[: min(n, special.size)] = special[: min(n, special.size)]
    xt = torch.as_tensor(x)
    ref = (-torch.nn.functional.logsigmoid(-xt.double())).numpy()
    torch_err = np.abs((-torch.nn.functional.logsigmoid(-xt)).double().numpy() - ref)
    rew = torch.full((n,), float("nan"), dtype=torch.float64, device=DEV)
    call("ts_gail_reward_rows", ptr(xt.to(DEV)), n, ptr(rew), stream())
    got = rew.cpu().numpy()
    assert np.isfinite(got).all()
    record_parity(f"gail_reward_rows/n{n}", got, ref, rtol=0.0, atol=8 * float(torch_err.max()) + 1e-7 * float(np.abs(ref).max()))


@gpu
@pytest.mark.parametrize("n_pi,n_exp", [(44, 42), (1, 1), (1000, 700), (3001, 2048)])
def test_disc_rows_vs_fp64_autograd(n_pi, n_exp):
    """Loss, accuracies and d loss / d logit of one discriminator step; exact zeros are counted on neither side, saturated
    rows (|x| = 100, 1e4) have gradients 0 or +-1 / n."""
    from tianshou_b200._cabi import call, ptr
    rng = np.random.default_rng(n_pi)
    x = (rng.standard_normal(n_pi + n_exp) * 3.0).astype(np.float32)
    x[::7] = 0.0
    x[3::11] = 100.0
    x[5::13] = -1e4
    xt = torch.as_tensor(x)
    st = stream()
    outs = []
    for _ in range(2):
        dl = torch.empty(n_pi + n_exp, device=DEV)
        row = torch.empty(4, device=DEV)
        call("ts_gail_disc_rows", ptr(xt.to(DEV)), n_pi, n_exp, ptr(dl), ptr(row), st)
        outs.append((dl.cpu(), row.cpu()))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    dl, row = outs[0][0].numpy(), outs[0][1].numpy()
    x64 = xt.double().requires_grad_(True)
    lp, le = x64[:n_pi], x64[n_pi:]
    loss = -torch.nn.functional.logsigmoid(-lp).mean() + -torch.nn.functional.logsigmoid(le).mean()
    loss.backward()
    record_parity(f"gail_disc_rows/{n_pi}_{n_exp}/loss", row[0:1], [float(loss.detach())], rtol=2e-5, atol=0.0)
    record_parity(f"gail_disc_rows/{n_pi}_{n_exp}/dlogits", dl, x64.grad.numpy(), rtol=0.0, atol=1e-6)
    assert row[1] == (xt[:n_pi] < 0).float().mean().item()
    assert row[2] == (xt[n_pi:] > 0).float().mean().item()
    assert row[3] == n_pi


def _disc_fp64_grad(disc, hidden, act, x_pi, x_exp):
    from oracle import oracle_gail as og
    d = og.disc_net(x_pi.shape[1], 0, hidden, act).double()
    with torch.no_grad():
        for q, p in zip(d.parameters(), disc.parameters(), strict=True):
            q.copy_(p.detach().cpu().double())
    lp = d(torch.as_tensor(x_pi, dtype=torch.float64)).reshape(-1)
    le = d(torch.as_tensor(x_exp, dtype=torch.float64)).reshape(-1)
    (-torch.nn.functional.logsigmoid(-lp).mean() + -torch.nn.functional.logsigmoid(le).mean()).backward()
    return torch.cat([p.grad.reshape(-1) for p in d.parameters()]).numpy()


@gpu
@pytest.mark.parametrize("act,hidden,N,dun", [(torch.nn.Tanh, (64, 64), 256, 2), (torch.nn.ReLU, (128, 128), 128, 3),
                                              (torch.nn.Tanh, (48, 40, 32), 120, 11)])
def test_disc_step_gradient_vs_fp64(act, hidden, N, dun):
    """The weight gradient of the LAST (for N % bsz != 0: merged) discriminator step of the device loop against float64
    autograd of (loss_pi + loss_exp) on a copy of the module."""
    from tianshou_b200.data import ReplayBuffer
    from tianshou_b200.data.batch import minibatch_bounds
    O, A = 17, 6
    torch.manual_seed(0)
    actor, critic, disc = _nets(O, A, (64, 64))
    disc = _disc(O, A, hidden, act)
    with torch.no_grad():
        for name, p in disc.named_parameters():
            if name.endswith("bias"):
                p.copy_(0.2 * torch.randn(p.shape))
    expert = ReplayBuffer(8)
    algo = _gail(actor, critic, disc, expert, A, disc_update_num=dun)
    rng = np.random.default_rng(1)
    bsz = N // dun
    lo, hi = minibatch_bounds(N, bsz, merge_last=True)[-1]
    x_all = rng.standard_normal((N, O + A)).astype(np.float32)
    x_exp = (rng.standard_normal((bsz, O + A)) + 0.5).astype(np.float32)
    perm = rng.permutation(N)
    ref = _disc_fp64_grad(disc, hidden, act, x_all[perm[lo:hi]], x_exp)
    src = torch.as_tensor(np.concatenate([x_all, x_exp]), device=DEV)
    rows = torch.as_tensor(np.concatenate([perm[lo:hi], N + np.arange(bsz)]), dtype=torch.int64, device=DEV)
    table = torch.zeros((1, 4), device=DEV)
    algo._disc_loop(src, rows, [(lo, hi)], bsz, table)
    got = algo._g_disc.grad.cpu().numpy()
    record_parity(f"gail_disc_grad/{act.__name__}_{'x'.join(map(str, hidden))}_N{N}_k{dun}", got, ref, rtol=2e-4,
                  atol=1e-4 * float(np.abs(ref).max()))
    assert int(table[0, 3].item()) == hi - lo


# ---------------------------------------------------------------------------------------------------------- goldens
def _assert_state(g, prefix, st):
    assert np.array_equal(np.asarray(st[1], dtype=np.uint32), g[prefix + "key"]) and int(st[2]) == int(g[prefix + "pos"]), prefix
    assert np.array_equal(np.array([float(st[3]), float(st[4])]), g[prefix + "gauss"]), prefix


@gpu
@pytest.mark.parametrize("variant", VARIANTS)
def test_gail_matches_reference(variant):
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden(f"{variant}.npz")
    algo, actor, critic, disc = _golden_algo(g)
    assert (algo._layered is not None) == (variant == "gail_ref_layered")
    E, cap, bs, repeat = int(g["cfg_E"]), int(g["cfg_cap"]), int(g["cfg_bs"]), int(g["cfg_repeat"])
    lr, disc_lr = float(g["cfg_lr"]), float(g["cfg_disc_lr"])
    captured = {}
    orig = algo._preprocess_batch

    def hook(batch, buffer, indices):
        b = orig(batch, buffer, indices)
        captured.update({k: b[k].detach().cpu().numpy().copy() for k in ("rew", "v_s", "returns", "adv", "logp_old")})
        return b

    algo._preprocess_batch = hook
    for u in range(2):
        o = f"u{u}_"
        buf = restore_vector_buffer(g, o, E, cap, device=DEV)
        np.random.seed(int(g[o + "np_seed"]))
        assert algo.disc_optim._optim.param_groups[0]["lr"] == pytest.approx(float(g[o + "disc_lr"]), rel=1e-12)
        with policy_within_training_step(algo.policy):
            stats = algo.update(buffer=buf, batch_size=bs, repeat=repeat)
        for k in ("rew", "v_s", "returns", "adv", "logp_old"):
            ref = g[o + k]
            record_parity(f"{variant}_u{u}/{k}", captured[k], ref, rtol=1e-5, atol=1e-5 * float(np.abs(ref).max()))
        table = algo.last_disc_table
        assert table.shape == (g[o + "disc_loss"].shape[0], 4)
        ref = g[o + "disc_loss"]
        record_parity(f"{variant}_u{u}/disc_loss", table[:, 0], ref, rtol=2e-4, atol=2e-5 * float(np.abs(ref).max()))
        assert list(table[:, 1]) == list(g[o + "acc_pi"]) and list(table[:, 2]) == list(g[o + "acc_exp"])
        assert g[o + "margin_pi"].min() > 1e-4 and g[o + "margin_exp"].min() > 1e-4
        assert stats.disc_loss.mean == pytest.approx(float(table[:, 0].mean()))
        ref_losses = g[o + "losses"]
        for col in range(4):
            # column 1 (the clipped surrogate) is a mean of O(1) terms that cancel to ~1e-3 with normalised advantages: its fp32
            # summation error is absolute (1.4e-7 observed), hence the 1e-6 floor
            record_parity(f"{variant}_u{u}/ppo_{col}", algo.last_loss_table[:, col], ref_losses[:, col], rtol=2e-4,
                          atol=2e-5 * max(1e-3, float(np.abs(ref_losses[:, col]).max())) + (1e-6 if col == 1 else 0.0))
        for mod, tag, rate in ((actor, "actor", lr), (critic, "critic", lr), (disc, "disc", disc_lr)):
            for i, p in enumerate(mod.parameters()):
                ref = g[f"{o}{tag}_{i}"]
                record_parity(f"{variant}_u{u}/{tag}_{i}", p.detach().cpu().numpy(), ref.reshape(p.shape), rtol=1e-3, atol=0.1 * rate)
        _assert_state(g, o + "rng_np_", np.random.get_state())
        _assert_state(g, o + "rng_exp_", algo.expert_buffer._random_state.get_state())
        if int(g["cfg_vector_expert"]):
            for e in range(4):
                _assert_state(g, f"{o}rng_exp{e}_", algo.expert_buffer._child_rng(e).get_state())


@gpu
def test_update_leaves_a_full_mirrored_buffer_unmodified():
    """With a full device-mirrored buffer ``_sample`` hands out the mirror's own rew column; the rewards must go elsewhere."""
    from tianshou_b200.data import Batch, ReplayBuffer, VectorReplayBuffer
    from tianshou_b200.utils import policy_within_training_step
    E, T, O, A = 16, 16, 11, 3
    rng = np.random.default_rng(4)
    buf = VectorReplayBuffer(E * T, E, device=DEV, device_mirror=True)
    for _ in range(T):
        buf.add(Batch(obs=rng.standard_normal((E, O)).astype(np.float32), act=rng.standard_normal((E, A)).astype(np.float32),
                      rew=rng.standard_normal(E), terminated=rng.random(E) < 0.05, truncated=np.zeros(E, bool),
                      obs_next=rng.standard_normal((E, O)).astype(np.float32), info=Batch()))
    expert = ReplayBuffer.from_data(rng.standard_normal((200, O)).astype(np.float32), rng.standard_normal((200, A)).astype(np.float32),
                                    np.zeros(200), np.zeros(200, bool), np.zeros(200, bool), np.zeros(200, bool),
                                    rng.standard_normal((200, O)).astype(np.float32))
    actor, critic, disc = _nets(O, A)
    algo = _gail(actor, critic, disc, expert, A, disc_update_num=2)
    host_before = np.asarray(buf._meta.rew).copy()
    dev_before = buf.device_columns()["rew"].clone()
    captured = {}
    orig = algo._preprocess_batch

    def hook(batch, buffer, indices):
        b = orig(batch, buffer, indices)
        captured["rew"] = b.rew.cpu().numpy()
        return b

    algo._preprocess_batch = hook
    np.random.seed(0)
    with policy_within_training_step(algo.policy):
        algo.update(buffer=buf, batch_size=64, repeat=2)
    assert np.array_equal(np.asarray(buf._meta.rew), host_before)
    assert torch.equal(buf.device_columns()["rew"], dev_before)
    assert not np.array_equal(captured["rew"], host_before)


@gpu
def test_state_dict_round_trip_continues_training():
    """state_dict() carries disc_net.* and both optimisers (actor-critic first); a reloaded copy continues bit-identically."""
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden("gail_ref_steps.npz")
    E, cap, bs = int(g["cfg_E"]), int(g["cfg_cap"]), int(g["cfg_bs"])
    algo, actor, critic, disc = _golden_algo(g)

    def run(a, u):
        np.random.seed(int(g[f"u{u}_np_seed"]))
        with policy_within_training_step(a.policy):
            a.update(buffer=restore_vector_buffer(g, f"u{u}_", E, cap, device=DEV), batch_size=bs, repeat=1)

    run(algo, 0)
    sd = algo.state_dict()
    assert any(k.startswith("disc_net.") for k in sd) and len(sd["_optimizers"]) == 2
    assert sd["_optimizers"][1]["state"][0]["step"] == 12
    algo2, actor2, critic2, disc2 = _golden_algo(g, expert=copy.deepcopy(algo.expert_buffer))
    algo2.load_state_dict(sd)
    assert algo2._g_disc.step == algo._g_disc.step == 12
    torch.testing.assert_close(algo2._g_disc.exp_avg_sq, algo._g_disc.exp_avg_sq, rtol=0, atol=0)
    run(algo, 1)
    run(algo2, 1)
    for a, b in ((actor, actor2), (critic, critic2), (disc, disc2)):
        for p, q in zip(a.parameters(), b.parameters()):
            assert torch.equal(p, q)


# ---------------------------------------------------------------------------------------------------------- API
@gpu
def test_constructor_refusals_and_update_errors(monkeypatch):
    from tianshou_b200.algorithm import AdamOptimizerFactory, RMSpropOptimizerFactory, UnsupportedModelError
    from tianshou_b200.algorithm.imitation import gail as gail_module
    from tianshou_b200.data import ReplayBuffer
    from tianshou_b200.utils import policy_within_training_step
    O, A = 11, 3
    expert = ReplayBuffer(8)
    actor, critic, disc = _nets(O, A)
    with pytest.raises(UnsupportedModelError, match="Box action space"):
        from tianshou_b200.algorithm import ProbabilisticActorPolicy
        from test_ppo_discrete_gpu import Discrete
        _gail(actor, critic, disc, expert, A, policy=ProbabilisticActorPolicy(actor=actor, dist_fn=_gaussian_dist,
                                                                             action_scaling=False, action_space=Discrete(3)))
    with pytest.raises(TypeError, match="known output dimension"):
        from tianshou_b200.algorithm import ProbabilisticActorPolicy
        lin = torch.nn.Linear(O, A).to(DEV)
        _gail(lin, critic, disc, expert, A, policy=ProbabilisticActorPolicy(actor=lin, dist_fn=_gaussian_dist, action_space=Box(A)))
    with pytest.raises(UnsupportedModelError):                                  # reads obs only: not a chain on obs + act
        from tianshou_b200.utils.net.common import Net
        from tianshou_b200.utils.net.continuous import ContinuousCritic
        _gail(actor, critic, ContinuousCritic(preprocess_net=Net(state_shape=(O,), hidden_sizes=(64,))).to(DEV), expert, A)
    with pytest.raises(UnsupportedModelError):
        _gail(actor, critic, torch.nn.Sequential(torch.nn.Linear(O + A, 1)).to(DEV), expert, A)
    with pytest.raises(UnsupportedModelError, match="single linear"):
        from tianshou_b200.utils.net.common import Net
        from tianshou_b200.utils.net.continuous import ContinuousCritic
        bad = ContinuousCritic(preprocess_net=Net(state_shape=(O,), action_shape=(A,), hidden_sizes=(64,), concat=True)).to(DEV)
        bad.last.model[0] = torch.nn.Linear(64, 2).to(DEV)
        _gail(actor, critic, bad, expert, A)
    with pytest.raises(UnsupportedModelError, match="Adam"):
        _gail(actor, critic, disc, expert, A, disc_optim=RMSpropOptimizerFactory(lr=1e-3))
    with pytest.raises(UnsupportedModelError, match="stack_num"):
        _gail(actor, critic, disc, ReplayBuffer(8, stack_num=2), A)
    wide = ReplayBuffer.from_data(np.zeros((4, O + 1), np.float32), np.zeros((4, A), np.float32), np.zeros(4), np.zeros(4, bool),
                                  np.zeros(4, bool), np.zeros(4, bool), np.zeros((4, O + 1), np.float32))
    with pytest.raises(UnsupportedModelError, match="do not match"):
        _gail(actor, critic, disc, wide, A)
    monkeypatch.setattr(gail_module, "world", lambda: (0, 2))
    with pytest.raises(UnsupportedModelError, match="single-GPU"):
        _gail(actor, critic, disc, expert, A)
    monkeypatch.undo()

    g = load_golden("gail_ref_steps.npz")
    algo, *_ = _golden_algo(g)
    buf = restore_vector_buffer(g, "u0_", int(g["cfg_E"]), int(g["cfg_cap"]), device=DEV)
    np.random.seed(3)
    before = np.random.get_state()
    with pytest.raises(RuntimeError, match="outside of a training step"):
        algo.update(buffer=buf, batch_size=40, repeat=1)
    after = np.random.get_state()
    assert np.array_equal(before[1], after[1]) and before[2] == after[2]
    algo.disc_update_num = len(buf) + 1
    with pytest.raises(AssertionError), policy_within_training_step(algo.policy):
        algo.update(buffer=buf, batch_size=40, repeat=1)
    after = np.random.get_state()
    assert np.array_equal(before[1], after[1]) and before[2] == after[2]


@gpu
def test_discriminator_loop_has_no_torch_host_sync():
    """Every discriminator step runs under torch.cuda.set_sync_debug_mode("error")."""
    from tianshou_b200.data.batch import minibatch_bounds
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden("gail_ref_merge.npz")
    algo, *_ = _golden_algo(g)
    buf = restore_vector_buffer(g, "u0_", int(g["cfg_E"]), int(g["cfg_cap"]), device=DEV)
    with policy_within_training_step(algo.policy):
        batch, indices = algo._sample(buf, 0)
        batch = algo._preprocess_batch(batch, buf, indices)
    N, dun = batch.obs.shape[0], int(g["cfg_dun"])
    bsz = N // dun
    bounds = minibatch_bounds(N, bsz, merge_last=True)
    src = algo._disc_input(batch, "gail_disc_src", N + len(bounds) * bsz)
    perm = np.random.default_rng(0).permutation(N)
    rows = torch.as_tensor(np.concatenate([np.concatenate([perm[lo:hi], N + s * bsz + np.arange(bsz)])
                                           for s, (lo, hi) in enumerate(bounds)]), device=DEV)
    table = torch.zeros((len(bounds), 4), device=DEV)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        algo._disc_loop(src, rows, bounds, bsz, table)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    algo._rms_end()
    assert bool(torch.isfinite(table).all()) and table[:, 3].sum().item() == N


# ---------------------------------------------------------------------------------------------------------- resources
def test_gail_kernels_are_spill_free(tmp_path):
    """ptxas's report for gail.cu (sm_90a): no stack frame and no spills in either kernel."""
    found = ptxas_report("gail.cu", tmp_path)
    for name in ("gail_reward_kernel", "gail_disc_kernel"):
        hits = [v for k, v in found.items() if name in k]
        assert hits == [(0, 0, 0)], (name, found)
