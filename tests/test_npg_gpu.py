"""NPG / TRPO on the device (algorithm/modelfree/npg.py, trpo.py; csrc/npg.cu).

Yardsticks:
  * the Fisher-vector product against float64 torch double backward of the reference's KL expression (npg.py:172-200) on
    copies of the same modules: 2e-4 relative + 1e-4 x max, the bar of the three-product weight-gradient MMAs;
  * the device conjugate gradient against a float64 CG on the same operator: 1e-4 x max (fp32 vectors, fp64 scalars);
  * KL and surrogate rows against float64 torch: 1e-5 relative (plain fp32 row arithmetic);
  * NPG and TRPO ``update()`` against the reference's own outputs (tests/golden/npg_ref_*.npz, trpo_ref_*.npz): the
    preprocessing at the 1e-5 bar, every per-minibatch statistic, the warnings exactly, the parameters after each update.
"""
import copy
import warnings

import numpy as np
import pytest
import torch

from ts_testutil import Box, load_golden, record_parity, restore_vector_buffer

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
VARIANTS = ["npg_ref_gauss", "trpo_ref_gauss", "npg_ref_mb", "trpo_ref_mb", "npg_ref_cat", "trpo_ref_cat", "trpo_ref_backtrack",
            "trpo_ref_fail", "trpo_ref_nobt"]


def _gaussian_dist(loc_scale):
    loc, scale = loc_scale
    return torch.distributions.Independent(torch.distributions.Normal(loc, scale), 1)


def _nets(categorical, O, A, hidden=(64, 64), act=None, shared=False):
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.continuous import ContinuousActorProbabilistic, ContinuousCritic
    from tianshou_b200.utils.net.discrete import DiscreteActor, DiscreteCritic
    act = act or (torch.nn.ReLU if categorical else torch.nn.Tanh)
    net_a = Net(state_shape=(O,), hidden_sizes=hidden, activation=act)
    net_c = net_a if shared else Net(state_shape=(O,), hidden_sizes=hidden, activation=act)
    if categorical:
        return DiscreteActor(preprocess_net=net_a, action_shape=(A,)).to(DEV), DiscreteCritic(preprocess_net=net_c).to(DEV)
    return (ContinuousActorProbabilistic(preprocess_net=net_a, action_shape=(A,), unbounded=True).to(DEV),
            ContinuousCritic(preprocess_net=net_c).to(DEV))


def _algo(cls, actor, critic, categorical, A, lr=1e-3, **kw):
    from tianshou_b200.algorithm import AdamOptimizerFactory, DiscreteActorPolicy, ProbabilisticActorPolicy
    if categorical:
        from test_ppo_discrete_gpu import Discrete
        policy = DiscreteActorPolicy(actor=actor, dist_fn=torch.distributions.Categorical, action_space=Discrete(A))
    else:
        policy = ProbabilisticActorPolicy(actor=actor, dist_fn=_gaussian_dist, action_scaling=True, action_bound_method="clip",
                                          action_space=Box(A))
    return cls(policy=policy, critic=critic, optim=AdamOptimizerFactory(lr=lr), **kw)


def _perturb(actor, seed, A):
    """Non-zero biases and distinct log-stds (the perturb_params recipe for any trunk)."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in actor.named_parameters():
            if name.endswith("bias"):
                p.copy_(0.3 * torch.randn(p.shape, generator=g))
        if hasattr(actor, "sigma_param"):
            actor.sigma_param.copy_(torch.linspace(-1.2, 0.3, A).reshape(actor.sigma_param.shape))


# ---------------------------------------------------------------------------------------------------------- FVP
def _fp64_head(actor, obs, categorical):
    a = actor
    if categorical:
        logits = a.last.model(a.preprocess.model.model(obs))
        return torch.distributions.Categorical(probs=torch.softmax(logits, -1))
    mu = a.mu.model(a.preprocess.model.model(obs))
    return _gaussian_dist((mu, a.sigma_param.reshape(-1).exp().expand_as(mu)))


def _fvp_fp64(actor, obs, v, categorical):
    """npg.py:172-200 without damping: d/dtheta (dKL/dtheta . v), KL(old || new).mean() at old = new, float64 autograd."""
    a = copy.deepcopy(actor).to("cpu", torch.float64)
    params = list(a.parameters())
    o = torch.as_tensor(obs, dtype=torch.float64)
    dist = _fp64_head(a, o, categorical)
    with torch.no_grad():
        old = _fp64_head(a, o, categorical)
    kl = torch.distributions.kl_divergence(old, dist).mean()
    grads = torch.autograd.grad(kl, params, create_graph=True)
    flat = torch.cat([g.reshape(-1) for g in grads])
    fv = torch.autograd.grad((flat * torch.as_tensor(v, dtype=torch.float64)).sum(), params)
    return torch.cat([g.reshape(-1) for g in fv]).numpy()


FVP_SHAPES = [  # (categorical, obs, act, hidden, activation, saturate)
    (False, 11, 1, (64, 64), torch.nn.Tanh, False),
    (False, 11, 6, (64, 64), torch.nn.Tanh, False),
    (False, 17, 17, (64, 64), torch.nn.Tanh, False),
    (False, 376, 17, (256, 256), torch.nn.Tanh, False),
    (False, 20, 4, (48, 40, 32), torch.nn.ReLU, False),
    (True, 8, 2, (64, 64), torch.nn.ReLU, False),
    (True, 8, 5, (64, 64), torch.nn.ReLU, True),
    (True, 8, 64, (64, 64), torch.nn.ReLU, True),
    (True, 376, 9, (256, 256), torch.nn.Tanh, False),
    (True, 20, 7, (48, 40, 32), torch.nn.ReLU, True),
]


@pytest.mark.parametrize("shape", FVP_SHAPES, ids=lambda s: f"{'cat' if s[0] else 'gauss'}_o{s[1]}_a{s[2]}_{'x'.join(map(str, s[3]))}")
def test_fvp_vs_fp64_double_backward(shape):
    """F v from the tangent pass + KL-Hessian rows + backward pass against fp64 double backward.  Saturated softmax rows (a few
    observations scaled x40) exercise the clamp of Categorical's logits; there the reference's double backward differs from
    the Gauss-Newton product by terms of dKL/dhead ~ 1e-7, inside the bar."""
    from tianshou_b200.algorithm import NPG
    categorical, O, A, hidden, act, saturate = shape
    torch.manual_seed(1)
    actor, critic = _nets(categorical, O, A, hidden, act)
    _perturb(actor, 3, A)
    algo = _algo(NPG, actor, critic, categorical, A)
    L = algo._layered
    B = 300
    rng = np.random.default_rng(5)
    obs = rng.standard_normal((B, O)).astype(np.float32)
    if saturate:
        obs[::17] *= 40.0
    v = rng.standard_normal(L.group.n).astype(np.float32)
    o = torch.as_tensor(obs, device=DEV)
    at = L.a_trunk.forward(o, B, "up")
    ah = L.a_head.forward(at[-1], B, "up")
    algo._fvp(at, ah, torch.as_tensor(v, device=DEV), B)
    got = L.group.grad.cpu().numpy()
    ref = _fvp_fp64(actor, obs, v, categorical)
    scale = float(np.abs(ref).max())
    record_parity(f"npg_fvp/{'cat' if categorical else 'gauss'}_o{O}_a{A}_{len(hidden)}x{hidden[0]}", got, ref, rtol=2e-4,
                  atol=1e-4 * scale)


# ---------------------------------------------------------------------------------------------------------- CG
def _cg_fp64(M, b, damping, nsteps=10, tol=1e-10):
    x = np.zeros_like(b)
    r, p = b.copy(), b.copy()
    rdotr = r @ r
    it = 0
    for _ in range(nsteps):
        z = M @ p + damping * p
        alpha = rdotr / (p @ z)
        x += alpha * p
        r -= alpha * z
        new = r @ r
        it += 1
        if new < tol:
            break
        p = r + new / rdotr * p
        rdotr = new
    return x, it


@pytest.mark.parametrize("case", ["ten_iterations", "early_exit"])
def test_cg_vs_fp64(case):
    """ts_cg_init / ts_cg_step (z = M p supplied by a plain matmul) against fp64 CG on M + 0.1 I.  "early_exit": M has two
    distinct eigenvalues, so the residual vanishes after 2 iterations and every later step must be a no-op."""
    from tianshou_b200._cabi import call, ptr, stream_ptr
    n = 3000
    rng = np.random.default_rng(11)
    Q, _ = np.linalg.qr(rng.standard_normal((n, 40)))
    if case == "early_exit":
        M = 0.5 * (Q @ Q.T)                                # eigenvalues 0.5 (x40) and 0: two clusters with the damping
        b = (Q @ rng.standard_normal(40) + 0.1 * rng.standard_normal(n)) * 1e-3
    else:
        M = (Q * rng.uniform(0.5, 50.0, 40)) @ Q.T
        b = rng.standard_normal(n)
    b = b.astype(np.float32).astype(np.float64)
    x_ref, it_ref = _cg_fp64(M, b, 0.1)
    Md = torch.as_tensor(M, dtype=torch.float32, device=DEV)
    g = torch.as_tensor(b, dtype=torch.float32, device=DEV)
    x, r, p, z = (torch.empty(n, device=DEV) for _ in range(4))
    state = torch.empty(3, dtype=torch.float64, device=DEV)
    iters = torch.zeros(1, device=DEV)
    st = stream_ptr(torch.device(DEV))
    call("ts_cg_init", ptr(g), ptr(x), ptr(r), ptr(p), n, ptr(state), st)
    for _ in range(10):
        torch.matmul(Md, p, out=z)
        call("ts_cg_step", ptr(x), ptr(r), ptr(p), ptr(z), n, 0.1, 1e-10, ptr(state), ptr(iters), st)
    assert int(iters.item()) == it_ref == int(state[2].item())
    if case == "early_exit":
        assert it_ref < 10 and state[1].item() == 1.0
    record_parity(f"npg_cg/{case}", x.cpu().numpy(), x_ref, rtol=0.0, atol=1e-4 * float(np.abs(x_ref).max()))


# ---------------------------------------------------------------------------------------------------------- rows
@pytest.mark.parametrize("categorical,A", [(False, 1), (False, 6), (False, 17), (True, 2), (True, 5), (True, 64)])
@pytest.mark.parametrize("ratio", [0, 1])
def test_surrogate_and_kl_rows_vs_fp64(categorical, A, ratio):
    """ts_npg_rows (loss rows, d loss / d head, d loss / d logstd rows) and ts_npg_kl_rows against fp64 torch."""
    from tianshou_b200._cabi import call, ptr, stream_ptr
    B = 700
    rng = np.random.default_rng(A + 10 * ratio)
    head = rng.standard_normal((B, A)) * (4.0 if categorical else 1.0)
    head_new = head + 0.3 * rng.standard_normal((B, A))
    ls, ls_new = rng.uniform(-1.0, 0.5, A), rng.uniform(-1.0, 0.5, A)
    act = rng.integers(0, A, B).astype(np.float64) if categorical else rng.standard_normal((B, A))
    adv, lpo = rng.standard_normal(B), rng.standard_normal(B) - 2.0
    f32 = lambda a: np.asarray(a, np.float32)
    head, head_new, ls, ls_new, act, adv, lpo = map(lambda a: f32(a).astype(np.float64), (head, head_new, ls, ls_new, act, adv, lpo))
    dh, dls_, dact, dadv, dlpo, dhn, dlsn = (torch.as_tensor(f32(a), device=DEV).contiguous()
                                             for a in (head, ls, act, adv, lpo, head_new, ls_new))
    st = stream_ptr(torch.device(DEV))
    loss_rows, dhead, dls, kl = (torch.empty(s, device=DEV) for s in (B, (B, A), (B, A), B))
    call("ts_npg_rows", ptr(dh), ptr(dls_), ptr(dact), ptr(dadv), ptr(dlpo), B, A, int(categorical), ratio, ptr(loss_rows),
         ptr(dhead), ptr(dls), st)
    call("ts_npg_kl_rows", ptr(dh), ptr(dls_), ptr(dhn), ptr(dlsn), B, A, int(categorical), ptr(kl), st)

    h = torch.tensor(head, requires_grad=True)
    s = torch.tensor(ls, requires_grad=True)
    eps32 = float(torch.finfo(torch.float32).eps)

    def cat_logits(hh):
        # Categorical(probs = softmax) in float64 but clamped at float32's eps, the clamp the fp32 rows apply
        # (a float64 Categorical clamps at 2.2e-16 and would disagree on saturated rows)
        return torch.softmax(hh, -1).clamp(eps32, 1.0 - eps32).log()

    def dist(hh, ss):
        return _gaussian_dist((hh, ss.exp().expand_as(hh)))

    if categorical:
        lp = cat_logits(h).gather(1, torch.tensor(act).long()[:, None])[:, 0]
    else:
        lp = dist(h, s).log_prob(torch.tensor(act))
    w = (lp - torch.tensor(lpo)).exp() if ratio else lp
    rows = -(w * torch.tensor(adv))
    rows.mean().backward()
    tag = f"{'cat' if categorical else 'gauss'}_a{A}_{'trpo' if ratio else 'npg'}"
    ref_rows = rows.detach().numpy()
    record_parity(f"npg_rows/{tag}/loss", loss_rows.cpu().numpy(), ref_rows, rtol=1e-5, atol=1e-6 * float(np.abs(ref_rows).max()))
    gh = h.grad.numpy()
    record_parity(f"npg_rows/{tag}/dhead", dhead.cpu().numpy(), gh, rtol=1e-4, atol=1e-5 * float(np.abs(gh).max()))
    if not categorical:
        gs = s.grad.numpy()
        record_parity(f"npg_rows/{tag}/dlogstd", dls.cpu().numpy().sum(0), gs, rtol=1e-4, atol=1e-5 * float(np.abs(gs).max()))
    with torch.no_grad():
        if categorical:
            po = torch.softmax(torch.tensor(head), -1)
            kl_ref = (po * (cat_logits(torch.tensor(head)) - cat_logits(torch.tensor(head_new)))).sum(-1).numpy()
        else:
            kl_ref = torch.distributions.kl_divergence(dist(torch.tensor(head), torch.tensor(ls)),
                                                       dist(torch.tensor(head_new), torch.tensor(ls_new))).numpy()
    record_parity(f"npg_rows/{tag}/kl", kl.cpu().numpy(), kl_ref, rtol=1e-4, atol=1e-6)


def test_categorical_kl_is_inf_where_a_new_probability_is_zero():
    """torch's rule (kl.py _kl_categorical_categorical): inf where q.probs == 0, 0 where p.probs == 0.  The yardstick is
    torch's fp32 kl_divergence on the same fp32 heads (a fp64 softmax would not underflow)."""
    from tianshou_b200._cabi import call, ptr, stream_ptr
    old = torch.tensor([[0.0, 1.0, -1.0], [0.0, 1.0, -1.0], [0.0, -200.0, 1.0], [0.5, 0.2, 0.1]])
    new = torch.tensor([[0.0, 1.0, -300.0], [0.0, 1.0, -1.0], [0.0, -300.0, 1.0], [0.1, 0.2, 0.5]])
    kl = torch.empty(4, device=DEV)
    old_d, new_d = old.to(DEV), new.to(DEV)
    call("ts_npg_kl_rows", ptr(old_d), None, ptr(new_d), None, 4, 3, 1, ptr(kl), stream_ptr(torch.device(DEV)))
    ref = torch.distributions.kl_divergence(torch.distributions.Categorical(probs=torch.softmax(old, -1)),
                                            torch.distributions.Categorical(probs=torch.softmax(new, -1)))
    got = kl.cpu()
    assert torch.isinf(got[0]) and torch.isinf(ref[0])
    assert got[1].item() == 0.0 and ref[1].item() == 0.0
    np.testing.assert_allclose(got[2:].numpy(), ref[2:].numpy(), rtol=1e-5, atol=1e-7)


# ---------------------------------------------------------------------------------------------------------- goldens
def _golden_algo(g):
    from tianshou_b200.algorithm import NPG, TRPO
    categorical, O, A = bool(g["cfg_categorical"]), int(g["cfg_obs"]), int(g["cfg_act"])
    actor, critic = _nets(categorical, O, A)
    with torch.no_grad():
        for mod, tag in ((actor, "actor"), (critic, "critic")):
            for i, p in enumerate(mod.parameters()):
                p.copy_(torch.as_tensor(g[f"p0_{tag}_{i}"]).reshape(p.shape))
    kw = {k[3:]: (g[k].item()) for k in g.files if k.startswith("kw_")}
    for k in ("optim_critic_iters", "max_backtracks"):
        if k in kw:
            kw[k] = int(kw[k])
    for k in ("return_scaling", "advantage_normalization"):
        if k in kw:
            kw[k] = bool(kw[k])
    cls = TRPO if int(g["cfg_trpo"]) else NPG
    return _algo(cls, actor, critic, categorical, A, lr=float(g["cfg_lr"]), **kw), actor, critic


@pytest.mark.parametrize("variant", VARIANTS)
def test_npg_trpo_match_reference(variant):
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden(f"{variant}.npz")
    algo, actor, critic = _golden_algo(g)
    assert algo._layered is not None and algo._layered.group is not algo._layered.critic_group
    trpo = bool(g["cfg_trpo"])
    E, cap, bs = int(g["cfg_E"]), int(g["cfg_cap"]), int(g["cfg_bs"])
    captured = {}
    orig = algo._preprocess_batch

    def hook(batch, buffer, indices):
        b = orig(batch, buffer, indices)
        captured.update({k: b[k].detach().cpu().numpy().copy() for k in ("v_s", "returns", "adv", "logp_old")})
        return b

    algo._preprocess_batch = hook
    lr = float(g["cfg_lr"])
    for u in range(2):
        o = f"u{u}_"
        buf = restore_vector_buffer(g, o, E, cap, device=DEV)
        np.random.seed(int(g[o + "np_seed"]))
        with warnings.catch_warnings(record=True) as w, policy_within_training_step(algo.policy):
            warnings.simplefilter("always")
            stats = algo.update(buffer=buf, batch_size=None if bs < 0 else bs, repeat=int(g["cfg_repeat"]))
        # update 0 starts from identical parameters: the 1e-5 bar.  Update 1 evaluates networks that already carry update 0's
        # differences (fp32 conjugate gradients in two summation orders, amplified by TRPO steps of up to 1.5 along the
        # natural direction): the parameters' bar
        bar = 1e-5 if u == 0 else 1e-3
        for k in ("v_s", "returns", "adv", "logp_old"):
            ref = g[o + k]
            record_parity(f"{variant}_u{u}/{k}", captured[k], ref, rtol=bar, atol=bar * max(1e-3, float(np.abs(ref).max())))
        got_w = [str(x.message) for x in w if issubclass(x.category, UserWarning) and "action_scaling" not in str(x.message)]
        assert got_w == list(g[o + "warnings"]), (got_w, list(g[o + "warnings"]))
        table = algo.last_stats_table
        assert table.shape[0] == g[o + "actor_loss"].shape[0]
        # CG iterations: the reference never exits early on these inputs; a residual within 1 decade of the tolerance may
        # legitimately take one iteration more or less in a different summation order
        margins = g[o + "cg_log10_rdotr_margin"]
        for m_it, (it_ref, margin) in enumerate(zip(g[o + "cg_iters"], margins)):
            if margin > 1.0:
                assert int(table[m_it, 4]) == int(it_ref)
        cols = [("actor_loss", 0), ("vf_loss", 1), ("kl", 2)] + ([("step_size", 3)] if trpo else [])
        for name, col in cols:
            ref = g[o + name]
            record_parity(f"{variant}_u{u}/{name}", table[:, col], ref, rtol=2e-3,
                          atol=1e-6 + 1e-4 * max(1e-3, float(np.abs(ref).max())))
        assert isinstance(stats.kl.mean, float)
        for mod, tag in ((actor, "actor"), (critic, "critic")):
            for i, p in enumerate(mod.parameters()):
                ref = g[f"{o}{tag}_{i}"]
                record_parity(f"{variant}_u{u}/{tag}_{i}", p.detach().cpu().numpy(), ref.reshape(p.shape), rtol=2e-3,
                              atol=0.1 * lr + 1e-3 * float(np.abs(ref).max()))


def test_trpo_line_search_decisions_are_away_from_their_boundaries():
    """The goldens' discrete decisions (each evaluated candidate: kl vs max_kl, new loss vs actor loss) have margins far
    beyond fp32 noise, so the device path must take the same branches."""
    for variant in [v for v in VARIANTS if v.startswith("trpo")]:
        g = load_golden(f"{variant}.npz")
        max_kl = float(g["kw_max_kl"]) if "kw_max_kl" in g.files else 0.01
        for u in range(2):
            o = f"u{u}_"
            kl, loss = g[o + "ls_kl"], g[o + "ls_new_loss"]
            actor = np.repeat(g[o + "actor_loss"], g[o + "ls_count"])
            assert np.all(np.abs(kl - max_kl) > 1e-3 * max_kl)
            assert np.all(np.abs(loss - actor) > 1e-4 * np.maximum(np.abs(actor), 1e-3))


# ---------------------------------------------------------------------------------------------------------- API
def test_critic_optimizer_state_dict_round_trip():
    """The torch optimiser covers critic.parameters() only (a2c.py:102-109); its Adam state survives state_dict()."""
    from tianshou_b200.algorithm import NPG
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden("npg_ref_gauss.npz")
    algo, actor, critic = _golden_algo(g)
    buf = restore_vector_buffer(g, "u0_", int(g["cfg_E"]), int(g["cfg_cap"]), device=DEV)
    np.random.seed(0)
    with policy_within_training_step(algo.policy):
        algo.update(buffer=buf, batch_size=None, repeat=1)
    opt = algo.optim._optim
    assert {id(p) for grp in opt.param_groups for p in grp["params"]} == {id(p) for p in critic.parameters()}
    sd = algo.state_dict()
    algo2, actor2, critic2 = _golden_algo(g)
    assert isinstance(algo2, NPG)
    algo2.load_state_dict(sd)
    f1, f2 = algo._layered.critic_group, algo2._layered.critic_group
    assert f2.step == f1.step == 5
    torch.testing.assert_close(f2.exp_avg, f1.exp_avg, rtol=0, atol=0)
    torch.testing.assert_close(f2.exp_avg_sq, f1.exp_avg_sq, rtol=0, atol=0)
    torch.testing.assert_close(algo2._layered.group.flat, algo._layered.group.flat, rtol=0, atol=0)


def test_unsupported_configurations_are_refused():
    from tianshou_b200.algorithm import NPG, TRPO, UnsupportedModelError
    actor, critic = _nets(True, 4, 2, shared=True)
    with pytest.raises(UnsupportedModelError, match="separate actor and critic trunks"):
        _algo(NPG, actor, critic, True, 2)
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.continuous import ContinuousActorProbabilistic, ContinuousCritic
    actor = ContinuousActorProbabilistic(preprocess_net=Net(state_shape=(5,), hidden_sizes=(32,)), action_shape=(2,), unbounded=True,
                                         conditioned_sigma=True).to(DEV)
    critic = ContinuousCritic(preprocess_net=Net(state_shape=(5,), hidden_sizes=(32,))).to(DEV)
    with pytest.raises(UnsupportedModelError, match="conditioned sigma"):
        _algo(TRPO, actor, critic, False, 2)
    g = load_golden("npg_ref_gauss.npz")
    algo, _, _ = _golden_algo(g)
    algo.minibatch_shuffle = "device"
    from tianshou_b200.utils import policy_within_training_step
    buf = restore_vector_buffer(g, "u0_", int(g["cfg_E"]), int(g["cfg_cap"]), device=DEV)
    with pytest.raises(UnsupportedModelError, match="device-generated order"), policy_within_training_step(algo.policy):
        algo.update(buffer=buf, batch_size=None, repeat=1)


@pytest.mark.parametrize("variant", ["npg_ref_mb", "trpo_ref_backtrack"])
def test_minibatch_loop_has_no_torch_host_sync(variant, monkeypatch):
    """Every minibatch of NPG runs under torch.cuda.set_sync_debug_mode("error"); in TRPO the one allowed sync is the
    line-search flag read (``TRPO._read_flag``), lifted out of the check and counted."""
    from tianshou_b200.algorithm import TRPO
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden(f"{variant}.npz")
    algo, _, _ = _golden_algo(g)
    reads = []
    orig = TRPO._read_flag

    def read(flag):
        torch.cuda.set_sync_debug_mode("default")
        try:
            reads.append(orig(flag))
            return reads[-1]
        finally:
            torch.cuda.set_sync_debug_mode("error")

    monkeypatch.setattr(TRPO, "_read_flag", staticmethod(read))
    buf = restore_vector_buffer(g, "u1_", int(g["cfg_E"]), int(g["cfg_cap"]), device=DEV)
    with policy_within_training_step(algo.policy):
        batch, indices = algo._sample(buf, 0)
        batch = algo._preprocess_batch(batch, buf, indices)
    N = batch.obs.shape[0]
    bs = int(g["cfg_bs"])
    from tianshou_b200.data.batch import minibatch_bounds
    bounds = minibatch_bounds(N, N if bs < 0 else bs, merge_last=True)
    perm = torch.randperm(N, device=DEV)
    stats = algo._alloc_stats(len(bounds))
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for m, (lo, hi) in enumerate(bounds):
            algo._minibatch(batch, perm[lo:hi], stats[m])
    finally:
        torch.cuda.set_sync_debug_mode("default")
    algo._rms_end()
    assert bool(torch.isfinite(stats[:, :4]).all())
    if isinstance(algo, TRPO):
        assert 1 <= len(reads) <= len(bounds) * algo.max_backtracks
    else:
        assert reads == []
