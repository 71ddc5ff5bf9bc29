"""Discrete SAC on the GPU: the categorical rows kernel against float64, ``DiscreteSAC.update()`` against outputs of the imported
reference (tests/golden/dsac_ref_*.npz from oracle/gen_golden_discrete_sac.py), the flat gradients of its three optimiser
steps against float64 autograd, the torch generator against the eager restatement, ``state_dict()`` round trips, the
refusals, the Collector's policy path and the kernel's register report."""
import copy

import numpy as np
import pytest
import torch

from oracle import oracle_discrete_sac as ods
from offpolicy_testutil import DEV, Box, Discrete, assert_spill_free, check_params, load_params, ptxas_report, sm_count, stream
from ts_testutil import load_golden, record_parity

gpu = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------------------ rows kernel
def _rows(logits, q1, q2, alpha, grad=True):
    from tianshou_b200._cabi import call, ptr
    B, A = logits.shape
    v, ent = torch.empty(B, device=DEV), torch.empty(B, device=DEV)
    probs = torch.empty(B, A, device=DEV)
    d = torch.empty(B, A, device=DEV) if grad else None
    call("ts_discrete_sac_rows", ptr(logits), ptr(q1), ptr(q2), alpha, B, A, ptr(v), ptr(ent), ptr(probs), ptr(d), 1.0 / B,
         stream())
    torch.cuda.synchronize()
    return v, ent, probs, d


def _rows_fp64(logits, q1, q2, alpha):
    """The reference expressions in float64 (Categorical(logits).probs / .entropy(), discrete_sac.py:151-155 / :178-183)."""
    z = logits.detach().cpu().double().requires_grad_(True)
    lp = z - z.logsumexp(-1, keepdim=True)
    p = lp.exp()
    H = -(lp.clamp(min=torch.finfo(torch.float64).min) * p).sum(-1)
    m = torch.min(q1, q2).cpu().double()
    v = (p * m).sum(-1) + alpha * H
    (-v.mean()).backward()
    return v.detach(), H.detach(), p.detach(), z.grad, lp.detach(), m


ROW_CASES = [(A, kind) for A in (1, 2, 6, 18, 33, 64, 1000) for kind in ("plain",)] + [
    (6, "saturated"), (18, "saturated"), (33, "equal_q"), (5, "past_grid_cap")]


@gpu
@pytest.mark.parametrize("A,kind", ROW_CASES, ids=[f"A{a}-{k}" for a, k in ROW_CASES])
def test_rows_kernel_vs_fp64(A, kind):
    """v, entropy, probs and d(-mean v)/d logits against float64 autograd.  The bars follow the kernel's arithmetic: each lane
    sums ceil(A / 32) terms in order, then five butterfly levels, every term itself a few roundings off, so a row's error is
    bounded by ~(A / 32 + 10) eps times the sum of the magnitudes of its terms."""
    g = torch.Generator(device="cpu").manual_seed(A * 7 + len(kind))
    B = 300
    if kind == "past_grid_cap":
        B = sm_count() * 16 * 8 + 37     # more rows than warps in the grid
    z = torch.randn(B, A, generator=g) * 3.0
    if kind == "saturated":      # logit spreads > 100: some probabilities underflow to 0 in fp32
        z[: B // 2] *= 60.0
    q1 = torch.randn(B, A, generator=g) * 5.0
    q2 = q1.clone() if kind == "equal_q" else torch.randn(B, A, generator=g) * 5.0
    alpha = 0.17
    z, q1, q2 = z.to(DEV), q1.to(DEV), q2.to(DEV)
    v, ent, probs, d = _rows(z, q1, q2, alpha)
    v64, H64, p64, d64, lp64, m64 = _rows_fp64(z, q1, q2, alpha)
    for t in (v, ent, probs, d):
        assert torch.isfinite(t).all()
    if kind == "saturated":
        assert bool((probs == 0).any()), "the case must underflow some probabilities"
    eps = float(np.finfo(np.float32).eps)
    k = (np.ceil(A / 32) + 10) * eps
    pa, za, lpa, ma = p64.numpy(), z.cpu().double().numpy(), lp64.numpy(), m64.numpy()
    lse = za[:, :1] - lpa[:, :1]
    # per element: p's relative error grows with |z - max| (the fp32 subtraction before exp), log p's absolute error with
    # |z| + |logsumexp| (the fp32 subtraction z - logsumexp)
    rel_p = k + eps * (za.max(-1, keepdims=True) - za)
    err_lp = eps * (np.abs(za) + np.abs(lse))
    bound_H = (pa * (rel_p * np.abs(lpa) + err_lp)).sum(-1) + k * (pa * np.abs(lpa)).sum(-1)
    bound_S = (pa * rel_p * np.abs(ma)).sum(-1) + k * (pa * np.abs(ma)).sum(-1)
    tag = f"dsac_rows/A{A}_{kind}"
    record_parity(f"{tag}/probs", probs.cpu().numpy(), pa, rtol=4 * eps, atol=4 * eps)
    assert np.all(np.abs(ent.cpu().numpy() - H64.numpy()) <= bound_H + 1e-30), f"{tag}: entropy past its bound"
    record_parity(f"{tag}/entropy", ent.cpu().numpy(), H64.numpy(), rtol=0.0, atol=float(bound_H.max()) + 1e-30)
    bound_v = bound_S + alpha * bound_H
    assert np.all(np.abs(v.cpu().numpy() - v64.numpy()) <= bound_v + 1e-30), f"{tag}: v past its bound"
    record_parity(f"{tag}/v", v.cpu().numpy(), v64.numpy(), rtol=0.0, atol=float(bound_v.max()) + 1e-30)
    # d_j = (alpha p_j (log p_j + H) - p_j (m_j - S)) / B: p_j's relative error on the whole bracket, plus the bracket's own
    S64 = (pa * ma).sum(-1, keepdims=True)
    bracket = alpha * (np.abs(lpa) + H64.numpy()[:, None]) + np.abs(ma) + np.abs(S64)
    bound = pa * (rel_p * bracket + alpha * (err_lp + bound_H[:, None]) + bound_S[:, None] + k * bracket) / B + 1e-30
    err = np.abs(d.cpu().numpy() - d64.numpy())
    assert np.all(err <= bound), f"{tag}: dlogits error {float((err - bound).max()):.3e} past its bound"
    record_parity(f"{tag}/dlogits", d.cpu().numpy(), d64.numpy(), rtol=0.0, atol=float(bound.max()))
    # the target call (no dlogits) gives the same rows; a second call is bit-identical
    v2, ent2, probs2, _ = _rows(z, q1, q2, alpha, grad=False)
    v3, ent3, probs3, d3 = _rows(z, q1, q2, alpha)
    assert torch.equal(v, v2) and torch.equal(ent, ent2) and torch.equal(probs, probs2)
    assert torch.equal(v, v3) and torch.equal(ent, ent3) and torch.equal(probs, probs3) and torch.equal(d, d3)


# ------------------------------------------------------------------------------------------------------------ builders
def _trunk(kind, O=None, H=None, W=None, hidden=None, feat=None, A=None, denom=255.0):
    from tianshou_b200.env.atari import DQNet, ScaledObsInputActionReprNet
    from tianshou_b200.utils.net.common import Net
    if kind == "mlp":
        return Net(state_shape=(O,), hidden_sizes=hidden)
    return ScaledObsInputActionReprNet(DQNet(4, H, W, A, features_only=True, output_dim_added_layer=feat), denom=denom)


def build_from_golden(g):
    from tianshou_b200.algorithm import AdamOptimizerFactory, DiscreteSAC
    from tianshou_b200.algorithm.modelfree.discrete_sac import DiscreteSACPolicy
    from tianshou_b200.algorithm.modelfree.sac import AutoAlpha
    from tianshou_b200.utils.net.discrete import DiscreteActor, DiscreteCritic
    A, kind = int(g["cfg_A"]), str(g["cfg_kind"])
    kw = (dict(O=int(g["cfg_obs"]), hidden=tuple(int(x) for x in g["cfg_hidden"])) if kind == "mlp"
          else dict(H=int(g["cfg_H"]), W=int(g["cfg_W"]), feat=int(g["cfg_feat"]), A=A))
    actor = DiscreteActor(preprocess_net=_trunk(kind, **kw), action_shape=A, softmax_output=False).to(DEV)
    c1 = DiscreteCritic(preprocess_net=_trunk(kind, **kw), last_size=A).to(DEV)
    c2 = DiscreteCritic(preprocess_net=_trunk(kind, **kw), last_size=A).to(DEV) if bool(g["cfg_critic2"]) else None
    for k, (m, pfx) in enumerate(((actor, "p0_actor_"), (c1, "p0_c1_"), (c2, "p0_c2_"))):
        if m is None:
            continue
        if bool(g["cfg_compact"]):        # initial weights from the seeded recipe the golden names
            from oracle.oracle_discrete_sac import seeded_params
            seeded_params(m, int(g["cfg_init_seed"]) + k)
        else:
            load_params(m, g, pfx)
    alpha = (AutoAlpha(float(0.98 * np.log(A)), 0.0, AdamOptimizerFactory(lr=float(g["cfg_alpha_lr"]))).to(DEV) if bool(g["cfg_auto"])
             else float(g["cfg_alpha"]))
    clr = float(g["cfg_critic_lr"])
    return DiscreteSAC(policy=DiscreteSACPolicy(actor=actor, action_space=Discrete(A)),
                       policy_optim=AdamOptimizerFactory(lr=float(g["cfg_actor_lr"])), critic=c1,
                       critic_optim=AdamOptimizerFactory(lr=clr), critic2=c2,
                       critic2_optim=AdamOptimizerFactory(lr=clr) if c2 is not None else None, tau=float(g["cfg_tau"]),
                       gamma=float(g["cfg_gamma"]), alpha=alpha, n_step_return_horizon=int(g["cfg_n_step"]))


def buffer_from_golden(g, mirror):
    from tianshou_b200.data import Batch, PrioritizedVectorReplayBuffer, VectorReplayBuffer
    E, cap = int(g["cfg_E"]), int(g["cfg_cap"])
    cnn = str(g["cfg_kind"]) == "cnn"
    kw = dict(stack_num=4, ignore_obs_next=True, save_only_last_obs=True) if cnn else {}
    if bool(g["cfg_per"]):
        buf = PrioritizedVectorReplayBuffer(E * cap, E, alpha=float(g["cfg_per_alpha"]), beta=float(g["cfg_per_beta"]), device=DEV,
                                            device_mirror=mirror, **kw)
    else:
        buf = VectorReplayBuffer(E * cap, E, device=DEV, device_mirror=mirror, **kw)
    for i in range(int(g["cfg_steps"])):
        s = {k: g[f"roll{i}_{k}"] for k in ("obs", "act", "rew", "terminated", "truncated")}
        if cnn:
            s["obs"] = np.repeat(s["obs"][:, None], 4, axis=1)        # only the last frame is stored
            s["obs_next"] = s["obs"]
        else:
            s["obs_next"] = g[f"roll{i}_obs_next"]
        buf.add(Batch(**s), buffer_ids=np.arange(E))
    if mirror:
        assert buf.device_columns() is not None
    return buf


# ------------------------------------------------------------------------------------------------------------ vs reference
@gpu
@pytest.mark.parametrize("variant,mirror", [(v, m) for v in ("mlp", "auto", "cnn") for m in (False, True)])
def test_update_matches_reference(variant, mirror):
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden(f"dsac_ref_{variant}.npz")
    algo = build_from_golden(g)
    buf = buffer_from_golden(g, mirror)
    per, auto = bool(g["cfg_per"]), bool(g["cfg_auto"])
    alr, clr = float(g["cfg_actor_lr"]), float(g["cfg_critic_lr"])
    cap = {}
    orig_pre, orig_post = algo._preprocess_batch, algo._postprocess_batch

    def pre(batch, buffer, indices):
        if per:
            cap["is_weight"] = batch.weight.detach().cpu().numpy().copy()
        b = orig_pre(batch, buffer, indices)
        cap["indices"], cap["returns"] = np.asarray(indices).copy(), b.returns.detach().cpu().numpy().copy()
        return b

    def post(batch, buffer, indices):
        cap["weight"] = batch.weight.detach().cpu().numpy().copy()
        return orig_post(batch, buffer, indices)

    algo._preprocess_batch, algo._postprocess_batch = pre, post
    for u in range(int(g["cfg_updates"])):
        np.random.seed(500 + u)
        torch.manual_seed(100 + u)
        with policy_within_training_step(algo.policy):
            stats = algo.update(buffer=buf, sample_size=int(g["cfg_bs"]))
        o, tag = f"u{u}_", f"dsac_{variant}_m{int(mirror)}_u{u}"
        assert np.array_equal(cap["indices"], g[o + "indices"]), "sampled indices differ from the reference's"
        if per:
            record_parity(f"{tag}/is_weight", cap["is_weight"], g[o + "is_weight"], rtol=1e-4, atol=1e-6)
            record_parity(f"{tag}/tree_leaves", np.asarray(buf.weight[np.arange(len(buf))]), g[o + "tree_leaves"], rtol=1e-4, atol=1e-7)
        ref_ret = g[o + "returns"]
        record_parity(f"{tag}/returns", cap["returns"].reshape(ref_ret.shape), ref_ret, rtol=1e-5, atol=1e-5 * float(np.abs(ref_ret).max()))
        record_parity(f"{tag}/td", cap["weight"], g[o + "weight"], rtol=1e-5, atol=2e-5 * float(np.abs(ref_ret).max()))
        got = np.array([stats.actor_loss, stats.critic1_loss, stats.critic2_loss])
        record_parity(f"{tag}/losses", got, g[o + "losses"], rtol=2e-5, atol=2e-6)
        record_parity(f"{tag}/alpha", np.array([stats.alpha]), np.array([float(g[o + "alpha"])]), rtol=1e-6, atol=0.0)
        if auto:
            record_parity(f"{tag}/alpha_loss", np.array([stats.alpha_loss]), np.array([float(g[o + "alpha_loss"])]), rtol=1e-5, atol=1e-7)
            record_parity(f"{tag}/log_alpha", np.array([algo.alpha._log_alpha.item()]), np.array([float(g[o + "log_alpha"])]),
                          rtol=0.0, atol=1e-6)
        else:
            assert stats.alpha_loss is None
        if o + "actor_0" in g:
            # a compact golden stores each tensor as ``golden_view`` (a fixed-stride sample)
            view = ods.golden_view if bool(g["cfg_compact"]) else None
            for mod, prefix, lr in ((algo.policy.actor, "actor_", alr), (algo.critic, "c1_", clr), (algo.critic2, "c2_", clr),
                                    (algo.critic_old, "c1old_", clr), (algo.critic2_old, "c2old_", clr)):
                check_params(tag, mod, g, o + prefix, lr, view)


# ------------------------------------------------------------------------------------------------------------ gradients
def _chain64(net):
    """float64 callable of a DiscreteActor / DiscreteCritic copy (the modules themselves cast their input to fp32)."""
    pre = net.preprocess
    body = pre.module.net if hasattr(pre, "module") else pre.model.model
    return lambda x: net.last.model(body(x))


def _copy64(mod, group, flat):
    c = copy.deepcopy(mod).to("cpu", torch.float64)
    with torch.no_grad():
        for (_, p), (_, q) in zip(mod.named_parameters(), c.named_parameters(), strict=True):
            q.copy_(group.view(flat, p).view(p.shape).to(torch.float64))
    return c


def _check_grads(tag, mod, group, grad, ref_mod):
    """The GEMMs are fp32-faithful (bf16x3) and the weight gradients sum B products per element: 2e-4 relative plus 1e-4 of
    the tensor's largest value, as in test_offpolicy_gpu."""
    for (name, p), (_, q) in zip(mod.named_parameters(), ref_mod.named_parameters(), strict=True):
        ref = q.grad.numpy()
        got = group.view(grad, p).view(p.shape).cpu().numpy()
        record_parity(f"{tag}/grad_{name}", got, ref, rtol=2e-4, atol=1e-4 * float(np.abs(ref).max()) + 1e-12)


def _grad_setup(kind, A, seed, per, last_hidden):
    """Networks and a filled buffer: 'mlp' (Net on flat fp32 observations) or 'cnn_stacked' (DQNet features trunks on stored
    uint8 [4, H, W] stacks: stack_num 1, obs_next = obs[next(i)])."""
    from tianshou_b200.data import Batch, PrioritizedVectorReplayBuffer, VectorReplayBuffer
    from tianshou_b200.utils.net.discrete import DiscreteActor, DiscreteCritic
    torch.manual_seed(seed)
    rng = np.random.default_rng(seed)
    E, T = 4, 64
    if kind == "mlp":
        O = 12
        trunk = lambda: _trunk("mlp", O=O, hidden=(64, 64))
        kw = {}
        obs_fn = lambda: rng.standard_normal((E, O)).astype(np.float32) * 2.0
    else:
        H = W = 36
        trunk = lambda: _trunk("cnn", H=H, W=W, feat=64, A=A)
        kw = dict(stack_num=1, ignore_obs_next=True)
        obs_fn = lambda: rng.integers(0, 256, (E, 4, H, W), dtype=np.uint8)
    actor = DiscreteActor(preprocess_net=trunk(), action_shape=A, hidden_sizes=last_hidden, softmax_output=False).to(DEV)
    with torch.no_grad():        # a wide logit spread: some rows nearly deterministic, some probabilities near 1e-8
        actor.last.model[-1].bias.copy_(torch.tensor([(0.0, 0.5, 0.0, 9.0, -9.0, 0.0)[a % 6] for a in range(A)]))
    crit = lambda: DiscreteCritic(preprocess_net=trunk(), hidden_sizes=last_hidden, last_size=A).to(DEV)
    buf = (PrioritizedVectorReplayBuffer(E * T, E, alpha=0.6, beta=0.4, device=DEV, **kw) if per
           else VectorReplayBuffer(E * T, E, device=DEV, **kw))
    obs = obs_fn()
    for t in range(T):
        nxt = obs_fn()
        term = rng.random(E) < 0.1
        trunc = np.full(E, t % 17 == 16) & ~term
        buf.add(Batch(obs=obs, act=rng.integers(0, A, E), rew=rng.standard_normal(E), terminated=term, truncated=trunc,
                      obs_next=nxt), buffer_ids=np.arange(E))
        obs = nxt
    if per:
        buf.update_weight(np.arange(E * T), rng.uniform(0.1, 2.0, E * T))
    return actor, crit, buf


def _obs64(kind, buf, idx, next_=False):
    if kind == "mlp":
        a = np.asarray(buf.obs_next)[idx] if next_ else np.asarray(buf.obs)[idx]
        return torch.as_tensor(a).to(torch.float64)
    a = np.asarray(buf.obs)[buf.next(idx) if next_ else idx]
    return torch.as_tensor((np.asarray(a, np.float64) / 255.0).astype(np.float32)).to(torch.float64)


GRAD_CASES = [
    ("mlp", True, False, True, ()),
    ("mlp", False, True, False, (32,)),
    ("cnn_stacked", True, False, True, ()),
    ("cnn_stacked", False, True, False, (32,)),
]


@gpu
@pytest.mark.parametrize("kind,per,auto,separate_critic2,last_hidden", GRAD_CASES,
                         ids=[f"{c[0]}-per{int(c[1])}-auto{int(c[2])}-c2{int(c[3])}-last{len(c[4])}" for c in GRAD_CASES])
def test_update_gradients_vs_fp64_autograd(kind, per, auto, separate_critic2, last_hidden):
    grad_case(kind, per, auto, separate_critic2, last_hidden)


def grad_case(kind, per, auto, separate_critic2, last_hidden, B=None, edge=""):
    """One update at batch ``B`` (the suite's own cases: 64 on frames, 256 on vectors): the flat gradient of each of the three
    optimiser steps, snapshotted before its Adam step, against float64
    autograd of the reference losses (discrete_sac.py:162-184) on copies of the modules with the same parameters, batch and
    returns; the 1-step returns against float64 of the target value; alpha's loss and step.  Adam's first step is lr * sign(g),
    so a gradient off by a constant factor leaves the parameters unchanged; this is the check that sees it."""
    from tianshou_b200.algorithm import AdamOptimizerFactory, DiscreteSAC
    from tianshou_b200.algorithm.flat_params import FlatGroup
    from tianshou_b200.algorithm.modelfree.discrete_sac import DiscreteSACPolicy
    from tianshou_b200.algorithm.modelfree.sac import AutoAlpha
    from tianshou_b200.utils import policy_within_training_step
    A, gamma = 6, 0.9
    actor, crit, buf = _grad_setup(kind, A, seed=len(kind) * 10 + int(per) + 2 * int(auto), per=per, last_hidden=last_hidden)
    c1 = crit()
    c2 = crit() if separate_critic2 else None
    alpha = AutoAlpha(float(0.98 * np.log(A)), float(np.log(0.3)), AdamOptimizerFactory(lr=3e-2)).to(DEV) if auto else 0.3
    algo = DiscreteSAC(policy=DiscreteSACPolicy(actor=actor, action_space=Discrete(A)), policy_optim=AdamOptimizerFactory(lr=1e-3),
                       critic=c1, critic_optim=AdamOptimizerFactory(lr=1e-3), critic2=c2,
                       critic2_optim=AdamOptimizerFactory(lr=1e-3) if c2 is not None else None, tau=0.005, gamma=gamma, alpha=alpha)
    groups = [algo._g_c[0], algo._g_c[1], algo._g_actor]
    init = [copy.deepcopy(m).to("cpu", torch.float64) for m in (actor, algo.critic_old, algo.critic2_old)]
    cap = {"adam": []}

    def adam(group, optimizer, mgn):
        cap["adam"].append((group, group.grad.clone(), [x.flat.clone() for x in groups]))
        FlatGroup.adam_step(group, optimizer, mgn)

    algo._adam = adam
    orig_pre, orig_post = algo._preprocess_batch, algo._postprocess_batch

    def pre(batch, buffer, indices):
        w = batch.__dict__.get("weight")
        cap.update(indices=np.asarray(indices).copy(), weight=None if w is None else w.detach().cpu().clone())
        b = orig_pre(batch, buffer, indices)
        cap["returns"] = b.returns.detach().reshape(-1).cpu().clone()
        return b

    def post(batch, buffer, indices):
        cap["prio_td"] = torch.as_tensor(batch.weight).detach().reshape(-1).cpu().clone()
        return orig_post(batch, buffer, indices)

    algo._preprocess_batch, algo._postprocess_batch = pre, post
    log_alpha0 = float(alpha._log_alpha.item()) if auto else None
    alpha0 = float(np.exp(log_alpha0)) if auto else 0.3
    if B is None:
        B = 64 if kind == "cnn_stacked" else 256
    np.random.seed(31)
    with policy_within_training_step(algo.policy):
        stats = algo.update(buffer=buf, sample_size=B)
    torch.cuda.synchronize()
    tag = f"dsac_grad{edge}/{kind}_per{int(per)}_auto{int(auto)}_c2{int(separate_critic2)}_last{len(last_hidden)}"
    assert [g for g, *_ in cap["adam"]] == groups
    idx = cap["indices"]
    obs, obs_next = _obs64(kind, buf, idx), _obs64(kind, buf, idx, next_=True)
    # target: V(s') of the initial actor and lagged critics, 1-step return r + gamma (1 - terminated) V(s')
    with torch.no_grad():
        lp = torch.log_softmax(_chain64(init[0])(obs_next), -1)
        m = torch.min(_chain64(init[1])(obs_next), _chain64(init[2])(obs_next))
        vn = (lp.exp() * m).sum(-1) - alpha0 * (lp.exp() * lp).sum(-1)
    term = torch.as_tensor(np.asarray(buf.terminated)[idx].astype(np.float64))
    R = torch.as_tensor(np.asarray(buf.rew)[idx].astype(np.float64)) + gamma * (1.0 - term) * vn
    record_parity(f"{tag}/returns", cap["returns"].numpy(), R.numpy(), rtol=1e-5, atol=1e-5 * float(R.abs().max()))
    R = cap["returns"].to(torch.float64)           # the losses below on the returns the update used
    w = cap["weight"].to(torch.float64) if per else torch.ones(B, dtype=torch.float64)
    act = torch.as_tensor(np.asarray(buf.act)[idx].astype(np.int64)).view(-1, 1)
    tds = []
    for k, (mod, losskey) in enumerate(((algo.critic, "critic1_loss"), (algo.critic2, "critic2_loss"))):
        group, grad, flats = cap["adam"][k]
        ref = _copy64(mod, group, flats[k])
        td = _chain64(ref)(obs).gather(1, act).view(-1) - R
        loss = (td.pow(2) * w).mean()
        loss.backward()
        tds.append(td.detach())
        _check_grads(f"{tag}/critic{k + 1}", mod, group, grad, ref)
        record_parity(f"{tag}/{losskey}", np.array([getattr(stats, losskey)]), np.array([loss.item()]), rtol=2e-5, atol=1e-7)
    record_parity(f"{tag}/prio_td", cap["prio_td"].numpy(), ((tds[0] + tds[1]) / 2).numpy(), rtol=1e-5, atol=1e-5 * float(R.abs().max()))
    # actor: -(alpha H + sum_a p min(Q1, Q2)).mean() with the critics after their steps, no gradient into them
    group, grad, flats = cap["adam"][2]
    ra = _copy64(actor, group, flats[2])
    with torch.no_grad():
        rc = [_copy64(m, algo._g_c[k], flats[k]) for k, m in enumerate((algo.critic, algo.critic2))]
        q = torch.min(_chain64(rc[0])(obs), _chain64(rc[1])(obs))
    lp = torch.log_softmax(_chain64(ra)(obs), -1)
    H = -(lp * lp.exp()).sum(-1)
    actor_loss = -(alpha0 * H + (lp.exp() * q).sum(-1)).mean()
    actor_loss.backward()
    _check_grads(f"{tag}/actor", actor, group, grad, ra)
    record_parity(f"{tag}/actor_loss", np.array([stats.actor_loss]), np.array([actor_loss.item()]), rtol=2e-5, atol=1e-6)
    assert len(idx) == B and cap["prio_td"].numel() == B, "the update must run on the B sampled rows"
    if B >= 64:      # a handful of rows need not reach the wide end of the logit spread
        assert float(lp.detach().exp().max()) > 0.99, "the logit spread must make some rows nearly deterministic"
    ties = float((_chain64(rc[0])(obs) == _chain64(rc[1])(obs)).double().mean())
    assert ties == (0.0 if separate_critic2 else 1.0), "critic2=None deep-copies the critic: every entry ties"
    if auto:          # sac.py:203-215 on the entropy rows: one Adam step, lr * sign(g)
        Hd = H.detach()
        record_parity(f"{tag}/entropy", algo._scratch["au_ent"].cpu().numpy(), Hd.numpy(), rtol=1e-5, atol=1e-6)
        deficit = float(0.98 * np.log(A)) - Hd
        record_parity(f"{tag}/alpha_loss", np.array([stats.alpha_loss]), np.array([-(log_alpha0 * deficit).mean().item()]),
                      rtol=1e-5, atol=1e-6)
        g_la = -deficit.mean().item()
        record_parity(f"{tag}/log_alpha", np.array([alpha._log_alpha.item()]), np.array([log_alpha0 - 3e-2 * np.sign(g_la)]),
                      rtol=0.0, atol=1e-6)
    else:
        assert stats.alpha_loss is None


# ------------------------------------------------------------------------------------------------------------ generator
@gpu
def test_generator_state_matches_eager_restatement():
    """The two discarded Categorical draws: after one update() the CUDA generator is where the eager restatement (the
    reference's update in plain torch on the same device) leaves it from the same state."""
    from oracle import oracle_discrete_sac as ods
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden("dsac_ref_mlp.npz")
    algo = build_from_golden(g)
    buf = buffer_from_golden(g, mirror=False)
    cap = {}
    orig_pre = algo._preprocess_batch

    def pre(batch, buffer, indices):
        cap["indices"], cap["w"] = np.asarray(indices).copy(), batch.weight.detach().cpu().numpy().copy()
        return orig_pre(batch, buffer, indices)

    algo._preprocess_batch = pre
    A, O, Hs = int(g["cfg_A"]), int(g["cfg_obs"]), tuple(int(x) for x in g["cfg_hidden"])
    nets = [ods.mlp_head_net(O, Hs, A) for _ in range(3)]
    for n, pfx in zip(nets, ("p0_actor_", "p0_c1_", "p0_c2_")):
        load_params(n, g, pfx)
    actor, c1, c2 = (n.to(DEV) for n in nets)
    olds = [copy.deepcopy(c1), copy.deepcopy(c2)]
    opts = [torch.optim.Adam(m.parameters(), lr=1e-3) for m in (actor, c1, c2)]
    E, cap_ = int(g["cfg_E"]), int(g["cfg_cap"])
    hb = dict(obs=np.asarray(buf.obs), act=np.asarray(buf.act), rew=np.asarray(buf.rew), done=np.asarray(buf.done),
              terminated=np.asarray(buf.terminated), obs_next=np.asarray(buf.obs_next), offset=np.arange(E + 1) * cap_,
              last_index=buf.last_index.copy(), lengths=buf._sizes.copy())
    np.random.seed(3)
    torch.cuda.manual_seed(1234)
    with policy_within_training_step(algo.policy):
        algo.update(buffer=buf, sample_size=int(g["cfg_bs"]))
    torch.cuda.synchronize()
    after_update = torch.cuda.get_rng_state()
    torch.cuda.manual_seed(1234)
    ods.discrete_sac_update(actor, [c1, c2], olds, opts, ods.flat_obs(hb["obs"], DEV), hb, cap["indices"], cap["w"], 0.95, 3, 0.05,
                            0.005, True)
    torch.cuda.synchronize()
    assert torch.equal(after_update, torch.cuda.get_rng_state())
    assert not torch.equal(after_update, (torch.cuda.manual_seed(1234), torch.cuda.get_rng_state())[1])


# ------------------------------------------------------------------------------------------------------------ state_dict
@gpu
@pytest.mark.parametrize("variant", ["auto", "cnn"])
def test_state_dict_round_trip_continues_identically(variant):
    """A fresh algorithm loaded from another's ``state_dict()`` after one update continues bit for bit: online, lagged and
    optimiser state, and AutoAlpha's log_alpha (its torch optimiser's state travels separately, as in the reference)."""
    from tianshou_b200.utils import policy_within_training_step
    g = load_golden(f"dsac_ref_{variant}.npz")
    a, buf_a = build_from_golden(g), buffer_from_golden(g, mirror=False)
    np.random.seed(1)
    with policy_within_training_step(a.policy):
        a.update(buffer=buf_a, sample_size=int(g["cfg_bs"]))
    torch.manual_seed(77)
    b = build_from_golden(g)
    with torch.no_grad():         # different weights before the load, so the load is what makes them equal
        for p in b.parameters():
            p.add_(0.01)
    b.load_state_dict(copy.deepcopy(a.state_dict()))
    if variant == "auto":        # AutoAlpha's own Adam is not one of the algorithm's optimisers (sac.py:168-215, as in the reference)
        b.alpha._optim.load_state_dict(copy.deepcopy(a.alpha._optim.state_dict()))
    for algo in (a, b):          # both continue on fresh, identical buffers with the same draws
        buf = buffer_from_golden(g, mirror=False)
        for u in range(2):
            np.random.seed(10 + u)
            torch.manual_seed(10 + u)
            with policy_within_training_step(algo.policy):
                algo.update(buffer=buf, sample_size=int(g["cfg_bs"]))
    for ga, gb in zip([a._g_actor, *a._g_c, *a._g_ct], [b._g_actor, *b._g_c, *b._g_ct], strict=True):
        assert torch.equal(ga.flat, gb.flat) and torch.equal(ga.exp_avg, gb.exp_avg) and torch.equal(ga.exp_avg_sq, gb.exp_avg_sq)
        assert ga.step == gb.step
    if variant == "auto":
        assert a.alpha._log_alpha.item() == b.alpha._log_alpha.item()


# ------------------------------------------------------------------------------------------------------------ refusals
@gpu
def test_refusals():
    from tianshou_b200.algorithm import AdamOptimizerFactory, DiscreteSAC, RMSpropOptimizerFactory, UnsupportedModelError
    from tianshou_b200.algorithm.modelfree.discrete_sac import DiscreteSACPolicy
    from tianshou_b200.env.atari import DQNet, ScaledObsInputActionReprNet
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.discrete import DiscreteActor, DiscreteCritic
    A = 3
    net = lambda **kw: Net(state_shape=(4,), hidden_sizes=(16,), **kw)

    def make(actor=None, c1=None, c2=None, opt=AdamOptimizerFactory, dev=DEV):
        actor = actor or DiscreteActor(preprocess_net=net(), action_shape=A, softmax_output=False)
        c1 = c1 or DiscreteCritic(preprocess_net=net(), last_size=A)
        return DiscreteSAC(policy=DiscreteSACPolicy(actor=actor.to(dev), action_space=Discrete(A)), policy_optim=opt(lr=1e-3),
                           critic=c1.to(dev), critic_optim=opt(lr=1e-3), critic2=None if c2 is None else c2.to(dev))

    make()      # the supported baseline builds
    # examples/atari/atari_sac.py: one DQNet trunk under the actor and both critics
    trunk = ScaledObsInputActionReprNet(DQNet(4, 36, 36, A, features_only=True, output_dim_added_layer=32))
    with pytest.raises(UnsupportedModelError, match="share parameters"):
        make(DiscreteActor(preprocess_net=trunk, action_shape=A, softmax_output=False),
             DiscreteCritic(preprocess_net=trunk, last_size=A), DiscreteCritic(preprocess_net=trunk, last_size=A))
    shared = net()
    with pytest.raises(UnsupportedModelError, match="share parameters"):
        make(DiscreteActor(preprocess_net=shared, action_shape=A, softmax_output=False), DiscreteCritic(preprocess_net=shared, last_size=A))
    with pytest.raises(UnsupportedModelError, match="softmax_output=True"):
        make(DiscreteActor(preprocess_net=net(), action_shape=A, softmax_output=True))
    with pytest.raises(UnsupportedModelError, match="must read it the same way"):
        make(c1=DiscreteCritic(preprocess_net=ScaledObsInputActionReprNet(net(), denom=2.0), last_size=A))
    with pytest.raises(UnsupportedModelError, match="must read it the same way"):
        make(c1=DiscreteCritic(preprocess_net=Net(state_shape=(5,), hidden_sizes=(16,)), last_size=A))
    with pytest.raises(UnsupportedModelError, match="Adam"):
        make(opt=RMSpropOptimizerFactory)
    with pytest.raises(UnsupportedModelError, match="no CPU path"):
        make(dev="cpu")
    with pytest.raises(UnsupportedModelError, match="critic: .*outside the fused layered-network family"):
        make(c1=DiscreteCritic(preprocess_net=net(norm_layer=torch.nn.LayerNorm), last_size=A))
    with pytest.raises(UnsupportedModelError, match="softmax preprocess"):
        make(c1=DiscreteCritic(preprocess_net=net(softmax=True), last_size=A))
    with pytest.raises(AssertionError):
        DiscreteSACPolicy(actor=DiscreteActor(preprocess_net=net(), action_shape=A, softmax_output=False), action_space=Box(A))


# ------------------------------------------------------------------------------------------------------------ policy
@gpu
def test_policy_forward_mode_and_sample():
    """discrete_sac.py:67-80: the mode outside a training step with deterministic_eval, a sample inside one."""
    from tianshou_b200.algorithm.modelfree.discrete_sac import DiscreteSACPolicy
    from tianshou_b200.data import Batch
    from tianshou_b200.utils import policy_within_training_step
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.discrete import DiscreteActor
    torch.manual_seed(0)
    A = 4
    actor = DiscreteActor(preprocess_net=Net(state_shape=(3,), hidden_sizes=(8,)), action_shape=A, softmax_output=False).to(DEV)
    with torch.no_grad():      # near-uniform probabilities: samples must spread over the actions
        actor.last.model[-1].weight.mul_(0.01)
    policy = DiscreteSACPolicy(actor=actor, action_space=Discrete(A))
    obs = np.random.default_rng(0).standard_normal((2000, 3)).astype(np.float32)
    out = policy(Batch(obs=obs, info=Batch()))
    assert torch.equal(out.act, out.logits.argmax(-1)) and out.dist.probs.shape == (2000, A)
    with policy_within_training_step(policy):
        out = policy(Batch(obs=obs, info=Batch()))
    assert len(set(out.act.cpu().tolist())) == A and not torch.equal(out.act, out.logits.argmax(-1))
    policy.deterministic_eval = False
    out = policy(Batch(obs=obs, info=Batch()))
    assert not torch.equal(out.act, out.logits.argmax(-1))


# ------------------------------------------------------------------------------------------------------------ resources
def test_rows_kernel_has_no_stack_frame_or_spills(tmp_path):
    report = ptxas_report("discrete_sac.cu", tmp_path)
    assert all("discrete_sac_rows_kernel" in e for e in report), report
    assert_spill_free(report)
