"""Shared helpers for the test-suite (golden fixture loading, model construction)."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def load_golden(name: str):
    return np.load(os.path.join(GOLDEN, name), allow_pickle=False)


PARAM_ORDER = ["a_w1", "a_b1", "a_w2", "a_b2", "a_w3", "a_b3", "a_logstd",
               "c_w1", "c_b1", "c_w2", "c_b2", "c_w3", "c_b3"]


class Box:
    """Minimal stand-in for gymnasium.spaces.Box (gymnasium is not a dependency)."""

    def __init__(self, dim: int, m: float = 1.0):
        self.shape = (dim,)
        self.low = -m * np.ones(dim, np.float32)
        self.high = m * np.ones(dim, np.float32)


def build_actor_critic(obs_dim: int, act_dim: int, device, seed: int = 0):
    import torch

    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.continuous import ContinuousActorProbabilistic, ContinuousCritic

    torch.manual_seed(seed)
    net_a = Net(state_shape=(obs_dim,), hidden_sizes=(64, 64), activation=torch.nn.Tanh)
    actor = ContinuousActorProbabilistic(preprocess_net=net_a, action_shape=(act_dim,), unbounded=True).to(device)
    net_c = Net(state_shape=(obs_dim,), hidden_sizes=(64, 64), activation=torch.nn.Tanh)
    critic = ContinuousCritic(preprocess_net=net_c).to(device)
    torch.nn.init.constant_(actor.sigma_param, -0.5)
    for m in list(actor.modules()) + list(critic.modules()):
        if isinstance(m, torch.nn.Linear):
            torch.nn.init.orthogonal_(m.weight, gain=np.sqrt(2))
            torch.nn.init.zeros_(m.bias)
    for m in actor.mu.modules():
        if isinstance(m, torch.nn.Linear):
            torch.nn.init.zeros_(m.bias)
            m.weight.data.copy_(0.01 * m.weight.data)
    return actor, critic


def named_params(actor, critic):
    import torch
    a1, a2 = [m for m in actor.preprocess.model.model if isinstance(m, torch.nn.Linear)]
    c1, c2 = [m for m in critic.preprocess.model.model if isinstance(m, torch.nn.Linear)]
    a3, c3 = actor.mu.model[0], critic.last.model[0]
    return {"a_w1": a1.weight, "a_b1": a1.bias, "a_w2": a2.weight, "a_b2": a2.bias, "a_w3": a3.weight,
            "a_b3": a3.bias, "a_logstd": actor.sigma_param, "c_w1": c1.weight, "c_b1": c1.bias, "c_w2": c2.weight,
            "c_b2": c2.bias, "c_w3": c3.weight, "c_b3": c3.bias}


def load_params(actor, critic, values: dict) -> None:
    import torch
    with torch.no_grad():
        for k, p in named_params(actor, critic).items():
            p.copy_(torch.as_tensor(values[k]).reshape(p.shape))


def gaussian_dist(loc_scale):
    import torch
    loc, scale = loc_scale
    return torch.distributions.Independent(torch.distributions.Normal(loc, scale), 1)


def build_ppo(obs_dim, act_dim, device, lr=3e-4, params=None, **kw):
    from tianshou_b200.algorithm import PPO, AdamOptimizerFactory, ProbabilisticActorPolicy
    actor, critic = build_actor_critic(obs_dim, act_dim, device)
    if params is not None:
        load_params(actor, critic, params)
    policy = ProbabilisticActorPolicy(actor=actor, dist_fn=gaussian_dist, action_scaling=True,
                                      action_bound_method="clip", action_space=Box(act_dim))
    algo = PPO(policy=policy, critic=critic, optim=AdamOptimizerFactory(lr=lr), **kw)
    return algo, actor, critic


def perturb_params(actor, critic, seed: int = 0) -> None:
    """Move the parameters of ``build_actor_critic`` away from values that hide indexing bugs: every bias ~ N(0, 0.3)
    (zero biases cannot tell one bias column from another), a distinct log-std per action dimension (a constant log-std
    cannot tell one dimension's 1 / sigma^2 from another's) and the actor head at full orthogonal scale instead of x0.01
    (so mu depends on the observation and the ratios spread over the clip range).  In place: works on the flat views."""
    import torch
    g = torch.Generator(device="cpu").manual_seed(seed)
    named = named_params(actor, critic)
    with torch.no_grad():
        for k, p in named.items():
            if k[2] == "b":
                p.copy_(0.3 * torch.randn(p.shape, generator=g, dtype=torch.float64))
        ls = named["a_logstd"]
        ls.copy_(torch.linspace(-1.2, 0.3, ls.numel(), dtype=torch.float64).reshape(ls.shape))
        named["a_w3"].mul_(100.0)


def param_offsets(flat, actor, critic) -> dict:
    """Offset of every module parameter inside the flat parameter buffer (the parameters are views of it)."""
    base = flat.data_ptr()
    return {k: (p.data.data_ptr() - base) // 4 for k, p in named_params(actor, critic).items()}


def ppo_reference_fp64(actor, critic, mb: dict, hp: dict) -> dict:
    """One minibatch of the PPO / A2C loss (modelfree/ppo.py:183-211, modelfree/a2c.py:262-266) in float64 with torch
    autograd on CPU, on deep copies of the SAME modules (their Linear layers and log-std parameter, so the gradients
    come back under the modules' own parameter names).  Independent of oracle_np's hand-written backward.

    mb: obs, act, adv, returns, logp_old, v_s (numpy).  hp: eps_clip, dual_clip (None / 0 = off), value_clip,
    advantage_normalization, adv_eps, vf_coef, ent_coef, loss_kind ("ppo" | "a2c").
    Returns v, mu, logp, ratio, value delta (value - v_s), the loss parts (loss, clip, vf, ent) and ``grads`` (13 arrays)."""
    import copy

    import torch
    a = copy.deepcopy(actor).to("cpu", torch.float64)
    c = copy.deepcopy(critic).to("cpu", torch.float64)
    t = {k: torch.as_tensor(np.asarray(v), dtype=torch.float64) for k, v in mb.items()}
    obs = t["obs"]
    # the modules' forward casts observations to float32; run their layers directly in float64 instead
    mu = a.mu.model(a.preprocess.model.model(obs))
    sigma = a.sigma_param.reshape(-1).exp().expand_as(mu)
    dist = torch.distributions.Independent(torch.distributions.Normal(mu, sigma), 1)
    logp = dist.log_prob(t["act"])
    value = c.last.model(c.preprocess.model.model(obs)).flatten()
    adv = t["adv"]
    ratio = (logp - t["logp_old"]).exp()
    if hp.get("loss_kind", "ppo") == "a2c":
        clip_loss = -(logp * adv).mean()
    else:
        if hp["advantage_normalization"]:
            adv = (adv - adv.mean()) / (adv.std() + hp["adv_eps"])          # torch std: ddof = 1
        eps = hp["eps_clip"]
        surr1, surr2 = ratio * adv, ratio.clamp(1.0 - eps, 1.0 + eps) * adv
        obj = torch.min(surr1, surr2)
        if hp.get("dual_clip"):
            obj = torch.where(adv < 0, torch.max(obj, hp["dual_clip"] * adv), obj)
        clip_loss = -obj.mean()
    R, vs = t["returns"], t["v_s"]
    if hp.get("value_clip"):
        v_clip = vs + (value - vs).clamp(-hp["eps_clip"], hp["eps_clip"])
        vf_loss = torch.max((R - value).pow(2), (R - v_clip).pow(2)).mean()
    else:
        vf_loss = (R - value).pow(2).mean()
    ent = dist.entropy().mean()
    loss = clip_loss + hp["vf_coef"] * vf_loss - hp["ent_coef"] * ent
    loss.backward()
    grads = {k: p.grad.numpy().copy() for k, p in named_params(a, c).items()}
    d = lambda x: x.detach().numpy().copy()
    return dict(v=d(value), mu=d(mu), logp=d(logp), ratio=d(ratio), delta=d(value - vs), loss=loss.item(),
                clip=clip_loss.item(), vf=vf_loss.item(), ent=ent.item(), grads=grads)


F32_EPS = float(np.finfo(np.float32).eps)


def sum_length_rel(rows: int) -> float:
    """The accumulation term of a sum over ``rows`` rows, as a fraction of the result's largest value.  It is the bound
    test_net_gpu documents for ``ts_net_gemm``: one fp32 accumulator takes (rows / 16) x 6 MMA additions, each rounding by up to
    2^-24.  It passes the 1e-4 of the gradient bars only beyond about 4,400 rows."""
    return (int(rows) + 15) // 16 * 6 * 2.0 ** -24


def ac_named_params(actor, critic) -> dict:
    """``named_params`` for every actor-critic the fused kernels accept: Gaussian (``mu`` head + ``a_logstd``) or
    categorical (DiscreteActor, ``last`` head, no log-std) and separate or shared trunks.  A shared trunk has one set of
    slots, reported under the ``a_*`` names only."""
    import torch
    a1, a2 = [m for m in actor.preprocess.model.model if isinstance(m, torch.nn.Linear)]
    c1, c2 = [m for m in critic.preprocess.model.model if isinstance(m, torch.nn.Linear)]
    categorical = hasattr(actor, "softmax_output")
    a3 = actor.last.model[0] if categorical else actor.mu.model[0]
    d = {"a_w1": a1.weight, "a_b1": a1.bias, "a_w2": a2.weight, "a_b2": a2.bias, "a_w3": a3.weight, "a_b3": a3.bias}
    if not categorical:
        d["a_logstd"] = actor.sigma_param
    if c1 is not a1:
        d.update({"c_w1": c1.weight, "c_b1": c1.bias, "c_w2": c2.weight, "c_b2": c2.bias})
    c3 = critic.last.model[0]
    d.update({"c_w3": c3.weight, "c_b3": c3.bias})
    return d


def actor_critic_reference_fp64(actor, critic, mb: dict, hp: dict, group_order: bool = False) -> dict:
    """``ppo_reference_fp64`` for the whole fused family: Tanh or ReLU trunks, a shared trunk (actor and critic copied
    together, so autograd adds both losses' gradients into the same leaves) and the categorical head as
    ``Categorical(probs=softmax(z))`` computes it -- renormalise, clamp with the FLOAT32 eps the reference's fp32 run
    uses (torch's own ``clamp_probs`` would take the float64 eps here), log.  Runs the modules' own Linear layers in
    float64 on CPU.  Returns v, mu (Gaussian: the mean; categorical: softmax(z) before renormalisation), pn (categorical:
    the renormalised probabilities), logp, the loss parts and ``grads`` keyed like ``ac_named_params``, or with
    ``group_order`` (networks of any depth) one flat float64 vector in ``ActorCritic(actor, critic).parameters()`` order,
    a shared trunk once -- the layout of the layer-wise path's ``FlatGroup``."""
    import copy

    import torch
    a, c = copy.deepcopy((actor, critic))        # one deepcopy: a shared trunk stays shared
    a.to("cpu", torch.float64)
    c.to("cpu", torch.float64)
    t = {k: torch.as_tensor(np.asarray(v), dtype=torch.float64) for k, v in mb.items()}
    obs = t["obs"]
    categorical = hasattr(a, "softmax_output")
    pn = None
    if categorical:
        z = a.last.model(a.preprocess.model.model(obs))
        mu = torch.softmax(z, dim=-1)
        pn = mu / mu.sum(-1, keepdim=True)
        lg = torch.log(pn.clamp(F32_EPS, 1.0 - F32_EPS))
        act = t["act"].reshape(obs.shape[0], -1)[:, 0].long()
        logp = lg.gather(1, act.view(-1, 1)).view(-1)
        ent = -(pn * lg).sum(-1)
    else:
        mu = a.mu.model(a.preprocess.model.model(obs))
        sigma = a.sigma_param.reshape(-1).exp().expand_as(mu)
        dist = torch.distributions.Independent(torch.distributions.Normal(mu, sigma), 1)
        logp = dist.log_prob(t["act"])
        ent = dist.entropy()
    value = c.last.model(c.preprocess.model.model(obs)).flatten()
    adv = t["adv"]
    ratio = (logp - t["logp_old"]).exp()
    if hp.get("loss_kind", "ppo") == "a2c":
        clip_loss = -(logp * adv).mean()
    else:
        if hp["advantage_normalization"]:
            adv = (adv - adv.mean()) / (adv.std() + hp["adv_eps"])
        eps = hp["eps_clip"]
        obj = torch.min(ratio * adv, ratio.clamp(1.0 - eps, 1.0 + eps) * adv)
        if hp.get("dual_clip"):
            obj = torch.where(adv < 0, torch.max(obj, hp["dual_clip"] * adv), obj)
        clip_loss = -obj.mean()
    R, vs = t["returns"], t["v_s"]
    if hp.get("value_clip"):
        v_clip = vs + (value - vs).clamp(-hp["eps_clip"], hp["eps_clip"])
        vf_loss = torch.max((R - value).pow(2), (R - v_clip).pow(2)).mean()
    else:
        vf_loss = (R - value).pow(2).mean()
    ent = ent.mean()
    loss = clip_loss + hp["vf_coef"] * vf_loss - hp["ent_coef"] * ent
    loss.backward()
    if group_order:
        from tianshou_b200.utils.net.common import ActorCritic
        grads = np.concatenate([p.grad.numpy().reshape(-1) for p in ActorCritic(a, c).parameters()])
    else:
        grads = {k: p.grad.numpy().copy() for k, p in ac_named_params(a, c).items()}
    d = lambda x: None if x is None else x.detach().numpy().copy()
    return dict(v=d(value), mu=d(mu), pn=d(pn), logp=d(logp), loss=loss.item(), clip=clip_loss.item(), vf=vf_loss.item(),
                ent=ent.item(), grads=grads)


def restore_vector_buffer(g, prefix: str, E: int, cap: int, device=None):
    """Rebuild a tianshou_b200 VectorReplayBuffer in the exact state stored in a golden file."""
    from tianshou_b200.data import Batch, VectorReplayBuffer
    buf = VectorReplayBuffer(E * cap, E, device=device)
    meta = Batch(obs=g[prefix + "buf_obs"].copy(), act=g[prefix + "buf_act"].copy(), rew=g[prefix + "buf_rew"].copy(),
                 terminated=g[prefix + "buf_terminated"].copy(), truncated=g[prefix + "buf_truncated"].copy(),
                 done=g[prefix + "buf_done"].copy(), obs_next=g[prefix + "buf_obs_next"].copy())
    buf.set_batch(meta)
    set_buffer_state(buf, g[prefix + "meta_last_index"], g[prefix + "meta_lengths"])
    return buf


def set_buffer_state(buf, last_index, lengths) -> None:
    buf.last_index[:] = last_index
    buf._sizes[:] = lengths
    buf._ins[:] = np.where(lengths > 0, (last_index - buf._offset + 1) % buf._cap, 0)
    buf._touch()


def synth_rollout(rng, E, steps, obs_dim, act_dim, p_term=1e-3, trunc_len=1000):
    """Synthetic HalfCheetah-shaped rollout (SURVEY 8d); yields per-step dicts of [E, ...] arrays."""
    t_in_ep = np.zeros(E, dtype=np.int64)
    obs = rng.standard_normal((E, obs_dim)).astype(np.float32)
    for _ in range(steps):
        act = rng.standard_normal((E, act_dim)).astype(np.float32)
        rew = rng.standard_normal(E)
        obs_next = rng.standard_normal((E, obs_dim)).astype(np.float32)
        term = rng.random(E) < p_term
        t_in_ep += 1
        trunc = (t_in_ep >= trunc_len) & ~term
        yield dict(obs=obs, act=act, rew=rew, terminated=term, truncated=trunc, obs_next=obs_next)
        done = term | trunc
        t_in_ep[done] = 0
        obs = np.where(done[:, None], rng.standard_normal((E, obs_dim)).astype(np.float32), obs_next)


# ---- observed-error bookkeeping: every parity test records what it measured; tests/conftest.py dumps the table to
# parity_report.json at the end of the session
PARITY: dict = {}


def record_parity(key: str, got, ref, rtol: float, atol: float) -> dict:
    """Assert ``|got - ref| <= atol + rtol * |ref|`` elementwise and record the observed errors under ``key``."""
    got = np.asarray(got, dtype=np.float64)
    ref = np.asarray(ref, dtype=np.float64)
    assert got.shape == ref.shape, f"{key}: shape {got.shape} vs {ref.shape}"
    err = np.abs(got - ref)
    scale = float(np.abs(ref).max()) if ref.size else 0.0
    worst = float((err - (atol + rtol * np.abs(ref))).max()) if ref.size else 0.0
    e = {"n": int(ref.size), "max_abs_err": float(err.max()) if ref.size else 0.0, "max_abs_ref": scale,
         "max_err_over_max_ref": float(err.max() / scale) if scale > 0 else 0.0,
         "rtol": rtol, "atol": atol, "margin": -worst, "ok": bool(worst <= 0.0)}
    prev = PARITY.get(key)
    if prev is None or e["max_err_over_max_ref"] >= prev["max_err_over_max_ref"]:
        PARITY[key] = e
    assert worst <= 0.0, (f"{key}: max |err| {e['max_abs_err']:.3e} (max |ref| {scale:.3e}, ratio {e['max_err_over_max_ref']:.3e}) "
                          f"exceeds atol {atol:g} + rtol {rtol:g} * |ref| by {worst:.3e}")
    return e
