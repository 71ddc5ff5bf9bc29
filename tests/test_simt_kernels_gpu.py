"""The fp32 SIMT actor-critic kernels (csrc/mlp.cu: critic_forward_kernel, actor_logp_kernel, ppo_grad_kernel,
grad_reduce_kernel, clip_adam_kernel) against float64 references, over every model family that runs them: categorical
heads, ReLU trunks, shared trunks, and tanh Gaussian networks wider than the tensor-core kernels' obs <= 32.

Every case asserts that it really runs the SIMT kernels (no layer-wise path, no weight image of the tensor-core
update).  The inputs reach the edges where these kernels can go wrong: observation widths that are not multiples of 4
(the zero-padded rows of the staged W1), more tiles than one wave of CTAs, softmax rows deep in the clamp of torch's
Categorical (some of them taking a clamped action), ReLU pre-activations that are exactly zero, and -- for
clip_adam_kernel -- every branch of its partial-row fold, the gradient clip and weight decay."""
import copy
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import oracle_np as onp
from test_tc_shapes_gpu import HP_SETS
from ts_testutil import (F32_EPS, Box, ac_named_params, actor_critic_reference_fp64, gaussian_dist, record_parity,
                         synth_rollout)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

# relu / categorical head / one preprocess Net for actor and critic, and the (obs, act) shapes of each family.  obs 1 / 5 /
# 11 / 17 / 27 / 33 are not multiples of 4; (60, 16) and (64, 4) are the largest training tiles that fit in 227 KB
FAMILIES = {
    "tanh_gauss": dict(relu=False, cat=False, shared=False, shapes=[(33, 1), (40, 5), (60, 16), (64, 4)]),
    "relu_gauss": dict(relu=True, cat=False, shared=False, shapes=[(1, 1), (5, 3), (17, 6), (64, 4)]),
    "tanh_gauss_shared": dict(relu=False, cat=False, shared=True, shapes=[(11, 3), (17, 6)]),
    "relu_cat_shared": dict(relu=True, cat=True, shared=True, shapes=[(4, 2), (6, 3), (8, 4), (60, 16)]),
    "relu_cat": dict(relu=True, cat=True, shared=False, shapes=[(4, 2), (27, 9)]),
    "tanh_cat": dict(relu=False, cat=True, shared=False, shapes=[(4, 2), (17, 16)]),
}
CASES = [(f, o, a) for f, spec in FAMILIES.items() for o, a in spec["shapes"]]
CASE_IDS = [f"{f}-obs{o}-act{a}" for f, o, a in CASES]


class _Discrete:
    def __init__(self, n):
        self.n = n


def _sms() -> int:
    return torch.cuda.get_device_properties(0).multi_processor_count


def _perturb(actor, critic, spec, seed):
    """Parameters that expose indexing bugs: orthogonal weights at gain sqrt(2) (the actor head at full scale), every bias
    ~ N(0, 0.3), a distinct log-std per action dimension.  ReLU trunks get every eighth b1 entry exactly 0 (with an
    all-zero observation row, z1 = 0 exactly there in both precisions, where torch's ReLU derivative is 0).  A tanh
    categorical head is 16x wider, so that saturated trunk outputs can separate its logits by 30 and more."""
    g = torch.Generator().manual_seed(seed)
    torch.manual_seed(seed)
    with torch.no_grad():
        for k, p in ac_named_params(actor, critic).items():
            if k == "a_logstd":
                p.copy_(torch.linspace(-1.2, 0.3, p.numel()).reshape(p.shape))
            elif k[2] == "w":
                w = torch.empty(p.shape)
                torch.nn.init.orthogonal_(w, gain=np.sqrt(2))
                if k == "a_w3" and spec["cat"] and not spec["relu"]:
                    w *= 16.0
                p.copy_(w)
            else:
                b = 0.3 * torch.randn(p.shape, generator=g)
                if k[2:] == "b1" and spec["relu"]:
                    b[::8] = 0.0
                p.copy_(b)


def _build(family, obs_dim, act_dim, algo_kind="ppo", lr=3e-4, weight_decay=0.0, **kw):
    from tianshou_b200.algorithm import A2C, PPO, AdamOptimizerFactory, DiscreteActorPolicy, ProbabilisticActorPolicy
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.continuous import ContinuousActorProbabilistic, ContinuousCritic
    from tianshou_b200.utils.net.discrete import DiscreteActor, DiscreteCritic
    spec = FAMILIES[family]
    seed = obs_dim * 100 + act_dim
    torch.manual_seed(seed)
    act_fn = torch.nn.ReLU if spec["relu"] else torch.nn.Tanh
    net_a = Net(state_shape=(obs_dim,), hidden_sizes=(64, 64), activation=act_fn)
    net_c = net_a if spec["shared"] else Net(state_shape=(obs_dim,), hidden_sizes=(64, 64), activation=act_fn)
    if spec["cat"]:
        actor = DiscreteActor(preprocess_net=net_a, action_shape=(act_dim,)).to(DEV)
        critic = DiscreteCritic(preprocess_net=net_c).to(DEV)
        policy = DiscreteActorPolicy(actor=actor, dist_fn=torch.distributions.Categorical, action_space=_Discrete(act_dim))
    else:
        actor = ContinuousActorProbabilistic(preprocess_net=net_a, action_shape=(act_dim,), unbounded=True).to(DEV)
        critic = ContinuousCritic(preprocess_net=net_c).to(DEV)
        policy = ProbabilisticActorPolicy(actor=actor, dist_fn=gaussian_dist, action_scaling=True, action_bound_method="clip",
                                          action_space=Box(act_dim))
    _perturb(actor, critic, spec, seed)
    cls = A2C if algo_kind == "a2c" else PPO
    algo = cls(policy=policy, critic=critic, optim=AdamOptimizerFactory(lr=lr, weight_decay=weight_decay), **kw)
    return algo, actor, critic


def _assert_simt(algo, family):
    """The case must run mlp.cu: not the layer-wise path, not the tensor-core update (no weight image)."""
    assert algo._layered is None and algo._flat.weight_image is None, f"{family}: not on the SIMT kernels"
    d = algo._desc
    assert (d.c_w1 == d.a_w1) == FAMILIES[family]["shared"]


def _offsets(flat, actor, critic) -> dict:
    base = flat.data_ptr()
    return {k: (p.data.data_ptr() - base) // 4 for k, p in ac_named_params(actor, critic).items()}


class _Fp64:
    """float64 copies of the modules, used to CHOOSE inputs (the yardstick is actor_critic_reference_fp64)."""

    def __init__(self, actor, critic, spec):
        self.a, self.c = copy.deepcopy((actor, critic))
        self.a.to("cpu", torch.float64)
        self.c.to("cpu", torch.float64)
        self.spec = spec
        self.trunks = [self.a.preprocess.model.model] + ([] if spec["shared"] else [self.c.preprocess.model.model])

    @torch.no_grad()
    def near_kink(self, obs):
        """Rows with a ReLU pre-activation within rounding distance of 0 (3e-5 of the sum of its terms' magnitudes:
        fp32 and fp64 may take different sides there).  Exact zeros are the deliberate ones and do not count."""
        x0 = torch.as_tensor(np.asarray(obs, np.float64))
        bad = torch.zeros(x0.shape[0], dtype=torch.bool)
        for seq in self.trunks:
            h = x0
            for m in seq:
                if isinstance(m, torch.nn.Linear):
                    z = m(h)
                    mag = h.abs() @ m.weight.abs().T + m.bias.abs()
                    bad |= ((z.abs() < 3e-5 * mag) & (z != 0)).any(1)
                    h = z
                else:
                    h = m(h)
        return bad.numpy()

    @torch.no_grad()
    def head(self, obs):
        x = torch.as_tensor(np.asarray(obs, np.float64))
        out = (self.a.last if self.spec["cat"] else self.a.mu).model(self.a.preprocess.model.model(x))
        return out.numpy()

    def probs(self, obs):
        z = self.head(obs)
        p = np.exp(z - z.max(1, keepdims=True))
        return p / p.sum(1, keepdims=True), z


def _saturated_rows(rng, f64, obs_dim, k):
    """Up to k large-magnitude observation rows whose fp64 logits separate by >= 30 (every other probability < 1e-13,
    far below the clamp at eps = 1.2e-7), none of them near a ReLU kink."""
    out = []
    for _ in range(40):
        x = (rng.standard_normal((4096, obs_dim)) * rng.uniform(5.0, 60.0, (4096, 1))).astype(np.float32)
        z = np.sort(f64.head(x), 1)
        ok = z[:, -1] - z[:, -2] >= 30.0
        if f64.spec["relu"]:
            ok &= ~f64.near_kink(x)
        out.extend(x[ok])
        if len(out) >= k:
            break
    return np.array(out[:k], dtype=np.float32).reshape(-1, obs_dim)


def _actions(rng, f64, obs, act_dim, sigma):
    if f64.spec["cat"]:
        pn, _ = f64.probs(obs)
        act = np.minimum((pn.cumsum(1) < rng.random((len(obs), 1))).sum(1), act_dim - 1)
        return act.astype(np.float32)
    return (f64.head(obs) + sigma * rng.standard_normal((len(obs), act_dim))).astype(np.float32)


def _inputs(rng, actor, critic, family, obs_dim, act_dim, n, hp, edges=True):
    """n minibatch rows around the current policy.  Edges: categorical heads get large-magnitude rows whose logits
    separate by >= 30, half of them taking a clamped action; ReLU trunks get all-zero observation rows.  Regular rows are
    redrawn until no probability lies within 4x of eps or 1 - eps and no ReLU pre-activation lies within rounding
    distance of 0.  Branch guard of test_tc_shapes_gpu / test_layered_gpu: no ratio within 1e-4 of 1 +- eps_clip (or of
    the dual clip), no value delta within 1e-4 of +-eps_clip and no two clipped value errors within 1e-4 of each other,
    so fp32 and fp64 take the same side of every clip, min and max.  Returns (mb, kind): kind 0 regular, 1 saturated,
    2 all-zero."""
    spec = FAMILIES[family]
    f64 = _Fp64(actor, critic, spec)
    sigma = None if spec["cat"] else np.exp(ac_named_params(actor, critic)["a_logstd"].detach().cpu().numpy().reshape(-1))
    obs = rng.standard_normal((n, obs_dim)).astype(np.float32)
    kind = np.zeros(n, dtype=np.int64)
    if edges and spec["cat"]:
        sat = _saturated_rows(rng, f64, obs_dim, min(max(8, n // 8), 64))
        rows = rng.choice(n, len(sat), replace=False)
        obs[rows], kind[rows] = sat, 1
    if edges and spec["relu"]:
        rows = rng.choice(np.nonzero(kind == 0)[0], 3, replace=False)
        obs[rows], kind[rows] = 0.0, 2
    for _ in range(100):
        bad = np.zeros(n, dtype=bool)
        if spec["relu"]:
            bad |= f64.near_kink(obs)
        if spec["cat"]:
            pn, _ = f64.probs(obs)
            near = ((pn > F32_EPS / 4) & (pn < 4 * F32_EPS)) | ((1 - pn > F32_EPS / 4) & (1 - pn < 4 * F32_EPS))
            bad |= near.any(1) & (kind != 1)
        if not bad.any():
            break
        kind[bad] = 0           # an all-zero row next to a kink in layer 2 becomes a regular row
        obs[bad] = rng.standard_normal((int(bad.sum()), obs_dim)).astype(np.float32)
    assert not bad.any()
    act = _actions(rng, f64, obs, act_dim, sigma)
    if spec["cat"]:
        pn, _ = f64.probs(obs)
        for j, r in enumerate(np.nonzero(kind == 1)[0]):
            if j % 2 == 0:       # a clamped action: any but the top one
                top = int(np.argmax(pn[r]))
                act[r] = (top + 1 + rng.integers(0, act_dim - 1)) % act_dim
    adv = rng.standard_normal(n).astype(np.float32)
    ret = rng.standard_normal(n).astype(np.float32)
    zeros = np.zeros(n)
    mb = dict(obs=obs, act=act, adv=adv, returns=ret, logp_old=zeros, v_s=zeros)
    ref = actor_critic_reference_fp64(actor, critic, mb, dict(loss_kind="a2c", vf_coef=0.5, ent_coef=0.0))
    logp, v = ref["logp"], ref["v"]
    lpo = (logp + 0.5 * rng.standard_normal(n)).astype(np.float32)
    v_s = (v + 0.3 * rng.standard_normal(n)).astype(np.float32)
    e, dual = hp.get("eps_clip", 0.0), hp.get("dual_clip") or 0.0
    A = adv.astype(np.float64)
    if hp.get("advantage_normalization"):
        A = (A - A.mean()) / (A.std(ddof=1) + 1e-8)
    for _ in range(100):
        ratio = np.exp(logp - lpo.astype(np.float64))
        bad = (np.abs(ratio - (1 - e)) < 1e-4) | (np.abs(ratio - (1 + e)) < 1e-4)
        if dual:
            bad |= np.abs(np.minimum(ratio * A, np.clip(ratio, 1 - e, 1 + e) * A) - dual * A) < 1e-4
        if not bad.any():
            break
        lpo[bad] = (logp[bad] + 0.5 * rng.standard_normal(int(bad.sum()))).astype(np.float32)
    for _ in range(100):
        dl = v - v_s.astype(np.float64)
        vc = v_s + np.clip(dl, -e, e)
        tie = (np.abs(dl) > e) & (np.abs(np.abs(ret - v) - np.abs(ret - vc)) < 1e-4)
        bad = (np.abs(np.abs(dl) - e) < 1e-4) | tie
        if not bad.any():
            break
        v_s[bad] = (v[bad] + 0.3 * rng.standard_normal(int(bad.sum()))).astype(np.float32)
    mb.update(logp_old=lpo, v_s=v_s)
    return mb, kind


def _assert_edges_reached(family, ref, mb, kind, min_rows):
    """The categorical clamp and the ReLU zeros must really be in the batch, or the test quietly stops testing them."""
    spec = FAMILIES[family]
    if spec["cat"]:
        low = ref["pn"] < F32_EPS / 4
        act = mb["act"].astype(np.int64)
        assert int(low.any(1).sum()) >= min_rows, f"only {int(low.any(1).sum())} rows reach the clamp"
        assert low[np.arange(len(act)), act].any(), "no row takes a clamped action"
    if spec["relu"]:
        assert (kind == 2).any(), "no all-zero observation row survived the kink guard"


# --------------------------------------------------------------------------------------------- forward kernels
def _torch_fp32(actor, critic, obs, act, spec):
    """torch's own fp32 evaluation of the same layers (CPU): the yardstick for what fp32 can achieve."""
    a, c = copy.deepcopy((actor, critic))
    a.cpu(), c.cpu()
    x = torch.from_numpy(obs)
    with torch.no_grad():
        v = c.last.model(c.preprocess.model.model(x)).flatten()
        if spec["cat"]:
            p = torch.softmax(a.last.model(a.preprocess.model.model(x)), -1)
            pn = p / p.sum(-1, keepdim=True)
            lg = torch.log(pn.clamp(F32_EPS, 1 - F32_EPS))
            lp = lg.gather(1, torch.from_numpy(act).long().view(-1, 1)).view(-1)
            return v.numpy(), p.numpy(), lp.numpy()
        mu = a.mu.model(a.preprocess.model.model(x))
        sigma = a.sigma_param.reshape(-1).exp()
        lp = torch.distributions.Normal(mu, sigma).log_prob(torch.from_numpy(act)).sum(-1)
        return v.numpy(), mu.numpy(), lp.numpy()


@pytest.mark.parametrize("family,obs_dim,act_dim", CASES, ids=CASE_IDS)
def test_forward_kernels_vs_fp64(family, obs_dim, act_dim):
    """ts_critic_forward with two inputs and ts_actor_logp with mu_out (categorical: softmax(z) before renormalisation) at
    one row, at and around one tile, and past two waves of CTAs."""
    from tianshou_b200 import ops
    spec = FAMILIES[family]
    algo, actor, critic = _build(family, obs_dim, act_dim)
    _assert_simt(algo, family)
    f64 = _Fp64(actor, critic, spec)
    sigma = None if spec["cat"] else np.exp(ac_named_params(actor, critic)["a_logstd"].detach().cpu().numpy().reshape(-1))
    rng = np.random.default_rng(obs_dim * 31 + act_dim)
    hp0 = dict(loss_kind="a2c", vf_coef=0.5, ent_coef=0.0)
    for n in (1, 127, 128, 129, 2 * _sms() * 128 + 5):
        obs = rng.standard_normal((n, obs_dim)).astype(np.float32)
        obs2 = rng.standard_normal((n, obs_dim)).astype(np.float32)
        act = _actions(rng, f64, obs, act_dim, sigma)
        z = np.zeros(n)
        ref = actor_critic_reference_fp64(actor, critic, dict(obs=obs, act=act, adv=z, returns=z, logp_old=z, v_s=z), hp0)
        ref2 = actor_critic_reference_fp64(actor, critic, dict(obs=obs2, act=act, adv=z, returns=z, logp_old=z, v_s=z), hp0)
        v1, v2 = ops.critic_forward(algo._flat.flat, algo._desc, torch.from_numpy(obs).to(DEV), torch.from_numpy(obs2).to(DEV))
        lp, mu = ops.actor_logp(algo._flat.flat, algo._desc, torch.from_numpy(obs).to(DEV), torch.from_numpy(act).to(DEV),
                                want_mu=True)
        v32, mu32, lp32 = _torch_fp32(actor, critic, obs, act, spec)
        v32b = _torch_fp32(actor, critic, obs2, act, spec)[0]
        tag = f"simt_fwd/{family}/{obs_dim}x{act_dim}/n{n}"
        for name, got, want, f32 in (("v", v1, ref["v"], v32), ("v_second", v2, ref2["v"], v32b), ("mu", mu, ref["mu"], mu32),
                                     ("logp", lp, ref["logp"], lp32)):
            scale = float(np.abs(want).max())
            err_torch = float(np.abs(f32.astype(np.float64) - want).max())
            # 8x torch fp32's own error against fp64, plus a floor of 4e-6 of max |ref| for the cases where torch's error
            # is accidentally tiny (one row): one 64-term fp32 dot product summed in another order than torch's GEMM can
            # be up to 64 x 2^-24 = 3.8e-6 of the sum of its terms' magnitudes away
            record_parity(f"{tag}/{name}", got.cpu().numpy(), want, rtol=0.0, atol=8.0 * err_torch + 4e-6 * scale)


# ------------------------------------------------------------------------------------------- ts_ppo_grad
def _grad_case(family, obs_dim, act_dim, hp_name, B, n_total, lo, tag):
    from tianshou_b200._cabi import call, ptr, stream_ptr
    cfg = dict(HP_SETS[hp_name])
    kind_ = cfg.pop("algo")
    if kind_ == "a2c":
        algo, actor, critic = _build(family, obs_dim, act_dim, "a2c", **cfg)
        hpr = dict(loss_kind="a2c", vf_coef=cfg["vf_coef"], ent_coef=cfg["ent_coef"], advantage_normalization=False)
    else:
        algo, actor, critic = _build(family, obs_dim, act_dim, **cfg)
        hpr = dict(cfg, adv_eps=1e-8)
    _assert_simt(algo, family)
    hp = algo._loss_hparams()
    rng = np.random.default_rng(obs_dim * 7 + act_dim + B)
    mb, kind = _inputs(rng, actor, critic, family, obs_dim, act_dim, B, hpr)
    ref = actor_critic_reference_fp64(actor, critic, mb, hpr)
    _assert_edges_reached(family, ref, mb, kind, min_rows=8)
    # the minibatch sits at permuted positions [lo, lo + B) of a larger rollout; the other rows are never read
    perm = rng.permutation(n_total).astype(np.int32)
    idx = perm[lo:lo + B]
    full = {}
    for k, v in mb.items():
        arr = np.zeros((n_total,) + v.shape[1:], dtype=np.float32)
        arr[idx] = v
        full[k] = arr
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    f = algo._flat
    d = {k: t(full[k]) for k in ("obs", "act", "adv", "returns", "logp_old", "v_s")}
    d_perm = t(perm)
    adv_mom = None
    if hp.advantage_normalization:
        sums = torch.zeros(2, dtype=torch.float64, device=DEV)
        adv_mom = torch.zeros(2, dtype=torch.float32, device=DEV)
        call("ts_minibatch_adv_sums", ptr(d["adv"]), ptr(d_perm), lo, lo + B, ptr(sums), stream_ptr())
        call("ts_adv_moments_finalize", ptr(sums), B, ptr(adv_mom), stream_ptr())
    f.partials.fill_(float("nan"))      # every row the fold reads must have been written by the kernel
    f.grad.fill_(float("nan"))
    n_part = C.c_int32(0)
    call("ts_ppo_grad", ptr(f.flat), C.byref(algo._desc), C.byref(hp), ptr(d["obs"]), ptr(d["act"]), ptr(d["adv"]),
         ptr(d["returns"]), ptr(d["logp_old"]), ptr(d["v_s"]), ptr(d_perm), lo, lo + B, B, ptr(adv_mom), ptr(f.partials),
         C.byref(n_part), stream_ptr())
    assert n_part.value == min((B + 127) // 128, _sms())
    call("ts_grad_reduce", ptr(f.partials), n_part.value, C.byref(algo._desc), ptr(f.grad), stream_ptr())
    got = f.grad.cpu().numpy()
    f.grad.zero_()
    f.partials.zero_()
    # read back at the offsets where the modules' own parameters live (checks the descriptor's mapping; a shared trunk is
    # one set of slots, checked once)
    for k, off in _offsets(f.flat, actor, critic).items():
        want = ref["grads"][k]
        gk = got[off:off + want.size].reshape(want.shape)
        # fp32 sums over the rows (within the CTA, then one add per CTA, then the fold): the bar of
        # test_ppo_grad_kernel_vs_oracle, 2e-4 relative + 2e-5 of the largest element
        record_parity(f"{tag}/{k}", gk, want, rtol=2e-4, atol=2e-5 * max(1e-6, float(np.abs(want).max())) + 1e-7)
    ex = got[f.n:f.n + 4]
    assert ex[3] == B
    record_parity(f"{tag}/clip_loss", -ex[0] / B, ref["clip"], rtol=1e-4, atol=1e-6)
    record_parity(f"{tag}/vf_loss", ex[1] / B, ref["vf"], rtol=1e-4, atol=1e-6)
    record_parity(f"{tag}/ent_loss", ex[2] / B, ref["ent"], rtol=2e-5, atol=1e-6)
    return ref


@pytest.mark.parametrize("hp_name", list(HP_SETS))
@pytest.mark.parametrize("family,obs_dim,act_dim", CASES, ids=CASE_IDS)
def test_ppo_grad_kernel_vs_fp64(family, obs_dim, act_dim, hp_name):
    """ts_ppo_grad + ts_grad_reduce on 300 permuted rows of 700 (three tiles, the last one partial), with the categorical
    clamp and ReLU zeros in the batch: every parameter gradient and the four loss sums against fp64 autograd."""
    _grad_case(family, obs_dim, act_dim, hp_name, 300, 700, 37, f"simt_grad/{hp_name}/{family}/{obs_dim}x{act_dim}")


@pytest.mark.parametrize("family", list(FAMILIES))
def test_ppo_grad_kernel_past_one_wave_vs_fp64(family):
    """B = 128 x #SMs + 77 rows: every CTA owns a tile and some own two (the grid-stride tile loop), n_partials = #SMs."""
    obs_dim, act_dim = FAMILIES[family]["shapes"][-1]
    B = 128 * _sms() + 77
    _grad_case(family, obs_dim, act_dim, "vclip_advnorm_ent", B, B + 100, 41, f"simt_grad_wave/{family}/{obs_dim}x{act_dim}")


# --------------------------------------------------------------------------- ts_clip_adam_step / ts_grad_reduce
ADAM_N = ["1", "255", "256", "257", "11085", "wave"]          # wave: #SMs x 256 - 4, the largest single-wave grid
ADAM_PARTIALS = ["0", "1", "3", "4", "5", "28", "29", "32", "33", "sms"]


def _resolve(x, sms):
    return {"wave": sms * 256 - 4, "sms": sms}.get(x) or int(x)


@pytest.mark.parametrize("n_partials", ADAM_PARTIALS)
@pytest.mark.parametrize("n", ADAM_N)
def test_clip_adam_step_and_grad_reduce_vs_torch(n, n_partials):
    """ts_clip_adam_step through the C ABI on synthetic vectors (the kernel reads only desc->n_params): three consecutive
    steps with the gradient clip off / above / below the norm, weight decay 0 / 0.01, from step 0 and resumed at step 57,
    against the partial rows folded in fp64, torch.nn.utils.clip_grad_norm_ and torch.optim.Adam(foreach=False).  Also
    the stats row, the loss sums copied into grad[n .. n + 4), the step count, and ts_grad_reduce's fold."""
    from tianshou_b200._cabi import ActorCriticDesc, PPOHParams, call, ptr, stream_ptr
    sms = _sms()
    n, n_p = _resolve(n, sms), _resolve(n_partials, sms)
    W = n + 4
    desc = ActorCriticDesc()
    desc.n_params = n
    gen = torch.Generator().manual_seed(n * 1000 + n_p)
    # Each element's partial rows share its sign (0.5 .. 1.5 of an equal share), so an fp32 sum of m of them is within
    # (m - 1) x 2^-24 of the fp64 sum, relative.  clip_adam_kernel: ceil(n_p / 32) rows per accumulator, up to 7 more in
    # the tail loop, then 3 + 2 tree levels; grad_reduce_kernel: n_p / 8 + 7 rows, then 3 levels
    fold_rel = (n_p / 32 + 12) * 2.0 ** -24
    reduce_rel = (n_p / 8 + 10) * 2.0 ** -24

    # Every gradient, every partial row and the resumed exp_avg share the sign of the element's parameter: neither the fold,
    # nor g + weight_decay x p, nor exp_avg's lerp cancels, so an fp32 rounding stays a relative error of its own size
    # instead of deciding the sign of a near-zero Adam step
    sign = torch.where(torch.randn(n, generator=gen) >= 0, 1.0, -1.0)

    def grad_rows(k):
        g = sign.double() * torch.randn(n, generator=gen, dtype=torch.float64).abs() * (1.0 + k)
        extra = torch.tensor([10.0 * torch.randn(1, generator=gen).item(), 1.0 + 10.0 * torch.rand(1, generator=gen).item(),
                              0.5 + torch.rand(1, generator=gen).item(), 0.0], dtype=torch.float64)
        target = torch.cat([g, extra])
        if n_p == 0:
            row = target.float()
            row[n + 3] = 300.0
            return None, row.double()
        w = 0.5 + torch.rand(n_p, W, generator=gen, dtype=torch.float64)
        rows = (target * (w / w.sum(0))).float()
        rows[:, n + 3] = 128.0                   # rows per tile: an exact integer sum
        return rows, rows.double().sum(0)

    tag = f"simt_adam/n{n}_p{n_p}"
    rows0, fold0 = grad_rows(0)
    out = torch.full((W,), float("nan"), device=DEV)
    if n_p > 0:
        call("ts_grad_reduce", ptr(rows0.to(DEV)), n_p, C.byref(desc), ptr(out), stream_ptr())
        record_parity(f"simt_grad_reduce/n{n}_p{n_p}", out.cpu().numpy(), fold0.numpy(), rtol=reduce_rel, atol=0.0)
    else:
        call("ts_grad_reduce", ptr(torch.zeros(W, device=DEV)), 0, C.byref(desc), ptr(out), stream_ptr())
        assert torch.equal(out, torch.zeros_like(out))

    lr, b1, b2, eps = 1e-3, 0.9, 0.999, 1e-8
    sq = float(np.sqrt(n))
    for clip_name, max_norm in (("off", 0.0), ("above", 100.0 * sq), ("below", 1e-2 * sq)):
        for wd in (0.0, 0.01):
            for step0 in (0, 57):
                cfg = f"{tag}/clip_{clip_name}_wd{wd}_step{step0}"
                p0 = sign * torch.randn(n, generator=gen).abs()
                m0 = 0.1 * sign * torch.randn(n, generator=gen).abs() if step0 else torch.zeros(n)
                v0 = 0.01 * torch.rand(n, generator=gen) + 1e-4 if step0 else torch.zeros(n)
                p_ref = p0.clone().to(DEV).requires_grad_(True)
                opt = torch.optim.Adam([p_ref], lr=lr, betas=(b1, b2), eps=eps, weight_decay=wd, foreach=False)
                if step0:
                    opt.state[p_ref] = {"step": torch.tensor(float(step0)), "exp_avg": m0.to(DEV).clone(),
                                        "exp_avg_sq": v0.to(DEV).clone()}
                pk, mk, vk = p0.to(DEV).clone(), m0.to(DEV).clone(), v0.to(DEV).clone()
                step = torch.tensor([step0], dtype=torch.int64, device=DEV)
                hp = PPOHParams(eps_clip=0.2, dual_clip=0.0, vf_coef=0.25, ent_coef=0.01, max_grad_norm=max_norm, adv_eps=1e-8,
                                lr=lr, beta1=b1, beta2=b2, adam_eps=eps, weight_decay=wd)
                for k in range(3):
                    rows, fold = (rows0, fold0) if k == 0 else grad_rows(k)
                    q = torch.zeros(n, dtype=torch.float64, requires_grad=True)
                    q.grad = fold[:n].clone()
                    if max_norm > 0:
                        norm = float(torch.nn.utils.clip_grad_norm_([q], max_norm))
                        assert (norm > max_norm) == (clip_name == "below")
                    else:
                        norm = float(torch.linalg.vector_norm(q.grad))
                    p_ref.grad = q.grad.float().to(DEV)
                    opt.step()
                    if rows is None:
                        grad = fold.float().to(DEV)
                        rows_d = None
                    else:
                        grad = torch.full((W,), float("nan"), device=DEV)     # grad[:n] is neither read nor written
                        rows_d = rows.to(DEV)
                    stats = torch.full((8,), float("nan"), device=DEV)
                    call("ts_clip_adam_step", ptr(pk), ptr(grad), ptr(rows_d), n_p, ptr(mk), ptr(vk), ptr(step), C.byref(desc),
                         C.byref(hp), ptr(stats), stream_ptr())
                    assert int(step.item()) == step0 + k + 1
                    e = fold[n:].numpy()
                    record_parity(f"{cfg}/loss_sums", grad[n:].cpu().numpy(), e, rtol=fold_rel, atol=0.0)
                    st = stats.cpu().numpy().astype(np.float64)
                    clip, vf, ent = -e[0] / e[3], e[1] / e[3], e[2] / e[3]
                    want = np.array([clip + 0.25 * vf - 0.01 * ent, clip, vf, ent])
                    # a few fp32 roundings of the folded sums, the loss formed from three of them
                    record_parity(f"{cfg}/stats_losses", st[:4], want, rtol=1e-5 + fold_rel,
                                  atol=1e-6 * (abs(clip) + abs(vf) + abs(ent)))
                    record_parity(f"{cfg}/stats_grad_norm", st[4:5], np.array([norm]), rtol=fold_rel + 1e-6, atol=0.0)
                    assert st[5] == e[3]
                    # test_offpolicy_kernels_gpu's Adam bars (the same fp32 operation order as torch's single-tensor step;
                    # the clip coefficient from an fp64 sum of squares), the moments widened by the fp32 fold: a gradient
                    # off by fold_rel moves exp_avg by as much and exp_avg_sq by twice as much, relative
                    record_parity(f"{cfg}/param", pk.cpu().numpy(), p_ref.detach().cpu().numpy(), rtol=1e-6, atol=2e-3 * lr)
                    s = opt.state[p_ref]
                    record_parity(f"{cfg}/exp_avg", mk.cpu().numpy(), s["exp_avg"].cpu().numpy(), rtol=2e-6 + fold_rel,
                                  atol=1e-7 * float(s["exp_avg"].abs().max()))
                    record_parity(f"{cfg}/exp_avg_sq", vk.cpu().numpy(), s["exp_avg_sq"].cpu().numpy(), rtol=2e-6 + 2 * fold_rel,
                                  atol=1e-7 * float(s["exp_avg_sq"].abs().max()))


# ----------------------------------------------------------------------------------------------- update level
UPDATE_KW = dict(gamma=0.99, gae_lambda=0.95, max_grad_norm=0.5, vf_coef=0.25, ent_coef=0.01, return_scaling=True,
                 eps_clip=0.2, value_clip=True, dual_clip=None, advantage_normalization=True, recompute_advantage=True)
UPDATE_HP = dict(eps_clip=0.2, dual_clip=None, vf_coef=0.25, ent_coef=0.01, max_grad_norm=0.5, adv_eps=1e-8, value_clip=True,
                 advantage_normalization=True, lr=3e-4, beta1=0.9, beta2=0.999, adam_eps=1e-8, weight_decay=0.0)


def _rollout_buffer(family, obs_dim, act_dim, E, T, seed):
    from tianshou_b200.data import Batch, VectorReplayBuffer
    cat = FAMILIES[family]["cat"]
    rng = np.random.default_rng(seed + 1)
    buf = VectorReplayBuffer(E * T, E, device=DEV)
    for s in synth_rollout(np.random.default_rng(seed), E, T, obs_dim, act_dim, p_term=0.03, trunc_len=15):
        if cat:
            s = dict(s, act=rng.integers(0, act_dim, E))
        buf.add(Batch(**s), buffer_ids=np.arange(E))
    return buf


CROSS = [("relu_gauss", 17, 6), ("relu_gauss", 5, 3), ("tanh_gauss_shared", 11, 3), ("tanh_cat", 17, 16),
         ("relu_cat_shared", 8, 4), ("relu_cat", 27, 9)]


@pytest.mark.parametrize("family,obs_dim,act_dim", CROSS, ids=[f"{f}-obs{o}-act{a}" for f, o, a in CROSS])
def test_update_matches_layered_path(family, obs_dim, act_dim, monkeypatch):
    """Families without a numpy oracle: PPO.update on the SIMT kernels against the same model built on the layer-wise
    path (pinned to the reference goldens and to fp64 in test_layered_gpu), same rollout, same numpy seed.  Step 0 starts
    from identical parameters: the loss columns at the tight bar; its gradient norm (the layer-wise table does not carry
    one) against the norm of the fp64 autograd gradient of the same minibatch.  Later rows and the final parameters: the
    Adam-trajectory bar of test_tc_shapes_gpu."""
    from tianshou_b200.utils import policy_within_training_step
    algo, actor, critic = _build(family, obs_dim, act_dim, **UPDATE_KW)
    _assert_simt(algo, family)
    monkeypatch.setenv("TS_B200_FORCE_LAYERED", "1")
    algo_l, actor_l, critic_l = _build(family, obs_dim, act_dim, **UPDATE_KW)
    monkeypatch.delenv("TS_B200_FORCE_LAYERED")
    assert algo_l._layered is not None
    named, named_l = ac_named_params(actor, critic), ac_named_params(actor_l, critic_l)
    for k in named:
        assert torch.equal(named[k], named_l[k]), k
    a0, c0 = copy.deepcopy((actor, critic))
    E, T, bs, repeat = 16, 25, 100, 2
    N = E * T
    captured = {}
    orig = algo._preprocess_batch

    def hook(batch, buffer, indices):
        b = orig(batch, buffer, indices)
        captured.update({k: b[k].detach().cpu().numpy().copy() for k in ("obs", "act", "v_s", "returns", "adv", "logp_old")})
        return b

    algo._preprocess_batch = hook
    tables = []
    for a in (algo, algo_l):
        buf = _rollout_buffer(family, obs_dim, act_dim, E, T, seed=obs_dim * 10 + act_dim)
        np.random.seed(4)
        with policy_within_training_step(a.policy):
            stats = a.update(buffer=buf, batch_size=bs, repeat=repeat)
        assert stats.gradient_steps == repeat * (N // bs)
        tables.append(a.last_loss_table)
    t_s, t_l = tables
    np.random.seed(4)
    idx = np.random.permutation(N)[:bs]
    mb = {k: captured[k][idx] for k in ("obs", "act", "adv", "logp_old", "v_s")}
    mb["returns"] = captured["returns"][idx]
    ref = actor_critic_reference_fp64(a0, c0, mb, dict(UPDATE_HP))
    norm = float(np.sqrt(sum(float((g.astype(np.float64) ** 2).sum()) for g in ref["grads"].values())))
    tag = f"simt_vs_layered/{family}/{obs_dim}x{act_dim}"
    record_parity(f"{tag}/step0_grad_norm", t_s[:1, 4], np.array([norm]), rtol=2e-4, atol=0.0)
    assert np.array_equal(t_s[:, 5], np.full(t_s.shape[0], float(bs)))
    for col, name in enumerate(["loss", "actor_loss", "vf_loss", "ent_loss"]):
        ref_col = t_l[:, col]
        unit = max(1e-3, float(np.abs(ref_col).max()), 1.0 if name == "actor_loss" else 0.0)
        record_parity(f"{tag}/step0_{name}", t_s[:1, col], ref_col[:1], rtol=2e-4, atol=2e-5 * unit)
        record_parity(f"{tag}/per_step_{name}", t_s[:, col], ref_col, rtol=1e-3, atol=3e-3 * unit)
    steps = t_s.shape[0]
    for k in named:
        record_parity(f"{tag}/param_{k}", named[k].detach().cpu().numpy(), named_l[k].detach().cpu().numpy(), rtol=1e-3,
                      atol=0.1 * 3e-4 * steps)


@pytest.mark.parametrize("obs_dim,act_dim", [(17, 6), (40, 5)], ids=["tensor_core-obs17-act6", "simt-obs40-act5"])
def test_weight_decay_update_vs_oracle(obs_dim, act_dim):
    """Adam with weight_decay = 0.01 through the tensor-core epoch kernel and through ts_clip_adam_step, against
    oracle_np.ppo_update (which adds weight_decay x p to the clipped gradient, as torch.optim.Adam does)."""
    from test_tc_shapes_gpu import _rollout
    from tianshou_b200.utils import policy_within_training_step
    algo, actor, critic = _build("tanh_gauss", obs_dim, act_dim, weight_decay=0.01, **UPDATE_KW)
    assert algo._layered is None and (algo._flat.weight_image is not None) == (obs_dim <= 32)
    p = {k: v.detach().cpu().numpy().copy() for k, v in ac_named_params(actor, critic).items()}
    buf, roll = _rollout(obs_dim, act_dim, 20, 50, seed=obs_dim + 1000 * act_dim)
    N, bs, repeat = 1000, 300, 2
    np.random.seed(4)
    perms = np.stack([np.random.permutation(N) for _ in range(repeat)])
    m = {k: np.zeros_like(v) for k, v in p.items()}
    v = {k: np.zeros_like(x) for k, x in p.items()}
    res = onp.ppo_update(p, m, v, 0, roll, perms, bs, repeat, dict(UPDATE_HP, weight_decay=0.01), onp.RunningMeanStd(),
                         0.99, 0.95, True)
    np.random.seed(4)
    with policy_within_training_step(algo.policy):
        algo.update(buffer=buf, batch_size=bs, repeat=repeat)
    table = algo.last_loss_table
    tag = f"simt_wd/{obs_dim}x{act_dim}"
    # test_tc_shapes_gpu._epoch_vs_oracle's bars: step 0 tight, later rows and parameters on the Adam-trajectory bar
    for col, name in enumerate(["loss", "actor_loss", "vf_loss", "ent_loss", "grad_norm"]):
        ref = res["grad_norms"] if col == 4 else res["losses"][:, col]
        unit = max(1e-3, float(np.abs(ref).max()), 1.0 if name == "actor_loss" else 0.0)
        record_parity(f"{tag}/step0_{name}", table[:1, col], ref[:1], rtol=2e-4, atol=2e-5 * unit)
        record_parity(f"{tag}/per_step_{name}", table[:, col], ref, rtol=1e-3, atol=3e-3 * unit)
    steps = res["losses"].shape[0]
    for k, pv in ac_named_params(actor, critic).items():
        record_parity(f"{tag}/param_{k}", pv.detach().cpu().numpy(), p[k], rtol=1e-3, atol=0.1 * 3e-4 * steps)


def test_categorical_fused_inference_six_actions():
    """Collector-side policy(batch) for a 6-action categorical head: the fused SIMT forward's probabilities against the
    torch modules."""
    from tianshou_b200.data import Batch
    algo, actor, critic = _build("relu_cat", 27, 6)
    _assert_simt(algo, "relu_cat")
    pol = algo.policy
    assert pol._fused_inference is not None
    obs = np.random.default_rng(6).standard_normal((300, 27)).astype(np.float32)
    with torch.no_grad():
        fused = pol(Batch(obs=obs, info=Batch())).logits
        pol.use_fused_inference = False
        ref = pol(Batch(obs=obs, info=Batch())).logits
        pol.use_fused_inference = True
    assert fused.shape == ref.shape == (300, 6)
    record_parity("simt_infer/relu_cat/27x6/probs", fused.cpu().numpy(), ref.cpu().numpy(), rtol=2e-5, atol=2e-6)


def test_simt_categorical_shape_past_shared_memory_is_refused():
    """obs 64 / 16 actions with a categorical head needs the same 235,536 B training tile as the Gaussian head: refused
    with a message naming the size."""
    from tianshou_b200.utils import policy_within_training_step
    algo, _, _ = _build("relu_cat", 64, 16, gamma=0.99, gae_lambda=0.95, max_grad_norm=0.5, vf_coef=0.25, ent_coef=0.0,
                        eps_clip=0.2, value_clip=False, advantage_normalization=False)
    buf = _rollout_buffer("relu_cat", 64, 16, 4, 8, seed=0)
    with pytest.raises(RuntimeError, match="235536 bytes of shared memory per block"):
        with policy_within_training_step(algo.policy):
            algo.update(buffer=buf, batch_size=16, repeat=1)
