"""Every minibatch step of the layer-wise PPO / A2C update (algorithm/layered.py: ``layered_update`` +
``LayeredActorCritic.minibatch_step``, the path of every network outside the fused kernels' envelope) against a float64
step taken from the update's OWN previous state, and the chunked whole-rollout passes against float64.

The layer-wise step is glued together in Python from about fifteen launches (row gathers, ``FusedStack`` forward and
backward per trunk and head, ``ts_ppo_rows``, ``ts_ppo_rows_stats``, ``ts_net_colsum`` for the log-std,
``FlatGroup.optimizer_step``).  ``test_layered_gpu`` holds it to the reference's goldens on fused shapes and to one wide
update through a trajectory bar, which grows with the step count: an error of about one Adam step confined to steps >= 2
(weights read before the previous write-back, a bias correction one step off, the advantage moments of another minibatch)
fits inside it.  Here no bar depends on the step index.

Teacher forcing needs no prefix runs on this path, since each step is one Python call: the update runs with
``minibatch_step`` and ``FlatGroup.optimizer_step`` wrapped.  Before step k the wrapper reads S_{k-1} (flat parameters,
exp_avg, exp_avg_sq, step count), the minibatch's rows and the advantage moments handed in; after it, the loss-table row,
the raw gradient (``ts_adam_step`` / ``ts_rmsprop_step`` take it const) and S_k.  Per step k:

1. the rows are ``perm[r][lo:hi]`` of the pass's permutation;
2. the advantage moments (advantage normalisation) are the float64 mean and unbiased std of those rows' advantages;
3. the loss row (loss, actor loss, vf loss, entropy) against float64 autograd at S_{k-1} on the step's rows; slot 4 is 0
   (the layer-wise row carries no gradient norm, ts_ppo_rows_stats' header) and slot 5 the row count;
4. the whole flat gradient, in ``FlatGroup`` order, against the float64 gradient;
5. exp_avg / exp_avg_sq (RMSprop: square_avg) against beta m_{k-1} + (1 - beta) g (g^2), g the float64 gradient after
   global-norm clipping and weight decay, m_{k-1} / v_{k-1} the update's own moments;
6. the parameters against one float64 Adam / RMSprop step from S_{k-1} with S_k's moments; the step count is k.

Pass boundary (repeat 2 + recompute_advantage): before the first step of pass 2, the v_s / returns / adv it wrote are
checked against the float64 critic at the parameters that end pass 1, followed by the GAE, return scaling and
RunningMeanStd arithmetic of oracle_np.add_returns_and_advantages.  Determinism: the same update from the same copied
state, run twice, gives bit-identical loss tables, parameters and moments.

Branch guard, at every S_{k-1}, before the step reads its rows: a row whose float64 ratio lies within 1e-4 of a clip
boundary or of the dual clip, whose value delta lies within 1e-4 of +-eps_clip, whose clipped value errors tie, that sits on
a ReLU kink or whose probabilities come near torch's clamp gets new inputs in place (logp_old, v_s or obs), so fp32 and
fp64 take the same branch everywhere and the comparison measures rounding.  The behaviour log-probs and stale values start
off the current policy (logp_old + 0.5 N(0, 1), v_s + 0.3 N(0, 1)); every PPO case asserts that rows fell on both sides of
each clip."""
import copy

import numpy as np
import pytest
import torch

from oracle import oracle_np as onp
from test_conv_kernels_gpu import U, _gemm_gamma
from test_epoch_steps_gpu import _assert_same_bits, _bits, _within
from test_simt_kernels_gpu import _Discrete, _Fp64, _saturated_rows
from ts_testutil import F32_EPS, Box, actor_critic_reference_fp64, gaussian_dist, record_parity, synth_rollout

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

PPO_KW = dict(gamma=0.99, gae_lambda=0.95, vf_coef=0.25, ent_coef=0.01, return_scaling=True, eps_clip=0.2, dual_clip=None,
              value_clip=True, advantage_normalization=True, recompute_advantage=False, max_grad_norm=0.5)
A2C_KW = dict(gamma=0.99, gae_lambda=0.95, vf_coef=0.5, ent_coef=0.01, return_scaling=True, max_grad_norm=0.5)

# network (obs, act, hidden, ReLU or Tanh, categorical, trunk: separate / ONE shared Net / two Net wrappers around one
# MLP), algorithm + optimiser, rollout E x T, minibatch size, repeat; clip="all": every step clips its gradient norm
CASES = {
    # Humanoid width; 800 rows in minibatches of 300 merge into 300 + 500 (the step scratch regrows); pass boundary
    "humanoid": dict(obs=376, act=17, hidden=(256, 256), relu=False, cat=False, trunk="separate", algo="ppo", E=16, T=50,
                     bs=300, repeat=2, kw=dict(recompute_advantage=True)),
    # three ReLU layers at odd widths (exact zeros in every layer), dual clip, every step clips
    "deep-odd": dict(obs=29, act=4, hidden=(96, 80, 40), relu=True, cat=False, trunk="separate", algo="ppo", E=10, T=90,
                     bs=150, repeat=1, clip="all", kw=dict(dual_clip=2.0, max_grad_norm=1e-3)),
    # the widest categorical head on ONE shared trunk (the critic's input gradient accumulates into the actor's); one row
    # in 16 saturated (every probability but one in torch's clamp); weight decay
    "cat64-shared": dict(obs=40, act=64, hidden=(128, 128), relu=True, cat=True, trunk="shared", algo="ppo", E=12, T=50,
                         bs=100, repeat=1, wd=0.01, saturate=16, kw=dict(advantage_normalization=False)),
    # A > 16 and widths off every tile multiple
    "cat23-odd": dict(obs=70, act=23, hidden=(200, 37), relu=False, cat=True, trunk="separate", algo="ppo", E=12, T=50,
                      bs=100, repeat=1, kw=dict(dual_clip=2.0)),
    # A2C with RMSprop (examples/mujoco/mujoco_a2c.py's optimiser) on a three-layer trunk
    "a2c-rmsprop": dict(obs=11, act=3, hidden=(64, 64, 64), relu=False, cat=False, trunk="separate", algo="a2c",
                        opt="rmsprop", E=12, T=50, bs=100, repeat=1, kw=dict()),
    # actor and critic hold two Net wrappers around ONE MLP: a shared trunk the parse finds by parameter identity
    "wrappers": dict(obs=17, act=6, hidden=(128, 128), relu=False, cat=False, trunk="wrappers", algo="ppo", E=12, T=50,
                     bs=100, repeat=1, kw=dict()),
}


def _build(c, seed):
    from tianshou_b200.algorithm import (A2C, PPO, AdamOptimizerFactory, DiscreteActorPolicy, ProbabilisticActorPolicy,
                                         RMSpropOptimizerFactory)
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.continuous import ContinuousActorProbabilistic, ContinuousCritic
    from tianshou_b200.utils.net.discrete import DiscreteActor, DiscreteCritic
    torch.manual_seed(seed)
    O, A = c["obs"], c["act"]
    act_fn = torch.nn.ReLU if c["relu"] else torch.nn.Tanh
    net_a = Net(state_shape=(O,), hidden_sizes=c["hidden"], activation=act_fn)
    if c["trunk"] == "shared":
        net_c = net_a
    else:
        net_c = Net(state_shape=(O,), hidden_sizes=c["hidden"], activation=act_fn)
        if c["trunk"] == "wrappers":
            net_c.model = net_a.model
    if c["cat"]:
        actor = DiscreteActor(preprocess_net=net_a, action_shape=(A,)).to(DEV)
        critic = DiscreteCritic(preprocess_net=net_c).to(DEV)
        policy = DiscreteActorPolicy(actor=actor, dist_fn=torch.distributions.Categorical, action_space=_Discrete(A))
        if c.get("saturate"):        # logits of a few units on ordinary rows, so that large rows can separate by 30
            with torch.no_grad():
                for m in actor.last.modules():
                    if isinstance(m, torch.nn.Linear):
                        m.weight.mul_(8.0)
    else:
        actor = ContinuousActorProbabilistic(preprocess_net=net_a, action_shape=(A,), unbounded=True).to(DEV)
        critic = ContinuousCritic(preprocess_net=net_c).to(DEV)
        policy = ProbabilisticActorPolicy(actor=actor, dist_fn=gaussian_dist, action_scaling=True, action_bound_method="clip",
                                          action_space=Box(A))
        with torch.no_grad():       # a distinct sigma per action dimension
            actor.sigma_param.copy_(torch.linspace(-1.2, 0.3, A).reshape(actor.sigma_param.shape))
    wd = c.get("wd", 0.0)
    if c.get("opt") == "rmsprop":
        optim = RMSpropOptimizerFactory(lr=7e-4, alpha=0.99, eps=1e-5, weight_decay=wd)
    else:
        optim = AdamOptimizerFactory(lr=3e-4, weight_decay=wd)
    if c["algo"] == "a2c":
        algo = A2C(policy=policy, critic=critic, optim=optim, **dict(A2C_KW, **c["kw"]))
    else:
        algo = PPO(policy=policy, critic=critic, optim=optim, **dict(PPO_KW, **c["kw"]))
    return algo, actor, critic


def _modules(net):
    """The Linear / Tanh / ReLU chain of a Net / MLP / Sequential."""
    from tianshou_b200.algorithm.netgraph import module_layers
    return module_layers(net)


@torch.no_grad()
def _forward_bound(mods, x):
    """(float64 output of the Linear / Tanh / ReLU chain ``mods`` (float64 copies) on the fp32 rows ``x``, a bound on the
    layer-wise stack's error per element).  Per layer the stack is within gamma(K) (|W| |a| + |b|) of float64 on its own fp32
    input (+ 4 ulp of tanhf; test_fused_stack_gpu's forward bar); an input error e moves a Linear output by at most |W| e,
    and Tanh / ReLU by at most e, so  e_i = gamma(K) (|W| (|a| + e_{i-1}) + |b|) + |W| e_{i-1}."""
    a = torch.as_tensor(np.asarray(x, np.float64))
    e = torch.zeros_like(a)
    for m in mods:
        if isinstance(m, torch.nn.Linear):
            W, b = m.weight.abs(), m.bias.abs()
            e_in = e @ W.T
            e = _gemm_gamma(m.in_features) * ((a.abs() + e) @ W.T + b) + e_in
            a = m(a)
        elif isinstance(m, torch.nn.Tanh):
            a = torch.tanh(a)
            e = e + 4 * U * a.abs()
        elif isinstance(m, torch.nn.ReLU):
            a = torch.relu(a)
        else:
            raise AssertionError(f"unexpected module {type(m).__name__}")
    return a.numpy(), e.numpy()


def _copy64(*mods):
    out = copy.deepcopy(mods)
    for m in out:
        m.to("cpu", torch.float64)
    return out


class _Order:
    """The pass orders ``layered_update`` walks: explicit rows, ready at once."""

    def __init__(self, rows: torch.Tensor) -> None:
        self.rows = rows

    def ready(self, r: int) -> None:
        pass


class Case:
    def __init__(self, name):
        self.name = name
        c = self.c = CASES[name]
        seed = c["obs"] * 100 + c["act"]
        self.algo, self.actor, self.critic = _build(c, seed)
        algo = self.algo
        self.L = L = algo._layered
        assert L is not None, f"{name}: must run on the layer-wise path without TS_B200_FORCE_LAYERED"
        assert L.shared == (c["trunk"] != "separate") and len(L.a_trunk.layers) == len(c["hidden"])
        self.g = g = L.group
        assert g.step_dev is None and g is L.critic_group
        self.spec = dict(shared=L.shared, cat=c["cat"], relu=c["relu"])
        self.ppo = c["algo"] == "ppo"
        self.kw = dict(PPO_KW if self.ppo else A2C_KW, **c["kw"])
        self.rng = np.random.default_rng(seed)
        # FlatGroup layout: (offset, size, kind) per parameter, kind "w" for a weight (a weight-gradient GEMM output),
        # "b" for a bias or the log-std (column sums)
        self.layout = [(g.offset(p), p.numel(), "w" if p.dim() == 2 else "b") for p in g.params]
        assert sum(n for _, n, _ in self.layout) == g.n
        buf = self._rollout(seed)
        self.N = N = c["E"] * c["T"]
        batch, indices = algo._sample(buf, 0)
        self.batch = algo._preprocess_batch(batch, buf, indices)
        assert torch.equal(indices.cpu(), torch.arange(N)), "a full buffer: batch row i is rollout row i"
        b = self.batch
        if self.ppo:       # a behaviour policy and a value net some updates old: every clip takes both branches
            b.logp_old.add_(torch.from_numpy(0.5 * self.rng.standard_normal(N)).float().to(DEV))
            b.v_s.add_(torch.from_numpy(0.3 * self.rng.standard_normal(N)).float().to(DEV))
        self.rms0 = algo._scratch["rms"].clone()
        self.repeat = c["repeat"]
        self.perm_host = np.stack([self.rng.permutation(N) for _ in range(self.repeat)]).astype(np.int32)
        self.perm = torch.from_numpy(self.perm_host).to(DEV)
        self.bounds = onp.minibatch_bounds(N, c["bs"])
        self.n_mb = len(self.bounds)
        self.state0 = self._state()
        assert self.state0[3] == 0 and not self.state0[1].any() and not self.state0[2].any()
        self.sides = dict(ratio_in=0, ratio_out=0, dual_on=0, dual_off=0, vclip_on=0, vclip_off=0)
        self.clipped: list[bool] = []
        self.moved_obs = 0

    def _rollout(self, seed):
        from tianshou_b200.data import Batch, VectorReplayBuffer
        c = self.c
        E, T, O, A = c["E"], c["T"], c["obs"], c["act"]
        buf = VectorReplayBuffer(E * T, E, device=DEV)
        sat = None
        if c.get("saturate"):
            f64 = _Fp64(self.actor, self.critic, dict(shared=self.algo._layered.shared, cat=True, relu=c["relu"]))
            sat = _saturated_rows(np.random.default_rng(seed + 2), f64, O, E * T // c["saturate"])
            assert len(sat) >= E * T // c["saturate"] // 2, f"{len(sat)} saturated rows found"
        act_rng = np.random.default_rng(seed + 1)
        for t, s in enumerate(synth_rollout(np.random.default_rng(seed), E, T, O, A, p_term=0.03, trunc_len=15)):
            if c["cat"]:
                s = dict(s, act=act_rng.integers(0, A, E))
            if sat is not None:
                obs = s["obs"].copy()
                for e in range(E):
                    i = t * E + e
                    if i % c["saturate"] == 0 and i // c["saturate"] < len(sat):
                        obs[e] = sat[i // c["saturate"]]
                s = dict(s, obs=obs)
            buf.add(Batch(**s), buffer_ids=np.arange(E))
        return buf

    def _state(self):
        g = self.g
        return (g.flat.cpu().numpy().astype(np.float64), g.exp_avg.cpu().numpy().astype(np.float64),
                g.exp_avg_sq.cpu().numpy().astype(np.float64), g.sync_step_from_device())

    def hpr(self):
        kw = self.kw
        if not self.ppo:
            return dict(loss_kind="a2c", vf_coef=kw["vf_coef"], ent_coef=kw["ent_coef"], advantage_normalization=False)
        return dict(eps_clip=kw["eps_clip"], dual_clip=kw["dual_clip"], value_clip=kw["value_clip"],
                    advantage_normalization=kw["advantage_normalization"], adv_eps=1e-8, vf_coef=kw["vf_coef"],
                    ent_coef=kw["ent_coef"])

    # ------------------------------------------------------------------------------------------------ float64 side
    def _columns(self, idx):
        b = self.batch
        return {k: getattr(b, k)[idx].cpu().numpy() for k in ("obs", "act", "adv", "returns", "logp_old", "v_s")}

    def guarded_reference(self, tag, idx):
        """float64 autograd at the current parameters on rows ``idx``; rows on a branch boundary get new inputs in place
        first (the step about to run reads them)."""
        rows = idx.cpu().numpy()
        hpr = self.hpr()
        for _ in range(20):
            mb = self._columns(idx)
            ref = actor_critic_reference_fp64(self.actor, self.critic, mb, hpr, group_order=True)
            lp_bad, vs_bad, obs_bad, sides = self.guard(ref, mb, hpr)
            if not (lp_bad.any() or vs_bad.any() or obs_bad.any()):
                for k, v in sides.items():
                    self.sides[k] += v
                return ref
            b = self.batch
            if lp_bad.any():
                new = ref["logp"][lp_bad] + 0.5 * self.rng.standard_normal(int(lp_bad.sum()))
                b.logp_old[torch.from_numpy(rows[lp_bad]).to(DEV)] = torch.from_numpy(new).float().to(DEV)
            if vs_bad.any():
                new = ref["v"][vs_bad] + 0.3 * self.rng.standard_normal(int(vs_bad.sum()))
                b.v_s[torch.from_numpy(rows[vs_bad]).to(DEV)] = torch.from_numpy(new).float().to(DEV)
            if obs_bad.any():
                assert not self.kw.get("recompute_advantage"), "the value recompute reads the rollout's observations"
                self.moved_obs += int(obs_bad.sum())
                new = self.rng.standard_normal((int(obs_bad.sum()), self.c["obs"]))
                b.obs[torch.from_numpy(rows[obs_bad]).to(DEV)] = torch.from_numpy(new).float().to(DEV)
        pytest.fail(f"{tag}: rows still on a branch boundary after 20 redraws")

    def guard(self, ref, mb, hpr):
        n = len(mb["adv"])
        obs_bad = np.zeros(n, dtype=bool)
        if self.c["relu"] or self.c["cat"]:
            f64 = _Fp64(self.actor, self.critic, self.spec)
            if self.c["relu"]:
                obs_bad |= f64.near_kink(mb["obs"])
            if self.c["cat"]:       # no probability within 4x of torch's clamp at eps or 1 - eps
                pn, _ = f64.probs(mb["obs"])
                obs_bad |= (((pn > F32_EPS / 4) & (pn < 4 * F32_EPS)) | ((1 - pn > F32_EPS / 4) & (1 - pn < 4 * F32_EPS))).any(1)
        lp_bad = np.zeros(n, dtype=bool)
        vs_bad = np.zeros(n, dtype=bool)
        sides = {}
        if self.ppo:
            e, dual = hpr["eps_clip"], hpr["dual_clip"] or 0.0
            ratio = np.exp(ref["logp"] - mb["logp_old"].astype(np.float64))
            lp_bad |= (np.abs(ratio - (1 - e)) < 1e-4) | (np.abs(ratio - (1 + e)) < 1e-4)
            inside = (ratio > 1 - e) & (ratio < 1 + e)
            sides.update(ratio_in=int(inside.sum()), ratio_out=int((~inside).sum()))
            if dual:
                A = mb["adv"].astype(np.float64)
                if hpr["advantage_normalization"]:
                    A = (A - A.mean()) / (A.std(ddof=1) + 1e-8)
                obj = np.minimum(ratio * A, np.clip(ratio, 1 - e, 1 + e) * A)
                lp_bad |= (A < 0) & (np.abs(obj - dual * A) < 1e-4)
                sides.update(dual_on=int(((A < 0) & (obj < dual * A)).sum()), dual_off=int(((A < 0) & (obj > dual * A)).sum()))
            if hpr["value_clip"]:
                v, vs, R = ref["v"], mb["v_s"].astype(np.float64), mb["returns"].astype(np.float64)
                dl = v - vs
                vc = vs + np.clip(dl, -e, e)
                vs_bad |= (np.abs(np.abs(dl) - e) < 1e-4) | ((np.abs(dl) > e) & (np.abs(np.abs(R - v) - np.abs(R - vc)) < 1e-4))
                sides.update(vclip_on=int((np.abs(dl) > e).sum()), vclip_off=int((np.abs(dl) < e).sum()))
        return lp_bad, vs_bad, obs_bad, sides

    # ------------------------------------------------------------------------------------------------ the checks
    def check_adv_moments(self, tag, idx, adv_moments):
        if not (self.ppo and self.kw["advantage_normalization"]):
            assert adv_moments is None, f"{tag}: advantage moments handed to a step without advantage normalisation"
            return
        a = self.batch.adv[idx].cpu().numpy().astype(np.float64)
        want = np.array([a.mean(), a.std(ddof=1)])
        # the sums are float64 over the same fp32 values: only the final rounding to fp32 (half an ulp) remains, + a float64
        # cancellation floor for a mean near 0
        _within(f"{tag}/adv_moments", adv_moments.cpu().numpy(), want, 4 * U * np.abs(want) + 1e-12 * float(np.abs(a).max()))

    def check_step(self, tag, k, pre, post, row, ref, B):
        g64 = ref["grads"]
        p0, m0, v0, step0 = pre
        p1, m1, v1, step1 = post[:4]
        grad = post[4]
        hp = self.algo._loss_hparams()
        # 3. the loss row: the step-0 bars of test_tc_shapes_gpu._epoch_vs_oracle (2e-4 relative, 2e-5 of max(1e-3, |value|);
        #    the actor loss in units of 1), on every step
        for col, name, want in ((0, "loss", ref["loss"]), (1, "actor_loss", ref["clip"]), (2, "vf_loss", ref["vf"]),
                                (3, "ent_loss", ref["ent"])):
            unit = max(1e-3, abs(want), 1.0 if name == "actor_loss" else 0.0)
            record_parity(f"{tag}/{name}", row[col:col + 1], np.array([want]), rtol=2e-4, atol=2e-5 * unit)
        assert row[4] == 0.0, f"{tag}: loss-table slot 4 is {row[4]}; the layer-wise row carries no gradient norm"
        assert row[5] == B, f"{tag}: {row[5]} rows in the loss table, minibatch has {B}"
        # 4. the raw gradient.  Per element of tensor t: 2e-4 |g| + a_t max_t |g| + 1e-7 with a_t = 1e-4 for a weight (a
        #    weight-gradient GEMM output, the MMA bar of test_epoch_steps_gpu) and 2e-5 for a bias / the log-std (column sums)
        gb = np.zeros_like(g64)
        for off, n, kind in self.layout:
            s = slice(off, off + n)
            gk = np.abs(g64[s])
            gb[s] = 2e-4 * gk + (1e-4 if kind == "w" else 2e-5) * gk.max() + 1e-7
        for i, (off, n, _) in enumerate(self.layout):
            s = slice(off, off + n)
            _within(f"{tag}/grad/param{i}", grad[s], g64[s], gb[s])
        # 5. moments.  Clipping scales the gradient by max_norm / (norm + 1e-6), off by the norm's 2e-4 relative: another
        #    2e-4 |g|
        norm = float(np.sqrt((g64 * g64).sum()))
        M = hp.max_grad_norm
        coef = min(M / (norm + 1e-6), 1.0) if M > 0 else 1.0
        if M > 0:
            assert abs(norm - M) > 1e-3 * M, f"{tag}: gradient norm {norm} at the clip threshold {M}: the branch is a tie"
        self.clipped.append(M > 0 and norm > M)
        gb = coef * (gb + (2e-4 * np.abs(g64) if self.clipped[-1] else 0.0))
        wd = hp.weight_decay
        gc = coef * g64 + wd * p0
        mag = np.abs(coef * g64) + np.abs(wd * p0)      # |terms| of gc: fp32 rounding of the kernel's g + wd p
        ulp = 4.0 * F32_EPS
        rms = self.c.get("opt") == "rmsprop"
        b2 = hp.beta2                                   # RMSprop: alpha
        v_ref = b2 * v0 + (1 - b2) * gc * gc
        # exp_avg_sq moves by (1 - beta2) d(g^2) = (1 - beta2)(2 |g| e + e^2) for a gradient error e, plus a few fp32
        # roundings of its terms
        v_bar = (1 - b2) * (2 * np.abs(gc) * gb + gb * gb) + ulp * (b2 * v0 + (1 - b2) * (mag + gb) ** 2) + 1e-30
        if rms:
            assert np.array_equal(_bits(m1), _bits(m0)), f"{tag}: RMSprop must leave exp_avg untouched"
        else:
            b1 = hp.beta1
            m_ref = b1 * m0 + (1 - b1) * gc
            # exp_avg moves by (1 - beta1) e, plus a few fp32 roundings of its terms
            m_bar = (1 - b1) * gb + ulp * (b1 * np.abs(m0) + (1 - b1) * mag) + 1e-30
        for i, (off, n, _) in enumerate(self.layout):
            s = slice(off, off + n)
            if not rms:
                _within(f"{tag}/exp_avg/param{i}", m1[s], m_ref[s], m_bar[s])
            _within(f"{tag}/exp_avg_sq/param{i}", v1[s], v_ref[s], v_bar[s])
        # 6. parameters: one fp64 step from S_{k-1} with S_k's moments.  Adam: the step is the kernel's own arithmetic on its
        #    own moments -- a few fp32 roundings of the step (8 ulp) and of the parameter (2 ulp).  RMSprop divides the
        #    clipped gradient itself: its error e moves the parameter by lr e / (sqrt(v) + eps) on top
        assert step1 == step0 + 1 == k, f"{tag}: step count {step1} after step {k} (before it: {step0})"
        if rms:
            den = np.sqrt(v1) + hp.adam_eps
            delta = hp.lr * gc / den
            p_bar = hp.lr * gb / den + 8 * F32_EPS * np.abs(delta) + 2 * F32_EPS * np.abs(p0) + 1e-30
        else:
            step_size = hp.lr / (1.0 - hp.beta1 ** step1)
            bc2_sqrt = np.sqrt(1.0 - hp.beta2 ** step1)
            delta = step_size * m1 / (np.sqrt(v1) / bc2_sqrt + hp.adam_eps)
            p_bar = 8 * F32_EPS * np.abs(delta) + 2 * F32_EPS * np.abs(p0) + 1e-30
        p_ref = p0 - delta
        for i, (off, n, _) in enumerate(self.layout):
            s = slice(off, off + n)
            _within(f"{tag}/param/param{i}", p1[s], p_ref[s], p_bar[s])

    def check_pass_boundary(self, tag):
        """v_s / returns / adv written by the recompute before pass 2, at the parameters that end pass 1."""
        algo, b = self.algo, self.batch
        (c64,) = _copy64(self.critic)
        mods = _modules(c64.preprocess) + _modules(c64.last)
        obs, obs_next = b.obs.cpu().numpy(), b.obs_next.cpu().numpy()
        v64, v_err = _forward_bound(mods, obs)
        vn64, vn_err = _forward_bound(mods, obs_next)
        v64, v_err, vn64, vn_err = (x.reshape(-1) for x in (v64, v_err, vn64, vn_err))
        rms = onp.RunningMeanStd()
        m, var, cnt = self.rms0.cpu().numpy().tolist()
        rms.mean, rms.var, rms.count = m, var, int(round(cnt))
        scale = float(np.sqrt(rms.var + 1e-8))
        roll = dict(obs=obs, obs_next=obs_next, rew=b.rew.cpu().numpy().astype(np.float64),
                    terminated=b.terminated.cpu().numpy().astype(bool), truncated=b.truncated.cpu().numpy().astype(bool),
                    unfinished=b.__dict__["_unfinished"].cpu().numpy().astype(bool))
        _, ret_ref, adv_ref = onp.add_returns_and_advantages(None, roll, rms, algo.gamma, algo.gae_lambda,
                                                             values=(v64, vn64))
        # v: the propagated forward bound of every row
        _within(f"{tag}/v_s", b.v_s.cpu().numpy(), v64, v_err + 1e-30)
        # adv: each TD error carries (1 + gamma) value errors (scaled by the return scale), the GAE sum weighs them by
        # (gamma lambda)^j, at most 1 / (1 - gamma lambda) in all; + fp32 output rounding
        v_bar = float(max(v_err.max(), vn_err.max()))
        gl = algo.gamma * algo.gae_lambda
        adv_err = (1 + algo.gamma) * v_bar * scale / (1 - gl)
        record_parity(f"{tag}/adv", b.adv.cpu().numpy(), adv_ref, rtol=1e-6, atol=adv_err)
        # returns = (adv + v_s * scale) / scale
        ret_err = adv_err + v_bar * scale
        record_parity(f"{tag}/returns", b.returns.cpu().numpy(), ret_ref, rtol=1e-6, atol=ret_err / scale)
        got = algo._scratch["rms"].cpu().numpy()
        assert got[2] == rms.count, f"{tag}: RunningMeanStd count {got[2]} vs {rms.count}"
        # mean of returns off by ret_err at most; the variance by 2 max|ret - mean| ret_err + ret_err^2
        ret_unscaled = ret_ref.astype(np.float64) * scale
        record_parity(f"{tag}/rms_mean", got[:1], np.array([rms.mean]), rtol=1e-9, atol=ret_err)
        var_err = 2 * float(np.abs(ret_unscaled - rms.mean).max()) * ret_err + ret_err ** 2
        record_parity(f"{tag}/rms_var", got[1:2], np.array([rms.var]), rtol=1e-9, atol=var_err)
        self.boundary_checked = True

    # ------------------------------------------------------------------------------------------------ runs
    def _update(self):
        from tianshou_b200.algorithm.layered import layered_update
        table = layered_update(self.algo, self.batch, self.c["bs"], self.repeat, _Order(self.perm))
        torch.cuda.synchronize()
        return table.cpu().numpy()

    def run_teacher_forced(self):
        L, g = self.L, self.g
        inner_step, inner_opt = L.minibatch_step, g.optimizer_step
        grads_in = []
        self.k = 0
        self.boundary_checked = False

        def optimizer_step(optimizer, max_grad_norm):
            torch.cuda.synchronize()
            grads_in.append(g.grad[:g.n].cpu().numpy().copy())
            inner_opt(optimizer, max_grad_norm)

        def minibatch_step(batch, idx, hp, adv_moments, optimizer, max_grad_norm, stats_row):
            torch.cuda.synchronize()
            self.k += 1
            k = self.k
            r, m = divmod(k - 1, self.n_mb)
            lo, hi = self.bounds[m]
            tag = f"{self.name}/pass{r + 1}/step{k}"
            assert batch is self.batch
            assert np.array_equal(idx.cpu().numpy(), self.perm_host[r][lo:hi]), f"{tag}: rows are not perm[{r}][{lo}:{hi}]"
            if r > 0 and m == 0 and self.kw.get("recompute_advantage"):
                self.check_pass_boundary(f"{self.name}/pass_boundary")
            self.check_adv_moments(tag, idx, adv_moments)
            ref = self.guarded_reference(tag, idx)
            pre = self._state()
            n_opt = len(grads_in)
            inner_step(batch, idx, hp, adv_moments, optimizer, max_grad_norm, stats_row)
            torch.cuda.synchronize()
            assert len(grads_in) == n_opt + 1, f"{tag}: {len(grads_in) - n_opt} optimiser steps in one minibatch step"
            grad = g.grad[:g.n].cpu().numpy()
            assert np.array_equal(_bits(grad), _bits(grads_in[-1])), f"{tag}: the optimiser step changed the gradient"
            self.check_step(tag, k, pre, (*self._state(), grad.astype(np.float64)), stats_row.cpu().numpy(), ref, hi - lo)
            if k == self.n_mb:      # the columns pass 1 read, nudges included (a recompute rewrites v_s / returns / adv)
                self.pass1_cols = {c: getattr(batch, c).clone() for c in ("v_s", "returns", "adv")}

        L.minibatch_step, g.optimizer_step = minibatch_step, optimizer_step
        try:
            table = self._update()
        finally:
            del L.minibatch_step, g.optimizer_step
        assert self.k == self.repeat * self.n_mb == table.shape[0]
        return table

    def replay(self, inputs):
        """The same update from state0 on ``inputs`` (the batch columns), without the wrappers."""
        g, b = self.g, self.batch
        for buf, x in ((g.flat, self.state0[0]), (g.exp_avg, self.state0[1]), (g.exp_avg_sq, self.state0[2])):
            buf.copy_(torch.from_numpy(x).float())
        g._step = 0
        self.algo._scratch["rms"].copy_(self.rms0)
        for k, v in inputs.items():
            getattr(b, k).copy_(v)
        table = self._update()
        return table, g.flat.clone(), g.exp_avg.clone(), g.exp_avg_sq.clone()

    def run(self):
        cols = ("obs", "v_s", "returns", "adv", "logp_old")
        table = self.run_teacher_forced()
        c = self.c
        if self.kw.get("recompute_advantage"):
            assert self.boundary_checked
        if self.ppo:
            want = ["ratio_in", "ratio_out"] + (["dual_on", "dual_off"] if self.kw["dual_clip"] else []) + \
                   (["vclip_on", "vclip_off"] if self.kw["value_clip"] else [])
            empty = [k for k in want if self.sides[k] == 0]
            assert not empty, f"{self.name}: no rows on the side(s) {empty} of their clip: {self.sides}"
        if c.get("clip") == "all":
            assert all(self.clipped), f"{self.name}: steps {[i + 1 for i, x in enumerate(self.clipped) if not x]} did not clip"
        if c["relu"]:
            h = self._columns(torch.arange(self.N, device=DEV))["obs"]
            f64 = _Fp64(self.actor, self.critic, self.spec)
            x = torch.as_tensor(h, dtype=torch.float64)
            for i, mod in enumerate(_modules(f64.a.preprocess)):
                x = mod(x)
                if isinstance(mod, torch.nn.ReLU):
                    assert (x == 0).any(), f"{self.name}: no exact ReLU zero after layer {i}"
        # determinism: the update twice from state0 on the columns the teacher-forced run read in pass 1, nudges included
        inputs = dict({k: getattr(self.batch, k).clone() for k in cols}, **self.pass1_cols)
        t1, p1, m1, v1 = self.replay(inputs)
        t2, p2, m2, v2 = self.replay(inputs)
        _assert_same_bits(f"{self.name}: loss table of two identical updates", t2, t1)
        for what, a, bb in (("params", p1, p2), ("exp_avg", m1, m2), ("exp_avg_sq", v1, v2)):
            assert torch.equal(a, bb), f"{self.name}: {what} differ between two identical updates"
        assert t1.shape[0] == table.shape[0]


@pytest.mark.parametrize("name", list(CASES))
def test_every_layered_step_vs_fp64_from_own_state(name):
    Case(name).run()


# ------------------------------------------------------------------------------------------- whole-rollout passes
def _gaussian_algo(O, A, hidden):
    c = dict(obs=O, act=A, hidden=hidden, relu=False, cat=False, trunk="separate", algo="ppo", kw=dict())
    algo, actor, critic = _build(c, O * 100 + A)
    assert algo._layered is not None
    return algo, actor, critic


def _check_passes(algo, actor, critic, n, tag, chunk):
    """critic_values and actor_logp on n rows against float64 on copies of the modules; the outputs start as NaN, so a row
    no chunk writes fails.  Every stack call is counted: the passes run in chunks of ``chunk`` rows, the last one partial."""
    L = algo._layered
    O, A = L.a_trunk.layers[0].in_dim, L.act_dim
    rng = np.random.default_rng(n)
    obs = rng.standard_normal((n, O)).astype(np.float32)
    act = rng.standard_normal((n, A)).astype(np.float32)
    calls = {"c": [], "a": []}
    stacks = {"c": L.c_trunk, "a": L.a_trunk}
    for key, st in stacks.items():
        inner = st.forward
        st.forward = (lambda inner, key: lambda x, rows, tag="a", **kw: calls[key].append(rows) or inner(x, rows, tag, **kw))(
            inner, key)
    try:
        v = torch.full((n,), float("nan"), device=DEV)
        lp = torch.full((n,), float("nan"), device=DEV)
        L.critic_values(torch.from_numpy(obs).to(DEV), v)
        L.actor_logp(torch.from_numpy(obs).to(DEV), torch.from_numpy(act).to(DEV), lp, algo._loss_hparams())
        torch.cuda.synchronize()
    finally:
        for st in stacks.values():
            del st.forward
    want = [chunk] * (n // chunk) + ([n % chunk] if n % chunk else [])
    assert calls["c"] == want and calls["a"] == want, f"{tag}: chunks {calls} vs {want}"
    a64, c64 = _copy64(actor, critic)
    v64, v_err = _forward_bound(_modules(c64.preprocess) + _modules(c64.last), obs)
    _within(f"{tag}/critic_values", v.cpu().numpy(), v64.reshape(-1), v_err.reshape(-1) + 1e-30)
    mu64, mu_err = _forward_bound(_modules(a64.preprocess) + _modules(a64.mu), obs)
    ls = a64.sigma_param.detach().reshape(-1).numpy()
    s2 = np.exp(2 * ls)
    d = act.astype(np.float64) - mu64
    terms = -d * d / (2 * s2) - ls - 0.5 * np.log(2 * np.pi)
    logp64 = terms.sum(1)
    # a mean error e moves a row's log-prob by |a - mu| / sigma^2 e per dimension; ts_ppo_rows' own fp32 arithmetic rounds
    # each of the A terms a few times and sums them: 8 (A + 2) ulp of the sum of their magnitudes
    bound = (np.abs(d) / s2 * mu_err).sum(1) + 8 * (A + 2) * U * (np.abs(terms).sum(1) + np.abs(ls).sum())
    _within(f"{tag}/actor_logp", lp.cpu().numpy(), logp64, bound)


@pytest.mark.parametrize("n", [1000, 999, 971, 97, 1])
def test_whole_rollout_passes_in_small_chunks_vs_fp64(n, monkeypatch):
    """_CHUNK = 97: 1000 rows = ten full chunks + 30, 999 = ten + 29, 971 = ten + a 1-row chunk, 97 = one full chunk and
    1 = one partial chunk.  The Humanoid-width network of the step test, so every chunk runs the wide GEMMs."""
    from tianshou_b200.algorithm import layered
    monkeypatch.setattr(layered, "_CHUNK", 97)
    algo, actor, critic = _gaussian_algo(376, 17, (256, 256))
    _check_passes(algo, actor, critic, n, f"layered_chunks/c97/n{n}", 97)


def test_whole_rollout_passes_over_two_real_chunks_vs_fp64():
    """The real _CHUNK at N = _CHUNK + 77 on a narrow three-layer network (layer-wise only through its depth): a full chunk
    and a 77-row one; every row written."""
    from tianshou_b200.algorithm import layered
    algo, actor, critic = _gaussian_algo(8, 3, (64, 64, 64))
    n = layered._CHUNK + 77
    _check_passes(algo, actor, critic, n, "layered_chunks/real/two_chunks", layered._CHUNK)
