"""Every optimiser step of the single-GPU PPO / A2C pass (``ts_ppo_update_dedup``: the persistent tensor-core epoch kernel,
or ts_ppo_grad + ts_clip_adam_step per step on the SIMT kernels) against a float64 step taken from the kernel's OWN
previous state.

The trajectory tests (test_tc_shapes_gpu._epoch_vs_oracle, test_simt_kernels_gpu) hold only row 0 of the loss table to a
tight bar: later rows follow two Adam trajectories that drift apart, so their bars grow with the step count, and an error
confined to steps >= 1 -- weights read before the previous step's write-back, a bias correction off by one step, the moments
of the wrong step -- is about one Adam step (~lr) and fits inside them.  Here no bar depends on the step index.

Teacher forcing by prefix runs: one rollout is preprocessed once; run k restarts from the same copied state (flat
parameters, exp_avg, exp_avg_sq, step counter, a zeroed weight image, fresh copies of the batch columns a pass rewrites)
and makes the same pass restricted to its first k minibatches.  S_k is the state run k leaves.  Per step k:

1. prefix determinism: rows 0 .. k-2 of run k's loss table are run k-1's table bit for bit (otherwise a step's result
   depends on work the kernel has not done yet);
2. loss row k-1 (loss, actor, vf, entropy, pre-clip gradient norm, rows) against float64 autograd at S_{k-1}'s parameters
   on minibatch k's rows;
3. exp_avg / exp_avg_sq of S_k against beta m_{k-1} + (1 - beta) g (g^2), g the float64 clipped gradient at S_{k-1} and
   m_{k-1}, v_{k-1} the kernel's own moments of S_{k-1};
4. the parameters of S_k against one float64 Adam / RMSprop step from S_{k-1}'s parameters with S_k's moments; the step
   counter of S_k is k;
5. the 128-byte control block in front of the weight image (grid-barrier state) is zero after every launch.

Pass boundaries: with repeat 2 and recompute_advantage, the v_s / returns / adv that pass 2 wrote are checked against the
critic, GAE, return scaling and RunningMeanStd in float64 (oracle_np.add_returns_and_advantages) at the parameters S_K that
ends pass 1, and the first steps of pass 2 are teacher-forced from S_K in the same way.

The behaviour log-probs and stale values of the rollout are moved off the current policy (logp_old + 0.5 N(0, 1),
v_s + 0.3 N(0, 1)), so that the ratio clip, the dual clip and the value clip all take both branches.  Branch guard of
test_tc_shapes_gpu._guarded_inputs, applied at every S_{k-1}: a row whose float64 ratio lies within 1e-4 of a clip
boundary, whose value delta lies within 1e-4 of +-eps_clip (or whose two clipped value errors tie), a ReLU row near a kink
or a categorical row near torch's probability clamp gets new inputs, and the case starts again -- so fp32 and fp64 take the
same side of every clip, min and max, and the comparison measures rounding."""
from dataclasses import dataclass

import numpy as np
import pytest
import torch

from oracle import oracle_np as onp
from tianshou_b200._cabi import OPT_RMSPROP
from test_simt_kernels_gpu import FAMILIES, _Discrete, _Fp64, _offsets, _perturb, _rollout_buffer
from test_tc_shapes_gpu import _rollout, _torch_fp32_forward
from ts_testutil import F32_EPS, Box, ac_named_params, actor_critic_reference_fp64, gaussian_dist, record_parity

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

PPO_KW = dict(gamma=0.99, gae_lambda=0.95, vf_coef=0.25, ent_coef=0.01, return_scaling=True, eps_clip=0.2, dual_clip=None,
              value_clip=True, advantage_normalization=True, recompute_advantage=False, max_grad_norm=0.5)
A2C_KW = dict(gamma=0.99, gae_lambda=0.95, vf_coef=0.5, ent_coef=0.01, return_scaling=True, max_grad_norm=0.5)

# family, network shape, algorithm + optimiser, rollout E x T, minibatch size, permutation source ("numpy": an explicit
# host permutation, "device": ts_make_permutation, "feed": the host permutation job's row feed), weight image on / off,
# clip: every step must clip ("all") / none may ("none"), pass2: check the pass boundary (alias: with the alias map)
CASES = {
    # merged wider last minibatch (300, 300, 400 rows: the launch is sized by the 4-tile one), pass boundary with the
    # next-observation alias map
    "tc-obs17-act6-ppo-merged-last-recompute-alias": dict(
        family="tanh_gauss", shape=(17, 6), algo="ppo", E=20, T=50, bs=300, perm="numpy", image=True,
        kw=dict(recompute_advantage=True), pass2=dict(alias=True)),
    # pass boundary without the alias map, no weight image (weights gathered by the CTAs), device permutation
    "tc-obs17-act6-ppo-recompute-no-alias-no-image-device-perm": dict(
        family="tanh_gauss", shape=(17, 6), algo="ppo", E=20, T=50, bs=250, perm="device", image=False,
        kw=dict(recompute_advantage=True, advantage_normalization=False), pass2=dict(alias=False)),
    # minibatches below one tile, dual clip, every step clips
    "tc-obs1-act1-ppo-bs64-dual-clip-every-step-clips": dict(
        family="tanh_gauss", shape=(1, 1), algo="ppo", E=8, T=64, bs=64, perm="numpy", image=True, clip="all",
        kw=dict(dual_clip=2.0, advantage_normalization=False, value_clip=False, max_grad_norm=1e-3)),
    # the widest network, A2C with RMSprop, rows from the host permutation job's feed
    "tc-obs32-act16-a2c-rmsprop-host-feed": dict(
        family="tanh_gauss", shape=(32, 16), algo="a2c", opt="rmsprop", E=12, T=50, bs=200, perm="feed", image=True,
        kw=dict()),
    # 32768-row minibatches: 256 tiles, several per CTA; weight decay; no step clips
    "tc-obs11-act3-ppo-bs32768-weight-decay-no-clip": dict(
        family="tanh_gauss", shape=(11, 3), algo="ppo", E=512, T=128, bs=32768, perm="numpy", image=True, clip="none",
        wd=0.01, kw=dict(max_grad_norm=1e3)),
    # SIMT kernels (one ts_ppo_grad + ts_clip_adam_step per step)
    "simt-relu_gauss-obs17-act6-a2c-adam": dict(
        family="relu_gauss", shape=(17, 6), algo="a2c", E=16, T=25, bs=100, perm="numpy", kw=dict()),
    "simt-tanh_gauss_shared-obs11-act3-ppo": dict(
        family="tanh_gauss_shared", shape=(11, 3), algo="ppo", E=16, T=25, bs=100, perm="numpy", kw=dict()),
    "simt-relu_cat_shared-obs8-act4-ppo-no-adv-norm-weight-decay": dict(
        family="relu_cat_shared", shape=(8, 4), algo="ppo", E=16, T=25, bs=100, perm="numpy", wd=0.01,
        kw=dict(advantage_normalization=False)),
    "simt-tanh_cat-obs17-act16-ppo-dual-clip": dict(
        family="tanh_cat", shape=(17, 16), algo="ppo", E=16, T=25, bs=100, perm="numpy", kw=dict(dual_clip=2.0)),
}
PASS2_STEPS = 3          # teacher-forced steps of pass 2


def _build(c):
    """test_simt_kernels_gpu._build with the optimiser of the case (Adam or RMSprop, weight decay)."""
    from tianshou_b200.algorithm import (A2C, PPO, AdamOptimizerFactory, DiscreteActorPolicy, ProbabilisticActorPolicy,
                                         RMSpropOptimizerFactory)
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.continuous import ContinuousActorProbabilistic, ContinuousCritic
    from tianshou_b200.utils.net.discrete import DiscreteActor, DiscreteCritic
    spec = FAMILIES[c["family"]]
    obs_dim, act_dim = c["shape"]
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
    if spec["cat"] and not spec["relu"]:
        # _perturb widens the tanh categorical head 16x to push rows into torch's probability clamp, test_simt_kernels_gpu's
        # subject; at orthogonal scale no probability comes near the clamp at any step, and the guard below has nothing to do
        with torch.no_grad():
            ac_named_params(actor, critic)["a_w3"].div_(16.0)
    wd = c.get("wd", 0.0)
    if c.get("opt") == "rmsprop":       # examples/mujoco/mujoco_a2c.py's optimiser
        optim = RMSpropOptimizerFactory(lr=7e-4, alpha=0.99, eps=1e-5, weight_decay=wd)
    else:
        optim = AdamOptimizerFactory(lr=3e-4, weight_decay=wd)
    if c["algo"] == "a2c":
        algo = A2C(policy=policy, critic=critic, optim=optim, **dict(A2C_KW, **c["kw"]))
    else:
        algo = PPO(policy=policy, critic=critic, optim=optim, **dict(PPO_KW, **c["kw"]))
    return algo, actor, critic


@dataclass
class State:
    p: torch.Tensor
    m: torch.Tensor
    v: torch.Tensor
    step: torch.Tensor

    def host(self):
        return (self.p.cpu().numpy().astype(np.float64), self.m.cpu().numpy().astype(np.float64),
                self.v.cpu().numpy().astype(np.float64), int(self.step.item()))


def _bits(a: np.ndarray) -> np.ndarray:
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def _assert_same_bits(what: str, got: np.ndarray, want: np.ndarray) -> None:
    diff = np.nonzero((_bits(got) != _bits(want)).reshape(got.shape[0], -1).any(1))[0]
    assert diff.size == 0, (f"{what}: differs bit for bit at row {int(diff[0])}: {got[diff[0]]} vs {want[diff[0]]} -- the "
                            f"result depends on work the kernel had not done yet")


def _within(key: str, got, want, bar) -> None:
    """|got - want| <= bar elementwise (bar: an array); the observed |err| / bar is recorded under ``key``."""
    got, want, bar = (np.asarray(x, dtype=np.float64) for x in (got, want, bar))
    err = np.abs(got - want)
    ratio = err / bar
    i = int(np.argmax(ratio))
    assert ratio[i] <= 1.0 and np.isfinite(got).all(), (
        f"{key}: element {i}: {got.flat[i]:.9g} vs {want.flat[i]:.9g} (|err| {err.flat[i]:.3e} > bar {bar.flat[i]:.3e}, "
        f"{ratio[i]:.3g}x)")
    record_parity(key + "/err_over_bar", ratio, np.zeros_like(ratio), rtol=0.0, atol=1.0)


class _Redraw(Exception):
    """Rows of the rollout that sit on a branch boundary at some S_{k-1}: new inputs, and the case starts again."""

    def __init__(self, lp=(), vs=(), obs=(), logp=None, v=None):
        super().__init__()
        self.lp, self.vs, self.obs, self.logp, self.v = lp, vs, obs, logp, v


class Case:
    def __init__(self, name):
        from tianshou_b200.data import Batch
        c = self.c = CASES[name]
        self.name = name
        self.spec = FAMILIES[c["family"]]
        self.algo, self.actor, self.critic = _build(c)
        algo, f = self.algo, self.algo._flat
        assert algo._layered is None
        assert (f.weight_image is not None) == (c["family"] == "tanh_gauss"), "tanh Gaussian (obs <= 32): tensor-core path"
        if not c.get("image", True):
            f.weight_image = None            # the epoch kernel then gathers + splits the weights in every CTA
        self.image = f.weight_image is not None
        obs_dim, act_dim = c["shape"]
        seed = obs_dim * 10 + act_dim
        if self.spec["cat"]:
            buf, self.roll = _rollout_buffer(c["family"], obs_dim, act_dim, c["E"], c["T"], seed), None
        else:
            buf, self.roll = _rollout(obs_dim, act_dim, c["E"], c["T"], seed)
        self.N = N = c["E"] * c["T"]
        batch, indices = algo._sample(buf, 0)
        self.batch = algo._preprocess_batch(batch, buf, indices)         # the rollout is preprocessed once
        assert torch.equal(indices.cpu(), torch.arange(N)), "a full buffer: batch row i is rollout row i"
        self.rms0 = algo._scratch["rms"].clone() if algo.return_scaling else None
        self.hp = algo._loss_hparams()
        self.ppo = c["algo"] == "ppo"
        self.rng = np.random.default_rng(seed)
        self.host = {k: getattr(self.batch, k).detach().cpu().numpy().copy()
                     for k in ("obs", "act", "v_s", "returns", "adv", "logp_old")}
        if self.ppo:       # a behaviour policy and a value net some updates old: every clip takes both branches
            self.host["logp_old"] = (self.host["logp_old"] + 0.5 * self.rng.standard_normal(N)).astype(np.float32)
            self.host["v_s"] = (self.host["v_s"] + 0.3 * self.rng.standard_normal(N)).astype(np.float32)
            self._upload()
        self.bounds = onp.minibatch_bounds(N, c["bs"])
        self.K = len(self.bounds)
        self.state0 = State(f.flat.clone(), f.exp_avg.clone(), f.exp_avg_sq.clone(), f.step_dev.clone())
        assert int(self.state0.step.item()) == 0 and not self.state0.m.any() and not self.state0.v.any()
        named = ac_named_params(self.actor, self.critic)
        self.offsets = {k: (off, named[k].numel(), tuple(named[k].shape))
                        for k, off in _offsets(f.flat, self.actor, self.critic).items()}
        assert sum(n for _, n, _ in self.offsets.values()) == f.n, "every flat slot belongs to one named parameter"
        repeat = 2 if "pass2" in c else 1
        if c["perm"] == "device":
            from tianshou_b200 import ops
            self.perm = ops.make_permutation(seed, 0, repeat, N, torch.device(DEV))
            ph = self.perm.cpu().numpy()
            assert all(np.array_equal(np.sort(r), np.arange(N)) for r in ph)
        else:
            np.random.seed(seed)
            ph = np.stack([np.random.permutation(N) for _ in range(repeat)]).astype(np.int32)
            self.perm = torch.from_numpy(ph).to(DEV)
        self.perm_host = ph
        self.feed_seed = seed if c["perm"] == "feed" else None
        self.Batch = Batch

    def _upload(self):
        for k in ("obs", "v_s", "logp_old"):
            col = getattr(self.batch, k)
            col.copy_(torch.from_numpy(self.host[k]).to(DEV).reshape(col.shape))

    def redraw(self, e: _Redraw):
        n_lp, n_vs, n_obs = len(e.lp), len(e.vs), len(e.obs)
        if n_lp:
            self.host["logp_old"][e.lp] = (e.logp + 0.5 * self.rng.standard_normal(n_lp)).astype(np.float32)
        if n_vs:
            self.host["v_s"][e.vs] = (e.v + 0.3 * self.rng.standard_normal(n_vs)).astype(np.float32)
        if n_obs:
            assert "pass2" not in self.c, "the alias map and the fp64 value recompute read the rollout's observations"
            self.host["obs"][e.obs] = self.rng.standard_normal((n_obs, self.c["shape"][0])).astype(np.float32)
        self._upload()

    # ------------------------------------------------------------------------------------------------ device runs
    def launch(self, state: State, bounds, perm_rows, batch_cols=None, nrep=1, recompute=False):
        """One ts_ppo_update_dedup call from ``state`` over ``bounds``: (S after the call, loss table, the batch it wrote)."""
        from tianshou_b200.algorithm.minibatch_order import MinibatchOrder
        algo, f = self.algo, self.algo._flat
        f.flat.copy_(state.p)
        f.exp_avg.copy_(state.m)
        f.exp_avg_sq.copy_(state.v)
        f.step_dev.copy_(state.step)
        if f.weight_image is not None:
            f.weight_image.zero_()
        if self.rms0 is not None:
            algo._scratch["rms"].copy_(self.rms0)
        b = self.Batch()
        b.__dict__.update(self.batch.__dict__)          # obs / obs_next stay the tensors the alias map was built from
        for k in ("v_s", "returns", "adv", "logp_old"):
            b.__dict__[k] = (batch_cols or self.batch.__dict__)[k].clone()
        stats = algo._alloc_stats(nrep * len(bounds))
        if self.feed_seed is None:
            algo._device_passes(b, perm_rows, bounds, self.hp, stats, nrep, recompute)
        else:
            assert perm_rows.data_ptr() == self.perm.data_ptr() and nrep == 1
            np.random.seed(self.feed_seed)           # the job draws the permutation of self.perm_host[0] again
            order = MinibatchOrder(algo, 1, self.N)
            assert order.feed is not None, "the host permutation job must feed the rows"
            try:
                algo._device_passes(b, order.rows, bounds, self.hp, stats, 1, recompute, feed=order.feed)
            finally:
                order.close(True)
            assert np.array_equal(order.rows.cpu().numpy(), self.perm_host[:1])
        torch.cuda.synchronize()
        if f.weight_image is not None:
            ctl = f.weight_image[:128].cpu().numpy()
            assert not ctl.any(), f"weight-image control block not zero after the launch: bytes {np.nonzero(ctl)[0].tolist()}"
        table = stats[:, :6].cpu().numpy()
        return State(f.flat.clone(), f.exp_avg.clone(), f.exp_avg_sq.clone(), f.step_dev.clone()), table, b

    # ------------------------------------------------------------------------------------------------ float64 side
    def hpr(self):
        c = dict(PPO_KW if self.ppo else A2C_KW, **self.c["kw"])
        if not self.ppo:
            return dict(loss_kind="a2c", vf_coef=c["vf_coef"], ent_coef=c["ent_coef"], advantage_normalization=False)
        return dict(eps_clip=c["eps_clip"], dual_clip=c["dual_clip"], value_clip=c["value_clip"],
                    advantage_normalization=c["advantage_normalization"], adv_eps=1e-8, vf_coef=c["vf_coef"],
                    ent_coef=c["ent_coef"])

    def reference(self, p_prev: torch.Tensor, rows: np.ndarray, cols: dict):
        """float64 autograd at parameters p_prev on ``rows``; raises _Redraw for rows on a branch boundary."""
        f = self.algo._flat
        f.flat.copy_(p_prev)              # the modules' parameters are views of the flat buffer
        mb = {k: cols[k][rows] for k in ("obs", "act", "adv", "returns", "logp_old", "v_s")}
        hpr = self.hpr()
        ref = actor_critic_reference_fp64(self.actor, self.critic, mb, hpr)
        self.guard(ref, mb, rows, hpr)
        g = np.zeros(f.n)
        for k, (off, n, _) in self.offsets.items():
            g[off:off + n] = ref["grads"][k].reshape(-1)
        return ref, g

    def guard(self, ref, mb, rows, hpr):
        obs_bad = np.zeros(len(rows), dtype=bool)
        if self.spec["relu"] or self.spec["cat"]:
            f64 = _Fp64(self.actor, self.critic, self.spec)
            if self.spec["relu"]:
                obs_bad |= f64.near_kink(mb["obs"])
            if self.spec["cat"]:       # test_simt_kernels_gpu._inputs: no probability within 4x of eps or 1 - eps
                pn, _ = f64.probs(mb["obs"])
                obs_bad |= (((pn > F32_EPS / 4) & (pn < 4 * F32_EPS)) | ((1 - pn > F32_EPS / 4) & (1 - pn < 4 * F32_EPS))).any(1)
        lp_bad = np.zeros(len(rows), dtype=bool)
        vs_bad = np.zeros(len(rows), dtype=bool)
        if self.ppo:
            e, dual = hpr["eps_clip"], hpr["dual_clip"] or 0.0
            ratio = np.exp(ref["logp"] - mb["logp_old"].astype(np.float64))
            lp_bad |= (np.abs(ratio - (1 - e)) < 1e-4) | (np.abs(ratio - (1 + e)) < 1e-4)
            if dual:
                A = mb["adv"].astype(np.float64)
                if hpr["advantage_normalization"]:
                    A = (A - A.mean()) / (A.std(ddof=1) + 1e-8)
                lp_bad |= (A < 0) & (np.abs(np.minimum(ratio * A, np.clip(ratio, 1 - e, 1 + e) * A) - dual * A) < 1e-4)
            if hpr["value_clip"]:
                v, vs, R = ref["v"], mb["v_s"].astype(np.float64), mb["returns"].astype(np.float64)
                dl = v - vs
                vc = vs + np.clip(dl, -e, e)
                vs_bad |= (np.abs(np.abs(dl) - e) < 1e-4) | ((np.abs(dl) > e) & (np.abs(np.abs(R - v) - np.abs(R - vc)) < 1e-4))
        if obs_bad.any() or lp_bad.any() or vs_bad.any():
            raise _Redraw(lp=rows[lp_bad], vs=rows[vs_bad], obs=rows[obs_bad], logp=ref["logp"][lp_bad], v=ref["v"][vs_bad])

    # ------------------------------------------------------------------------------------------------ the checks
    def check_step(self, tag, prev: State, cur: State, row: np.ndarray, rows: np.ndarray, cols: dict, clipped: list):
        ref, g = self.reference(prev.p, rows, cols)
        p0, m0, v0, step0 = prev.host()
        p1, m1, v1, step1 = cur.host()
        hp = self.hp
        # 2. the loss row: the step-0 bars of _epoch_vs_oracle (2e-4 relative, 2e-5 of max(1e-3, |value|); the actor loss in
        #    units of 1), here on every step
        for col, name, want in ((0, "loss", ref["loss"]), (1, "actor_loss", ref["clip"]), (2, "vf_loss", ref["vf"]),
                                (3, "ent_loss", ref["ent"])):
            unit = max(1e-3, abs(want), 1.0 if name == "actor_loss" else 0.0)
            record_parity(f"{tag}/{name}", row[col:col + 1], np.array([want]), rtol=2e-4, atol=2e-5 * unit)
        norm = float(np.sqrt((g * g).sum()))
        # pre-clip norm: test_simt_kernels_gpu's step-0 norm bar against the fp64 autograd gradient (2e-4 relative)
        record_parity(f"{tag}/grad_norm", row[4:5], np.array([norm]), rtol=2e-4, atol=0.0)
        assert row[5] == len(rows), f"{tag}: {row[5]} rows in the loss table, minibatch has {len(rows)}"
        # 3. moments.  Gradient bar per element of tensor t: the ts_ppo_grad bars, 2e-4 |g| + a_t max_t |g| + 1e-7 (a_t =
        #    1e-4 for a tensor-core weight-gradient GEMM output, 2e-5 otherwise); when clipping, the coefficient
        #    max_norm / (norm + 1e-6) is off by the norm's 2e-4 relative, another 2e-4 |g|
        M = hp.max_grad_norm
        coef = min(M / (norm + 1e-6), 1.0) if M > 0 else 1.0
        if M > 0:
            assert abs(norm - M) > 1e-3 * M, f"{tag}: gradient norm {norm} at the clip threshold {M}: the branch is a tie"
        clipped.append(M > 0 and norm > M)
        gb = np.zeros_like(g)
        tc = self.c["family"] == "tanh_gauss"            # the tensor-core kernels, with or without the weight image
        for k, (off, n, _) in self.offsets.items():
            gk = np.abs(g[off:off + n])
            a = 1e-4 if (tc and k[2] in "wb" and k[2:] != "b3") else 2e-5
            gb[off:off + n] = 2e-4 * gk + a * gk.max() + 1e-7 + (2e-4 * gk if clipped[-1] else 0.0)
        gb *= coef
        wd = hp.weight_decay
        gc = coef * g + wd * p0
        mag = np.abs(coef * g) + np.abs(wd * p0)      # |terms| of gc: fp32 rounding of the kernel's g + wd p
        ulp = 4.0 * F32_EPS
        rms = hp.optimizer == OPT_RMSPROP
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
        for k, (off, n, _) in self.offsets.items():
            s = slice(off, off + n)
            if not rms:
                _within(f"{tag}/exp_avg/{k}", m1[s], m_ref[s], m_bar[s])
            _within(f"{tag}/exp_avg_sq/{k}", v1[s], v_ref[s], v_bar[s])
        # 4. parameters: one fp64 step from S_{k-1} with S_k's moments.  Adam: the step is the kernel's own arithmetic on
        #    its own moments -- a few fp32 roundings of the step (8 ulp) and of the parameter (2 ulp).  RMSprop divides the
        #    clipped gradient itself: its error e moves the parameter by lr e / (sqrt(v) + eps) on top
        assert step1 == step0 + 1, f"{tag}: step counter {step1}, expected {step0 + 1}"
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
        for k, (off, n, _) in self.offsets.items():
            s = slice(off, off + n)
            _within(f"{tag}/param/{k}", p1[s], p_ref[s], p_bar[s])

    def prefix_pass(self, tag, start: State, r: int, n_steps: int, cols: dict, batch_cols=None):
        """Runs 1 .. n_steps of pass r from ``start``: every step checked; returns (S_{n_steps}, its loss table)."""
        prev, prev_table, clipped = start, None, []
        perm_rows = self.perm[r:r + 1]
        for k in range(1, n_steps + 1):
            cur, table, _ = self.launch(start, self.bounds[:k], perm_rows, batch_cols=batch_cols)
            step_tag = f"{tag}/step{k}"
            if prev_table is not None:
                _assert_same_bits(f"{step_tag}: loss rows 0..{k - 2} of run {k} vs run {k - 1}", table[:k - 1], prev_table)
            lo, hi = self.bounds[k - 1]
            self.check_step(step_tag, prev, cur, table[k - 1], self.perm_host[r][lo:hi], cols, clipped)
            prev, prev_table = cur, table
        want = self.c.get("clip")
        if want == "all":
            assert all(clipped), f"{tag}: steps {[i + 1 for i, x in enumerate(clipped) if not x]} did not clip"
        elif want == "none":
            assert not any(clipped), f"{tag}: steps {[i + 1 for i, x in enumerate(clipped) if x]} clipped"
        return prev, prev_table

    # ------------------------------------------------------------------------------------------------ pass boundary
    def check_pass2(self, S_K: State, table_K: np.ndarray):
        algo, f = self.algo, self.algo._flat
        tag = f"{self.name}/pass2"
        K, N = self.K, self.N
        alias = self.c["pass2"]["alias"]
        if not alias:
            algo._next_alias = None              # the recompute evaluates the critic on both inputs in full
        assert (algo._next_alias_map(self.batch) is not None) == alias
        S2, table2, b2 = self.launch(self.state0, self.bounds, self.perm, nrep=2, recompute=True)
        _assert_same_bits(f"{tag}: pass 1 of the repeat-2 update vs the prefix run over all {K} steps", table2[:K], table_K)
        # the value recompute at S_K, float64: critic, GAE, return scaling and RunningMeanStd with the state of pass 1
        p64 = {k: S_K.p.cpu().numpy().astype(np.float64)[off:off + n].reshape(shape)
               for k, (off, n, shape) in self.offsets.items()}
        rms = onp.RunningMeanStd()
        if self.rms0 is not None:
            m, var, cnt = self.rms0.cpu().numpy().tolist()
            rms.mean, rms.var, rms.count = m, var, int(round(cnt))
        scale = float(np.sqrt(rms.var + 1e-8)) if self.rms0 is not None else 1.0
        v64 = onp.critic_forward(p64, self.roll["obs"])
        v_ref, ret_ref, adv_ref = onp.add_returns_and_advantages(p64, self.roll, rms if self.rms0 is not None else None,
                                                                 algo.gamma, algo.gae_lambda)
        f.flat.copy_(S_K.p)
        v32 = _torch_fp32_forward(self.actor, self.critic, self.roll["obs"])[0]
        v32n = _torch_fp32_forward(self.actor, self.critic, self.roll["obs_next"])[0]
        v64n = onp.critic_forward(p64, self.roll["obs_next"])
        err_torch = max(float(np.abs(v32 - v64).max()), float(np.abs(v32n - v64n).max()))
        # v: test_tc_shapes_gpu's forward bar (8x torch fp32's own error + 2e-6 of max |v|)
        v_bar = 8.0 * err_torch + 2e-6 * float(np.abs(v64).max())
        record_parity(f"{tag}/v_s", b2.v_s.cpu().numpy(), v64, rtol=0.0, atol=v_bar)
        # adv: each TD error carries (1 + gamma) value errors (scaled by the return scale), the GAE sum weighs them by
        # (gamma lambda)^j, at most 1 / (1 - gamma lambda) in all; + fp32 output rounding
        gl = algo.gamma * algo.gae_lambda
        adv_err = (1 + algo.gamma) * v_bar * scale / (1 - gl)
        record_parity(f"{tag}/adv", b2.adv.cpu().numpy(), adv_ref, rtol=1e-6, atol=adv_err)
        # returns = (adv + v_s * scale) / scale
        ret_err = adv_err + v_bar * scale
        record_parity(f"{tag}/returns", b2.returns.cpu().numpy(), ret_ref, rtol=1e-6, atol=ret_err / scale)
        if self.rms0 is not None:
            got = algo._scratch["rms"].cpu().numpy()
            assert got[2] == rms.count, f"{tag}: RunningMeanStd count {got[2]} vs {rms.count}"
            # mean of returns off by ret_err at most; the variance by 2 max|ret - mean| ret_err + ret_err^2
            ret_unscaled = ret_ref.astype(np.float64) * scale
            record_parity(f"{tag}/rms_mean", got[:1], np.array([rms.mean]), rtol=1e-9, atol=ret_err)
            var_err = 2 * float(np.abs(ret_unscaled - rms.mean).max()) * ret_err + ret_err ** 2
            record_parity(f"{tag}/rms_var", got[1:2], np.array([rms.var]), rtol=1e-9, atol=var_err)
        # the first steps of pass 2, teacher-forced from S_K on the columns pass 2 wrote
        cols = dict(self.host, **{k: getattr(b2, k).cpu().numpy() for k in ("v_s", "returns", "adv")})
        batch_cols = dict(self.batch.__dict__, **{k: getattr(b2, k) for k in ("v_s", "returns", "adv")})
        J = min(K, PASS2_STEPS)
        S_J, table_J = self.prefix_pass(tag, S_K, 1, J, cols, batch_cols=batch_cols)
        _assert_same_bits(f"{tag}: steps 1..{J} of pass 2 in the repeat-2 update vs the teacher-forced runs", table2[K:K + J],
                          table_J)
        if J == K:
            for name, a, b in (("params", S2.p, S_J.p), ("exp_avg", S2.m, S_J.m), ("exp_avg_sq", S2.v, S_J.v)):
                assert torch.equal(a, b), f"{tag}: {name} after the repeat-2 update differ from the teacher-forced pass 2"

    def run(self):
        S_K, table_K = self.prefix_pass(f"{self.name}/pass1", self.state0, 0, self.K, self.host)
        if "pass2" in self.c:
            self.check_pass2(S_K, table_K)


@pytest.mark.parametrize("name", list(CASES))
def test_every_epoch_step_vs_fp64_from_own_state(name):
    case = Case(name)
    for attempt in range(6):
        try:
            case.run()
            return
        except _Redraw as e:
            case.redraw(e)
    pytest.fail(f"{name}: rows still on a branch boundary after {attempt + 1} redraws")
