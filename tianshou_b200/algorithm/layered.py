"""Actor-critic structure, and the networks OUTSIDE the fused 17-64-64 kernels' shape envelope layer by layer on the tensor cores.

``parse_actor_critic`` reads the actor / critic modules once: every on-policy algorithm runs what it accepts, and
``fused_descriptor`` picks out the shapes the persistent tensor-core / SIMT update kernels were written for (two-layer
64-wide trunks, obs <= 64).  Everything else that is still a Linear / ReLU | Tanh actor-critic -- wider or deeper trunks,
large observations (Humanoid: 376), the reference's shared-trunk discrete PPO net at other widths -- runs in
``LayeredActorCritic``: every Linear forward / input gradient / weight gradient is one ``ts_net_gemm`` launch (wgmma,
fp32-faithful), the PPO / A2C loss between them is ``ts_ppo_rows``, the optimiser ``ts_adam_step`` / ``ts_rmsprop_step`` (global-norm clip + Adam or RMSprop).
Same public behaviour as the fused path (ppo.py:146-224, a2c.py:115-153); single GPU.

Reference structures covered: ``ContinuousActorProbabilistic(unbounded=True, conditioned_sigma=False)`` +
``ContinuousCritic`` (utils/net/continuous.py:96-238), ``DiscreteActor(softmax_output=True)`` + ``DiscreteCritic`` on
separate or ONE shared ``Net`` (utils/net/discrete.py:29-123, test/discrete/test_ppo_discrete.py:90-100).
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Any

import torch
from torch import nn

from .. import ops
from .._cabi import AC_CATEGORICAL, AC_RELU, STATS_STRIDE, ActorCriticDesc, call, ptr, stream_ptr
from .flat_params import DeviceScratch, FlatGroup, UnsupportedModelError
from .netgraph import ACT_NONE, ACT_RELU, FusedStack, _Layer, compile_sequential, layer_params, module_layers

_CHUNK = 131072          # rows per forward chunk of the whole-rollout passes (bounds the activation scratch)


@dataclass
class ActorCriticSpec:
    """The structure of an accepted actor-critic.  ``group_params``: the parameters of each layer-wise ``FlatGroup`` in
    module order -- one group (``ActorCritic(actor, critic).parameters()``, a shared trunk once), or the actor's and the
    critic's when ``split``."""
    obs_dim: int
    act_dim: int
    categorical: bool
    shared: bool
    sigma_param: nn.Parameter | None
    a_trunk: list[_Layer]
    a_head: list[_Layer]
    c_trunk: list[_Layer]
    c_head: list[_Layer]
    group_params: list[list[nn.Parameter]]


def parse_actor_critic(actor: Any, critic: Any, *, split: bool) -> ActorCriticSpec:
    """Validate the actor / critic modules and compile their layers; raises ``UnsupportedModelError`` for anything the
    kernels do not run.  Pure: allocates nothing and works on modules on any device.  ``split``: the actor and the critic
    get one parameter group each (NPG / TRPO step the actor along the natural gradient and the critic with its own
    optimiser).  A trunk is shared when actor and critic hold the very same trunk parameters; sharing only some of them is
    refused (the two backward passes would overwrite each other's gradient in the shared slots)."""
    categorical = hasattr(actor, "softmax_output")
    if categorical and not actor.softmax_output:
        raise UnsupportedModelError("actor: DiscreteActor needs softmax_output=True (Categorical over probabilities)")
    if not categorical:
        if getattr(actor, "_c_sigma", False) or not hasattr(actor, "sigma_param"):
            raise UnsupportedModelError("actor: conditioned sigma unsupported (need state-independent sigma_param)")
        if not getattr(actor, "_unbounded", False):
            raise UnsupportedModelError("actor: only unbounded=True (mu without tanh) is supported")
    if getattr(critic, "apply_preprocess_net_to_obs_only", False):
        raise UnsupportedModelError("critic: apply_preprocess_net_to_obs_only unsupported")
    for net, what in ((actor.preprocess, "actor"), (critic.preprocess, "critic")):
        if getattr(net, "softmax", False):
            raise UnsupportedModelError(f"{what}: softmax trunk output unsupported")
    a_mods = module_layers(actor.preprocess)
    first = next((m for m in a_mods if isinstance(m, nn.Linear)), None)
    if first is None:
        raise UnsupportedModelError("actor trunk has no Linear layer")
    obs_dim = int(first.in_features)
    a_trunk = compile_sequential(a_mods, (obs_dim,))
    c_trunk = compile_sequential(module_layers(critic.preprocess), (obs_dim,))
    a_head = compile_sequential(module_layers(actor.last if categorical else actor.mu), (a_trunk[-1].out_dim,))
    c_head = compile_sequential(module_layers(critic.last), (c_trunk[-1].out_dim,))
    if a_head[-1].act != ACT_NONE or c_head[-1].act != ACT_NONE or c_head[-1].out_dim != 1:
        raise UnsupportedModelError("heads must end in a linear layer (critic: one output)")
    act_dim = int(a_head[-1].out_dim)
    if act_dim > 64:
        raise UnsupportedModelError("action width > 64 unsupported")
    a_ids, c_ids = set(map(id, actor.parameters())), set(map(id, critic.parameters()))
    trunk_ids = [id(p) for p in layer_params(a_trunk)]
    shared = trunk_ids == [id(p) for p in layer_params(c_trunk)] and [L.act for L in a_trunk] == [L.act for L in c_trunk]
    if (a_ids & c_ids) != (set(trunk_ids) if shared else set()):
        raise UnsupportedModelError("partially shared trunks are unsupported")
    if split and shared:
        raise UnsupportedModelError("a critic-only optimiser (NPG / TRPO) needs separate actor and critic trunks; "
                                    "shared trunks are unsupported")
    params = list({id(p): p for p in [*actor.parameters(), *critic.parameters()]}.values())   # ActorCritic order, shared once
    sigma_param = None if categorical else actor.sigma_param
    covered = {id(p) for p in layer_params([*a_trunk, *c_trunk, *a_head, *c_head])}
    if [id(p) for p in params if id(p) not in covered] != ([] if categorical else [id(sigma_param)]):
        raise UnsupportedModelError("actor / critic hold parameters outside the Linear layers")
    return ActorCriticSpec(obs_dim, act_dim, categorical, shared, sigma_param, a_trunk, a_head, c_trunk, c_head,
                           [list(actor.parameters()), list(critic.parameters())] if split else [params])


def fused_descriptor(spec: ActorCriticSpec) -> tuple[ActorCriticDesc, list[nn.Parameter]] | None:
    """(descriptor, parameters in flat-buffer order) for the fused tensor-core / SIMT kernels, or None when the networks are
    outside their envelope: trunks exactly Linear+act -> Linear+act, 64 wide, one activation (Tanh or ReLU) in both, each
    head a single Linear, obs_dim <= 64, act_dim <= 16.  Two families: the MuJoCo one (Gaussian head, separate trunks) and
    the reference's discrete PPO test net (test/discrete/test_ppo_discrete.py:90-100), optionally on ONE shared trunk, which
    appears once in the flat buffer while both networks' descriptor offsets alias it."""
    trunks = (spec.a_trunk, spec.c_trunk)
    if any(len(t) != 2 or any(L.kind != "linear" or L.act == ACT_NONE or L.out_dim != 64 for L in t) for t in trunks):
        return None
    if len({L.act for t in trunks for L in t}) != 1 or len(spec.a_head) != 1 or len(spec.c_head) != 1:
        return None
    if spec.obs_dim > 64 or spec.act_dim > 16:
        return None
    (a1, a2), (c1, c2), a3, c3 = spec.a_trunk, spec.c_trunk, spec.a_head[0], spec.c_head[0]
    named = [("a_w1", a1.weight), ("a_b1", a1.bias), ("a_w2", a2.weight), ("a_b2", a2.bias), ("a_w3", a3.weight),
             ("a_b3", a3.bias)]
    if not spec.categorical:
        named.append(("a_logstd", spec.sigma_param))
    if not spec.shared:
        named += [("c_w1", c1.weight), ("c_b1", c1.bias), ("c_w2", c2.weight), ("c_b2", c2.bias)]
    named += [("c_w3", c3.weight), ("c_b3", c3.bias)]
    d = ActorCriticDesc()
    d.obs_dim, d.act_dim, d.hidden = spec.obs_dim, spec.act_dim, 64
    d.flags = (AC_RELU if a1.act == ACT_RELU else 0) | (AC_CATEGORICAL if spec.categorical else 0)
    d.a_logstd = -1
    off = 0
    for name, p in named:
        setattr(d, name, off)
        off += p.numel()
    if spec.shared:
        d.c_w1, d.c_b1, d.c_w2, d.c_b2 = d.a_w1, d.a_b1, d.a_w2, d.a_b2
    d.n_params = off
    return d, [p for _, p in named]


class LayeredActorCritic:
    def __init__(self, spec: ActorCriticSpec, device: torch.device) -> None:
        """One ``FlatGroup`` per entry of ``spec.group_params``: ``group`` holds the actor, ``critic_group`` the critic
        (the same group unless the spec is split)."""
        self.device = device
        self.categorical, self.shared, self.act_dim = spec.categorical, spec.shared, spec.act_dim
        groups = [FlatGroup(p, device) for p in spec.group_params]
        self.group, self.critic_group = groups[0], groups[-1]
        self.a_trunk, self.a_head = FusedStack(spec.a_trunk, self.group, "a_trunk"), FusedStack(spec.a_head, self.group, "a_head")
        self.c_trunk = self.a_trunk if self.shared else FusedStack(spec.c_trunk, self.critic_group, "c_trunk")
        self.c_head = FusedStack(spec.c_head, self.critic_group, "c_head")
        self.sigma_param = spec.sigma_param
        self._a_act, self._c_act = spec.a_trunk[-1].act, spec.c_trunk[-1].act
        self._scratch = DeviceScratch(device)
        self._buf = self._scratch.tensor

    # ------------------------------------------------------------------ helpers
    def _logstd_ptr(self, buf: torch.Tensor) -> int | None:
        return None if self.categorical else buf.data_ptr() + 4 * self.group.offset(self.sigma_param)

    def _act_rows(self, act: torch.Tensor) -> torch.Tensor:
        a = act.reshape(act.shape[0], -1).to(torch.float32)
        return a.reshape(-1).contiguous() if self.categorical else a.contiguous()

    # ------------------------------------------------------------------ whole-rollout passes (no grad)
    def critic_values(self, obs: torch.Tensor, out: torch.Tensor) -> None:
        """out[r] = critic(obs[r])  (a2c.py:123-126) in row chunks."""
        n = obs.shape[0]
        for lo in range(0, n, _CHUNK):
            hi = min(n, lo + _CHUNK)
            t = self.c_trunk.forward(obs[lo:hi], hi - lo, "vp")
            h = self.c_head.forward(t[-1], hi - lo, "vp")
            out[lo:hi].copy_(h[-1].view(-1))

    def actor_logp(self, obs: torch.Tensor, act: torch.Tensor, out: torch.Tensor, hp: Any) -> None:
        """out[r] = log pi(act[r] | obs[r])  (ppo.py:157-161)."""
        n = obs.shape[0]
        a = self._act_rows(act)
        for lo in range(0, n, _CHUNK):
            hi = min(n, lo + _CHUNK)
            t = self.a_trunk.forward(obs[lo:hi], hi - lo, "lp")
            h = self.a_head.forward(t[-1], hi - lo, "lp")
            call("ts_ppo_rows", ptr(h[-1]), None, self._logstd_ptr(self.group.flat), ptr(a[lo:hi]), None, None, None, None, hi - lo,
                 self.act_dim, int(self.categorical), C.byref(hp), hi - lo, None, ptr(out[lo:hi]), None, None, None, None,
                 stream_ptr(self.device))

    def actor_head(self, obs: torch.Tensor) -> torch.Tensor:
        """mu / logits for ``obs`` (Collector-side inference)."""
        t = self.a_trunk.forward(obs, obs.shape[0], "inf")
        return self.a_head.forward(t[-1], obs.shape[0], "inf")[-1]

    # ------------------------------------------------------------------ one optimiser step
    def minibatch_step(self, batch: Any, idx: torch.Tensor, hp: Any, adv_moments: torch.Tensor | None, optimizer: torch.optim.Optimizer,
                       max_grad_norm: float | None, stats_row: torch.Tensor) -> None:
        """Gather the minibatch rows, forward, loss rows, backward, clip + Adam, stats  (ppo.py:179-216, algorithm_base.py:496-500)."""
        st = stream_ptr(self.device)
        B, A = int(idx.numel()), self.act_dim
        obs = ops.gather_rows(batch.obs, idx)
        act = ops.gather_rows(self._act_rows(batch.act), idx)
        adv, ret = ops.gather_rows(batch.adv, idx), ops.gather_rows(batch.returns, idx)
        lpo, vso = ops.gather_rows(batch.logp_old, idx), ops.gather_rows(batch.v_s, idx)
        at = self.a_trunk.forward(obs, B, "up")
        ah = self.a_head.forward(at[-1], B, "up")
        ct = at if self.shared else self.c_trunk.forward(obs, B, "up")
        ch = self.c_head.forward(ct[-1], B, "up")
        logp = self._buf("logp", B)
        dhead, dval = self._buf("dhead", (B, A)), self._buf("dval", (B, 1))
        dls = None if self.categorical else self._buf("dls", (B, A))
        rows = self._buf("loss_rows", (B, 3))
        call("ts_ppo_rows", ptr(ah[-1]), ptr(ch[-1]), self._logstd_ptr(self.group.flat), ptr(act), ptr(adv), ptr(ret), ptr(lpo), ptr(vso),
             B, A, int(self.categorical), C.byref(hp), B, ptr(adv_moments), ptr(logp), ptr(dhead), ptr(dval), ptr(dls), ptr(rows), st)
        call("ts_ppo_rows_stats", ptr(rows), B, C.byref(hp), ptr(stats_row), st)
        # backward: heads -> d loss / d (trunk pre-activation), then the trunk(s)
        dz_a = self._buf("dz_a", (B, self.a_trunk.layers[-1].out_dim))
        self.a_head.backward(ah, dhead, B, "up", input_grad=True, input_act=(self._a_act, at[-1]) if self._a_act != ACT_NONE else None,
                             dx_out=dz_a)
        if self.shared:
            self.c_head.backward(ch, dval, B, "up", input_grad=True, input_act=(self._c_act, ct[-1]) if self._c_act != ACT_NONE else None,
                                 dx_out=dz_a, dx_accumulate=True)
            self.a_trunk.backward(at, dz_a, B, "up", dy_preact=True)
        else:
            dz_c = self._buf("dz_c", (B, self.c_trunk.layers[-1].out_dim))
            self.c_head.backward(ch, dval, B, "up", input_grad=True, input_act=(self._c_act, ct[-1]) if self._c_act != ACT_NONE else None,
                                 dx_out=dz_c)
            self.a_trunk.backward(at, dz_a, B, "up", dy_preact=True)
            self.c_trunk.backward(ct, dz_c, B, "up", dy_preact=True)
        if dls is not None:
            call("ts_net_colsum", ptr(dls), A, B, A, self._logstd_ptr(self.group.grad), 0, st)
        self.group.optimizer_step(optimizer, max_grad_norm)


def layered_update(algo: Any, batch: Any, batch_size: int | None, repeat: int, order: Any) -> torch.Tensor:
    """The repeat x minibatch loop (ppo.py:164-224) on a layered actor-critic in the passes' ``MinibatchOrder``; returns the
    device loss table [steps, 8]."""
    from ..data.batch import minibatch_bounds
    L: LayeredActorCritic = algo._layered
    N = batch.obs.shape[0]
    bounds = minibatch_bounds(N, batch_size or N, merge_last=True)
    n_mb = len(bounds)
    hp = algo._loss_hparams()
    stats = torch.zeros((repeat * n_mb, STATS_STRIDE), dtype=torch.float32, device=L.device)
    for r in range(repeat):
        if algo.recompute_adv and r > 0:
            algo._add_returns_and_advantages(batch, None, None)
        order.ready(r)
        perm = order.rows[r]
        for m, (lo, hi) in enumerate(bounds):
            adv_mom = algo._minibatch_adv_moments(batch, perm, lo, hi, 1) if algo.advantage_normalization else None
            idx = perm[lo:hi].to(torch.int64)
            L.minibatch_step(batch, idx, hp, adv_mom, algo.optim._optim, algo.optim._max_grad_norm, stats[r * n_mb + m])
    return stats
