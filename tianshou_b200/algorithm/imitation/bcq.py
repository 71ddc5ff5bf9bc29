"""Batch-constrained Q-learning (arXiv:1812.02900) with the whole ``update()`` and the policy's sample-and-select on the device.

Reference: tianshou/algorithm/imitation/bcq.py (BCQTrainingStats :23-28, BCQPolicy :34-116, BCQ :119-263),
utils/net/continuous.py:378-490 (Perturbation, VAE), algorithm_base.py:906-951 (OfflineAlgorithm), utils/lagged_network.py:8-80
(Polyak).

Per ``update(buffer, sample_size)``:
  host : index draw (numpy RandomState streams -- the reference's transitions); the VAE's ``eps`` through ``_noise_fn`` (the
         networks' device); the B * N target latents, then the B actor latents, each ``torch.randn`` on torch's CPU generator
         into pinned memory and uploaded without blocking; one D2H of the four losses at the end.
  GPU  : row gathers (device mirror or one upload); VAE: encoder -> the [mean | log_std] head (one [2L, H] GEMM) ->
         ``ts_bcq_vae_reparam`` (z straight into the decoder input) -> decoder -> ``ts_bcq_vae_loss`` -> decoder backward with its
         input gradient over z -> ``ts_bcq_vae_head_bwd`` -> head and encoder backward -> Adam; target: ``ts_bcq_decode_input``
         (s' repeated N times beside the clamped latents) -> decoder -> ``ts_bcq_act_rows`` -> both lagged critics ->
         ``ts_bcq_target``; per critic forward / MSE / backward + Adam; actor: decoder on [s | z] -> the perturbation network on
         row 0 (an ``MLP`` preprocess) or on every row (a ``Net``) -> ``ts_bcq_perturb`` -> critic 1 -> ``ts_td3_actor_rows`` ->
         critic 1's input gradient over the action columns -> ``ts_bcq_perturb_bwd`` -> perturbation backward + Adam; Polyak of
         the lagged perturbation network and both lagged critics.
Every Linear layer's forward / input gradient / weight gradient is one wgmma GEMM launch (csrc/net_gemm.cu).  The critic pair,
the critic step and Polyak are the twin-critic core's (algorithm/twin_critic.py, modelfree/sac.py); the perturbation network is
its actor.  The gradients the reference computes and then discards (the actor loss into the VAE and into critic 1) are cleared
by the next ``zero_grad`` there, so they are not computed here.
"""
from __future__ import annotations

import weakref
from copy import deepcopy
from dataclasses import dataclass
from typing import Any, Literal, cast

import numpy as np
import torch
from torch import nn

from ..._cabi import call, ptr, stream_ptr
from ...data import Batch, ReplayBuffer, to_torch
from ...utils.net.common import MLP, Net
from ..base import OfflineAlgorithm, Policy, TrainingStats, _space_kind
from ..flat_params import FlatGroup, UnsupportedModelError, bind_optimizer
from ..netgraph import ACT_NONE, FusedStack, _Layer, module_layers
from ..modelfree.sac import ContinuousTwinCritic, _linear_relu_chain
from ..optim import OptimizerFactory
from ..twin_critic import _EvalModeModule, cuda_device_of

LATENT_CLIP = 0.5          # VAE.decode's clamp of a drawn latent (continuous.py:486)


@dataclass(kw_only=True)
class BCQTrainingStats(TrainingStats):
    actor_loss: float
    critic1_loss: float
    critic2_loss: float
    vae_loss: float


class BCQPolicy(Policy):
    """BCQ's policy (bcq.py:34-116): per observation, ``forward_sampled_times`` actions decoded by the VAE, perturbed, and the one
    critic 1 values most (the first index of the maximum).

    Once a ``BCQ`` has bound the networks, ``forward`` with grad disabled and the modules on CUDA runs on the device: the B latent
    draws of (S, L) on torch's CPU generator in observation order (the reference's draws), one upload, one decoder forward over
    B * S rows, the perturbation network (B rows for an ``MLP`` preprocess, B * S for a ``Net``), critic 1, ``ts_bcq_select`` and
    one copy of the [B, A] actions to the host.  Otherwise it runs the reference's loop."""

    def __init__(self, *, actor_perturbation: nn.Module, action_space: Any, critic: nn.Module, vae: nn.Module,
                 forward_sampled_times: int = 100, observation_space: Any | None = None, action_scaling: bool = False,
                 action_bound_method: Literal["clip", "tanh"] | None = "clip") -> None:
        super().__init__(action_space=action_space, observation_space=observation_space, action_scaling=action_scaling,
                         action_bound_method=action_bound_method)
        self.actor_perturbation = actor_perturbation
        self.critic = critic
        self.vae = vae
        self.forward_sampled_times = forward_sampled_times
        self._fused: Any = None          # weakref to the BCQ that bound these networks

    def forward(self, batch: Batch, state: Any = None, **kwargs: Any) -> Batch:
        algo = self._fused() if self._fused is not None else None
        if algo is not None and not torch.is_grad_enabled() and algo._networks_bound():
            return cast(Batch, Batch(act=algo._select_actions(batch.obs)))
        device = next(self.parameters()).device
        obs_group: torch.Tensor = to_torch(batch.obs, device=device)
        act_group = []
        for obs_orig in obs_group:
            obs = (obs_orig.reshape(1, -1)).repeat(self.forward_sampled_times, 1)
            act = self.actor_perturbation(obs, self.vae.decode(obs))
            q1 = self.critic(obs, act)
            max_indice = q1.argmax(0)
            act_group.append(act[max_indice].cpu().data.numpy().flatten())
        return cast(Batch, Batch(act=np.array(act_group)))


def describe_perturbation(pert: Any) -> tuple[list[_Layer], list[nn.Parameter], int, int, bool]:
    """Perturbation(preprocess_net=MLP | Net, ...) -> (the Linear/ReLU chain on [s | a] ending in a linear layer of width A, its
    parameters, obs width, A, per_row).  ``per_row``: a ``Net`` preprocess (logits per row); an ``MLP`` (or a plain Sequential)
    yields row 0 of its output, which perturbs every row (continuous.py:409)."""
    pre = getattr(pert, "preprocess_net", None)
    if pre is None or getattr(pert, "max_action", None) is None or getattr(pert, "phi", None) is None:
        raise UnsupportedModelError("BCQ actor_perturbation: a Perturbation (preprocess_net, max_action, phi) expected")
    if isinstance(pre, Net):
        per_row = True
        if pre.softmax:
            raise UnsupportedModelError("BCQ actor_perturbation: softmax preprocess output unsupported")
    elif isinstance(pre, (MLP, nn.Sequential)):
        per_row = False
    else:
        raise UnsupportedModelError(f"BCQ actor_perturbation: preprocess_net must be an MLP or a Net, got {type(pre).__name__}")
    first = module_layers(pre)
    if not first or not isinstance(first[0], nn.Linear):
        raise UnsupportedModelError("BCQ actor_perturbation: preprocess_net must start with a Linear layer")
    layers = _linear_relu_chain(pre, int(first[0].in_features), "actor_perturbation.preprocess_net")
    if layers[-1].act != ACT_NONE:
        raise UnsupportedModelError("BCQ actor_perturbation: preprocess_net must end in a Linear layer (the logits)")
    A = layers[-1].out_dim
    O = layers[0].in_dim - A
    if O < 1:
        raise UnsupportedModelError(f"BCQ actor_perturbation: input width {layers[0].in_dim} leaves no room for {A} action columns")
    params: list[nn.Parameter] = []
    for L in layers:
        params += [L.weight, L.bias]
    return layers, params, O, A, per_row


def describe_vae(vae: Any, obs_dim: int, act_dim: int) -> tuple[list[_Layer], _Layer, list[_Layer], list[nn.Parameter], int]:
    """VAE -> (encoder chain on [s | a], the virtual [2L, H] head layer whose rows are (mean.weight ; log_std.weight) --
    adjacent in the flat buffer, so the head is one GEMM --, decoder chain on [s | z] ending in a linear layer of width A, the
    parameters in flat order, L)."""
    for name in ("encoder", "mean", "log_std", "decoder", "latent_dim", "max_action"):
        if getattr(vae, name, None) is None:
            raise UnsupportedModelError(f"BCQ vae: a VAE with {name} expected")
    L = int(vae.latent_dim)
    enc = _linear_relu_chain(vae.encoder, obs_dim + act_dim, "vae.encoder")
    mean, log_std = vae.mean, vae.log_std
    if not (isinstance(mean, nn.Linear) and isinstance(log_std, nn.Linear)):
        raise UnsupportedModelError("BCQ vae: mean / log_std must be Linear layers")
    H = enc[-1].out_dim
    if mean.in_features != H or log_std.in_features != H:
        raise UnsupportedModelError(f"BCQ vae: hidden_dim {mean.in_features} differs from the encoder's output width {H}")
    if mean.out_features != L or log_std.out_features != L:
        raise UnsupportedModelError(f"BCQ vae: latent_dim {L} differs from the mean / log_std width {mean.out_features}")
    dec_first = module_layers(vae.decoder)
    if not dec_first or not isinstance(dec_first[0], nn.Linear) or dec_first[0].in_features != obs_dim + L:
        width = dec_first[0].in_features if dec_first and isinstance(dec_first[0], nn.Linear) else None
        raise UnsupportedModelError(f"BCQ vae: the decoder must take obs {obs_dim} + latent {L} inputs, it takes {width}")
    dec = _linear_relu_chain(vae.decoder, obs_dim + L, "vae.decoder")
    if dec[-1].out_dim != act_dim or dec[-1].act != ACT_NONE:
        raise UnsupportedModelError(f"BCQ vae: the decoder must end in a Linear layer of width {act_dim}")
    params: list[nn.Parameter] = []
    for Ly in enc:
        params += [Ly.weight, Ly.bias]
    params += [mean.weight, log_std.weight, mean.bias, log_std.bias]
    for Ly in dec:
        params += [Ly.weight, Ly.bias]
    head = _Layer("linear", mean.weight, mean.bias, ACT_NONE, H, 2 * L)
    return enc, head, dec, params, L


class BCQ(ContinuousTwinCritic, OfflineAlgorithm):
    """Batch-constrained Q-learning (arXiv:1812.02900), reference API and semantics (bcq.py:119-263).

    The update reproduces what ``BCQ._update_with_batch`` computes, in its order:

    * the VAE step: ``vae_loss = mse(a, recon) + KL / 2`` with ``z = mean + std * eps`` (``eps`` from ``_noise_fn``, default
      ``torch.randn`` on the networks' device, the reference's ``randn_like``);
    * the target with the updated VAE: s' repeated N = ``num_sampled_action`` times, decoded with latents drawn on torch's CPU
      generator and clamped to +-0.5, NOT perturbed (the lagged perturbation network only moves by Polyak, as in the
      reference), ``lmbda * min + (1 - lmbda) * max`` of the lagged critics, the max over the N samples,
      ``rew + logical_not(done) * gamma * q``: one step, ``done``, no importance weight;
    * both critics take the plain MSE Adam step against that target;
    * the actor step: s decoded again with a fresh CPU draw, perturbed, ``-mean Q1`` against the updated critic 1.  With an
      ``MLP`` preprocess the perturbation network's output is indexed ``[0]``, so row 0's perturbation applies to the whole
      batch (reference behaviour, kept); with a ``Net`` every row has its own;
    * Polyak of the lagged perturbation network and both lagged critics.

    The update reads its four losses from the device once, at its end.  Refused with ``UnsupportedModelError``: a prioritised
    buffer, layers outside the fused family, softmax preprocess outputs, ``apply_preprocess_net_to_obs_only``, a VAE whose widths
    do not match its chains, optimisers other than Adam, modules off the GPU, non-Box action spaces.
    """

    def __init__(self, *, policy: BCQPolicy, actor_perturbation_optim: OptimizerFactory, critic_optim: OptimizerFactory,
                 vae_optim: OptimizerFactory, critic2: nn.Module | None = None, critic2_optim: OptimizerFactory | None = None,
                 gamma: float = 0.99, tau: float = 0.005, lmbda: float = 0.75, num_sampled_action: int = 10) -> None:
        super().__init__(policy=policy)
        if _space_kind(policy.action_space) != "continuous":
            raise UnsupportedModelError(f"BCQ supports Box action spaces only, got {policy.action_space=}")
        self.tau = tau
        self.actor_perturbation_target = _EvalModeModule(deepcopy(self.policy.actor_perturbation))
        self.critic_target = _EvalModeModule(deepcopy(self.policy.critic))
        self.critic2 = critic2 or deepcopy(self.policy.critic)
        self.critic2_target = _EvalModeModule(deepcopy(self.critic2))
        self.gamma = gamma
        self.lmbda = lmbda
        self.num_sampled_action = num_sampled_action
        if int(num_sampled_action) < 1:
            raise ValueError(f"num_sampled_action must be at least 1, got {num_sampled_action}")
        pert = self.policy.actor_perturbation
        _, _, obs_dim, _, self._per_row = describe_perturbation(pert)
        self._build_networks(lagged=(self.critic_target.module, self.critic2_target.module),
                             lagged_actor=self.actor_perturbation_target.module, policy_optim=actor_perturbation_optim,
                             critic_optim=critic_optim, critic2_optim=critic2_optim, actor=pert, obs_dim=obs_dim)
        self.actor_perturbation_optim = self.policy_optim
        dev = self._dev
        vae = self.policy.vae
        if cuda_device_of(vae) != dev:
            raise UnsupportedModelError(f"BCQ vae lives on {cuda_device_of(vae)}, the other networks on {dev}")
        enc, head, dec, v_params, self.latent_dim = describe_vae(vae, self.obs_dim, self.act_dim)
        self._g_vae = FlatGroup(v_params, dev)
        self._enc, self._head, self._dec = (FusedStack(enc, self._g_vae, "vae.encoder"), FusedStack([head], self._g_vae, "vae.head"),
                                            FusedStack(dec, self._g_vae, "vae.decoder"))
        self.vae_optim = self._create_optimizer(vae, vae_optim)
        bind_optimizer(self.vae_optim, self._g_vae)
        # the VAE's eps: torch.randn on the networks' device (randn_like, continuous.py:470)
        self._noise_fn = lambda shape: torch.randn(shape, device=dev)
        self.policy._fused = weakref.ref(self)

    @property
    def critic(self) -> nn.Module:
        """Critic 1 is the policy's (bcq.py:175): not a module of its own here, so ``state_dict()`` keeps the reference's keys."""
        return self.policy.critic

    def _describe_actor(self, actor: nn.Module, obs_dim: int) -> tuple[list[_Layer], list[nn.Parameter], int]:
        layers, params, _, A, _ = describe_perturbation(actor)
        return layers, params, A

    def _preprocess_batch(self, batch: Batch, buffer: ReplayBuffer, indices: np.ndarray) -> Batch:
        """Nothing: BCQ's one-step target is part of its update (bcq.py:210-237), there is no n-step return."""
        return batch

    # ------------------------------------------------------------------ helpers
    def _cpu_latents(self, rows: int) -> torch.Tensor:
        """``torch.randn((rows, L))`` on torch's CPU generator (VAE.decode, continuous.py:485-487) drawn into pinned memory and
        uploaded without blocking the host."""
        z = torch.randn((rows, self.latent_dim), pin_memory=True)
        return z.to(self._dev, non_blocking=True)

    def _decode(self, s: torch.Tensor, N: int, z: torch.Tensor, tag: str) -> tuple[torch.Tensor, torch.Tensor]:
        """VAE.decode on s repeated N times with the drawn latents z: (decoder input [s | clamp(z)], decoder output)."""
        B, O, L = s.shape[0], self.obs_dim, self.latent_dim
        x = self._buf(tag + "_dx", (B * N, O + L))
        call("ts_bcq_decode_input", ptr(s), B, N, O, ptr(z), L, LATENT_CLIP, ptr(x), stream_ptr(self._dev))
        return x, self._dec.forward(x, B * N, tag)[-1]

    def _perturb(self, x_dec: torch.Tensor, y: torch.Tensor, groups: int, S: int, tag: str
                 ) -> tuple[list[torch.Tensor], torch.Tensor, int, int]:
        """Perturbation.forward on the decoded actions of ``groups`` groups of S rows, into critic 1's input [s | perturbed]:
        (the perturbation network's activations, that input, its logits rows, its group size)."""
        O, A, st = self.obs_dim, self.act_dim, stream_ptr(self._dev)
        pert = self.policy.actor_perturbation
        rows, G = groups * S, (groups * S if self._per_row else groups)
        step = 1 if self._per_row else S
        xp = self._buf(tag + "_xp", (G, O + A))
        call("ts_bcq_act_rows", ptr(x_dec), O + self.latent_dim, ptr(y), step, G, O, A, float(self.policy.vae.max_action), ptr(xp), st)
        p_acts = self._actor.forward(xp, G, tag)
        group = 1 if self._per_row else S
        xq = self._buf(tag + "_xq", (rows, O + A))
        call("ts_bcq_perturb", ptr(p_acts[-1]), group, ptr(y), rows, A, float(self.policy.vae.max_action), float(pert.max_action),
             float(pert.phi * pert.max_action), ptr(x_dec), O + self.latent_dim, O, ptr(xq), st)
        return p_acts, xq, G, group

    def _networks_bound(self) -> bool:
        """The device policy path applies: every module of the policy still on this algorithm's CUDA device."""
        return all(p.device == self._dev for p in self.policy.parameters())

    # ------------------------------------------------------------------ policy
    def _select_actions(self, obs: Any) -> np.ndarray:
        """BCQPolicy.forward on the device (bcq.py:100-116)."""
        dev, st = self._dev, stream_ptr(self._dev)
        obs = torch.as_tensor(np.asarray(obs) if not isinstance(obs, torch.Tensor) else obs)
        B = obs.shape[0]
        S, O, A, L = int(self.policy.forward_sampled_times), self.obs_dim, self.act_dim, self.latent_dim
        host = torch.empty(B * O + B * S * L, dtype=torch.float32, pin_memory=True)
        host[:B * O].copy_(obs.reshape(-1))
        z = host[B * O:].view(B * S, L)
        for b in range(B):                                    # the reference's draws, one (S, L) per observation, in order
            torch.randn((S, L), out=z[b * S:(b + 1) * S])
        dev_in = host.to(dev, non_blocking=True)
        s, z_d = dev_in[:B * O].view(B, O), dev_in[B * O:].view(B * S, L)
        x_dec, y = self._decode(s, S, z_d, "pf")
        _, xq, _, _ = self._perturb(x_dec, y, B, S, "pf")
        q = self._c[0].forward(xq, B * S, "pf")[-1]
        act = self._buf("pf_act", (B, A))
        call("ts_bcq_select", ptr(q), B, S, ptr(xq), O + A, O, A, ptr(act), None, st)
        return act.cpu().numpy()

    # ------------------------------------------------------------------ update
    def _sample(self, buffer: ReplayBuffer, sample_size: int | None) -> tuple[Batch, Any]:
        """Indices from the buffer's host RNG streams (identical to the reference's draws); rows stay on the device."""
        from ... import ops
        if hasattr(buffer, "update_weight") or hasattr(buffer, "get_weight"):
            raise UnsupportedModelError("BCQ: prioritised replay unsupported -- the reference's losses carry no importance weight")
        indices = np.asarray(buffer.sample_indices(sample_size), dtype=np.int64)
        dev = self._dev
        cols = buffer.device_columns() if hasattr(buffer, "device_columns") else None
        at = torch.from_numpy(indices).pin_memory().to(dev, non_blocking=True) if cols is not None else indices
        rows = lambda key, where: ops.buffer_rows(buffer, key, where, dev, cols=cols).contiguous()
        batch = Batch()
        d = batch.__dict__
        d["obs"], d["act"] = rows("obs", at), rows("act", at)
        d["obs_next"] = rows("obs_next", at) if buffer._save_obs_next else rows("obs", buffer.next(indices))
        d["rew"], d["done"] = rows("rew", at).view(-1), rows("done", at).view(-1)
        d["info"] = Batch()
        return batch, indices

    def _vae_step(self, obs: torch.Tensor, act: torch.Tensor, out_loss: torch.Tensor) -> None:
        """The VAE step (bcq.py:201-208): forward with z = mean + std * eps, the loss, backward, Adam."""
        B, O, A, L = obs.shape[0], self.obs_dim, self.act_dim, self.latent_dim
        st = stream_ptr(self._dev)
        x = self._buf("v_x", (B, O + A))
        self._concat(obs, act, x)
        e_acts = self._enc.forward(x, B, "v")
        h_acts = self._head.forward(e_acts[-1], B, "v")
        head = h_acts[-1]
        eps = self._noise_fn((B, L)).to(self._dev, torch.float32).contiguous()
        std, xz = self._buf("v_std", (B, L)), self._buf("v_xz", (B, O + L))
        call("ts_bcq_vae_reparam", ptr(head), ptr(eps), B, L, ptr(obs), O, ptr(std), ptr(xz), st)
        d_acts = self._dec.forward(xz, B, "v")
        dy = self._buf("v_dy", (B, A))
        call("ts_bcq_vae_loss", ptr(d_acts[-1]), ptr(act), ptr(head), ptr(std), B, A, L, float(self.policy.vae.max_action), ptr(dy),
             ptr(out_loss), st)
        dz = self._buf("v_dz", (B, L))
        self._dec.backward(d_acts, dy, B, "v", input_grad=True, input_cols=(O, O + L), dx_out=dz)
        dhead = self._buf("v_dhead", (B, 2 * L))
        call("ts_bcq_vae_head_bwd", ptr(head), ptr(std), ptr(eps), ptr(dz), B, L, ptr(dhead), st)
        enc_act = self._enc.layers[-1].act
        dh = self._head.backward(h_acts, dhead, B, "v", input_grad=True,
                                 input_act=(enc_act, e_acts[-1]) if enc_act != ACT_NONE else None)
        self._enc.backward(e_acts, dh, B, "v", dy_preact=True)
        self._adam(self._g_vae, self.vae_optim._optim, self.vae_optim._max_grad_norm)

    def _target(self, obs_next: torch.Tensor, rew: torch.Tensor, done: torch.Tensor) -> torch.Tensor:
        """The one-step target with the updated VAE (bcq.py:211-237)."""
        B, N, O, A = obs_next.shape[0], int(self.num_sampled_action), self.obs_dim, self.act_dim
        st = stream_ptr(self._dev)
        x_dec, y = self._decode(obs_next, N, self._cpu_latents(B * N), "t")
        xc = self._buf("t_xc", (B * N, O + A))
        call("ts_bcq_act_rows", ptr(x_dec), O + self.latent_dim, ptr(y), 1, B * N, O, A, float(self.policy.vae.max_action), ptr(xc), st)
        q = [self._lagged_forward(k, xc, B * N, "tq")[-1] for k in range(2)]
        out = self._buf("target", B)
        call("ts_bcq_target", ptr(q[0]), ptr(q[1]), B, N, float(self.lmbda), float(1 - self.lmbda), ptr(rew), ptr(done),
             float(self.gamma), ptr(out), st)
        return out

    def _actor_step(self, obs: torch.Tensor, out_loss: torch.Tensor) -> None:
        """The perturbation step (bcq.py:247-253) against the updated critic 1."""
        B, O, A = obs.shape[0], self.obs_dim, self.act_dim
        st = stream_ptr(self._dev)
        pert = self.policy.actor_perturbation
        x_dec, y = self._decode(obs, 1, self._cpu_latents(B), "a")
        p_acts, xq, G, group = self._perturb(x_dec, y, 1, B, "a")          # the group is the whole batch
        c_acts = self._c[0].forward(xq, B, "aq")
        dq = self._buf("adq", (B, 1))
        call("ts_td3_actor_rows", ptr(c_acts[-1]), None, None, B, A, 1.0, 0.0, ptr(dq), ptr(out_loss), st)
        dact = self._buf("dact", (B, A))
        self._c[0].backward(c_acts, dq, B, "aq", param_grads=False, input_grad=True, input_cols=(O, O + A), dx_out=dact)
        dl = self._buf("dlogits", (G, A))
        call("ts_bcq_perturb_bwd", ptr(p_acts[-1]), group, G, ptr(y), ptr(dact), A, float(self.policy.vae.max_action),
             float(pert.max_action), float(pert.phi * pert.max_action), ptr(dl), st)
        self._actor.backward(p_acts, dl, G, "a")
        self._adam(self._g_actor, self.policy_optim._optim, self.policy_optim._max_grad_norm)

    def _device_update(self, batch: Batch) -> torch.Tensor:
        """Everything of one update after the sampling, with no host synchronisation; returns the device losses (actor, critic 1,
        critic 2, vae)."""
        obs, act = batch.obs, batch.act
        B = obs.shape[0]
        losses = self._buf("losses", 4)
        self._vae_step(obs, act, losses[3:4])
        target = self._target(batch.obs_next, batch.rew, batch.done)
        x = self._buf("cu_x", (B, self.obs_dim + self.act_dim))
        self._concat(obs, act, x)
        self._critic_step(0, x, target, None, self.critic_optim, losses[1:2])
        self._critic_step(1, x, target, None, self.critic2_optim, losses[2:3])
        self._actor_step(obs, losses[0:1])
        self._polyak()
        return losses

    def _update_with_batch(self, batch: Batch) -> BCQTrainingStats:
        l = self._device_update(batch).cpu().numpy()        # the only host read of the update
        return BCQTrainingStats(actor_loss=float(l[0]), critic1_loss=float(l[1]), critic2_loss=float(l[2]), vae_loss=float(l[3]))
