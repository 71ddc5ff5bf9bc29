"""The intrinsic curiosity module (ICM, arXiv:1705.05363) as a wrapper around an off-policy or on-policy algorithm, with the
curiosity forward pass, the intrinsic reward and the ICM update on the device.

Reference: tianshou/algorithm/modelbased/icm.py (ICMTrainingStats :22-35, _ICMMixin :38-109, ICMOffPolicyWrapper :112-178,
ICMOnPolicyWrapper :181-248), utils/net/discrete.py:377-428 (IntrinsicCuriosityModule), algorithm_base.py:99-140 and :954-1060
(the stats wrapper and the wrapper bases), :801-802 (the n-step return reads ``buffer.rew``, not ``batch.rew``).

Per ``update()``, around the wrapped algorithm's own update:
  preprocess : one feature-net pass over ``[obs ; obs_next]`` (2B rows: dense rows, or the uint8 frame slots of both halves
               for the first convolution's gather) -> ``ts_icm_inputs`` -> forward and inverse model GEMM chains -> ``ts_icm_rows``
               (per-row losses, their gradients, the intrinsic reward ``rew + fp32(mse * reward_scale)`` into a new float64
               tensor, the three losses).  Then the wrapped algorithm's preprocess.
  update     : the wrapped update, then the two models' backward passes (input gradients over phi1 for the forward model, over
               [phi1 | phi2] for the inverse) -> ``ts_icm_feature_grad`` -> one backward of the feature net over the 2B rows ->
               one Adam step over the ICM's flat group -> one host read of the three losses.
  postprocess: the wrapped algorithm's (a prioritised buffer's priorities), then the original reward back on the batch.

Off-policy the reward with the curiosity term is set on the batch but never read: the wrapped n-step return reads the buffer's
rewards, as the reference's does, so the wrapped update is the unwrapped one and only the ICM learns.  On-policy it is the reward
GAE reads, also in every recomputation of PPO's advantages.  Only the wrapper's schedulers step (the ICM optimiser's); a
scheduler of the wrapped algorithm does not advance while it is wrapped, as in the reference.
"""
from __future__ import annotations

from typing import Any

import numpy as np
import torch
from torch import nn

from ... import ops
from ..._cabi import call, ptr, stream_ptr
from ...data import Batch, ReplayBuffer
from ...utils.net.discrete import IntrinsicCuriosityModule
from ..base import (Algorithm, OffPolicyAlgorithm, OffPolicyWrapperAlgorithm, OnPolicyAlgorithm, OnPolicyWrapperAlgorithm,
                    TrainingStats, TrainingStatsWrapper)
from ..flat_params import DeviceScratch, FlatGroup, UnsupportedModelError, bind_optimizer
from ..netgraph import ACT_NONE, FusedStack, _out_shape, compile_sequential, layer_params, module_layers
from ..obs_source import DeviceObsSource, device_obs_source
from ..optim import OptimizerFactory
from ..twin_critic import cuda_device_of


class ICMTrainingStats(TrainingStatsWrapper):
    def __init__(self, wrapped_stats: TrainingStats, *, icm_loss: float, icm_forward_loss: float, icm_inverse_loss: float) -> None:
        self.icm_loss = icm_loss
        self.icm_forward_loss = icm_forward_loss
        self.icm_inverse_loss = icm_inverse_loss
        super().__init__(wrapped_stats)


def _off_policy_supported() -> tuple[type, ...]:
    from ..modelfree.c51 import C51
    from ..modelfree.discrete_sac import DiscreteSAC
    from ..modelfree.dqn import DQN
    from ..modelfree.fqf import FQF
    from ..modelfree.iqn import IQN
    from ..modelfree.qrdqn import QRDQN
    return (DQN, QRDQN, C51, IQN, FQF, DiscreteSAC)       # RainbowDQN is a C51


def _chain(mods: list[nn.Module], shape: tuple[int, ...], what: str) -> list:
    try:
        return compile_sequential(mods, shape)
    except UnsupportedModelError as e:
        raise UnsupportedModelError(f"ICM {what}: {e}") from e


def _model_chain(mlp: nn.Module, in_dim: int, out_dim: int, what: str) -> list:
    try:
        mods = module_layers(mlp)
    except UnsupportedModelError as e:
        raise UnsupportedModelError(f"ICM {what}: {e}") from e
    layers = _chain(mods, (in_dim,), what)
    if not layers or layers[-1].kind != "linear" or layers[-1].act != ACT_NONE or layers[-1].out_dim != out_dim:
        raise UnsupportedModelError(f"ICM {what}: must end in a linear layer of {out_dim} outputs without activation")
    return layers


class _ICMMixin:
    """The ICM on the device (icm.py:38-109).  The wrapper base sets ``wrapped_algorithm``; ``_icm_init`` reads the module's three
    chains into one flat group bound to the ICM optimiser."""

    wrapped_algorithm: Algorithm
    _on_policy: bool

    def _icm_init(self, model: IntrinsicCuriosityModule, optim: OptimizerFactory, lr_scale: float, reward_scale: float,
                  forward_loss_weight: float) -> None:
        w = self.wrapped_algorithm
        space = w.policy.action_space
        if not hasattr(space, "n") or hasattr(space, "nvec"):
            raise UnsupportedModelError(f"ICM needs a Discrete action space, got {type(space).__name__}")
        n = int(space.n)
        if self._on_policy:
            from ..modelfree.ppo import A2C, PPO
            if type(w) not in (PPO, A2C):
                raise UnsupportedModelError(f"ICMOnPolicyWrapper runs on the device around PPO and A2C, not {type(w).__name__}")
            if not w._spec.categorical:
                raise UnsupportedModelError("ICMOnPolicyWrapper needs a categorical actor")
            if w._ranks()[1] > 1:
                raise UnsupportedModelError("ICM does not all-reduce its gradient: a data-parallel update over more than one rank "
                                            "is not supported")
            dev, in_shape = w.device, None
        else:
            if not isinstance(w, _off_policy_supported()):
                raise UnsupportedModelError(f"ICMOffPolicyWrapper runs on the device around DQN, QR-DQN, C51, Rainbow, IQN, FQF "
                                            f"and DiscreteSAC, not {type(w).__name__}")
            if getattr(w, "_seq", False):
                raise UnsupportedModelError("ICM does not read the sequences of a Recurrent Q-network (DRQN)")
            dev, in_shape = w._dev, tuple(w._in_shape)
        if cuda_device_of(model) != dev:
            raise UnsupportedModelError(f"the ICM module lives on {cuda_device_of(model)}, the wrapped algorithm on {dev}")
        F, A = int(model.feature_dim), int(model.action_dim)
        if A != n:
            raise UnsupportedModelError(f"the ICM module has action_dim {A} for {n} actions")
        fnet = model.feature_net
        try:
            fmods = module_layers(fnet)
        except UnsupportedModelError as e:
            raise UnsupportedModelError(f"ICM feature net: {e}") from e
        first = next((m for m in fmods if isinstance(m, (nn.Linear, nn.Conv2d))), None)
        if hasattr(fnet, "input_shape"):
            shape = tuple(fnet.input_shape)
        elif isinstance(first, nn.Linear):
            shape = (int(first.in_features),)
        elif isinstance(first, nn.Conv2d) and in_shape is not None and len(in_shape) == 3:
            shape = in_shape        # DQNet(...).net: the wrapped network's observation shape
        else:
            raise UnsupportedModelError("ICM feature net: cannot infer its input shape (an MLP, or a convolutional net around a "
                                        "wrapped algorithm that reads image observations)")
        feat = _chain(fmods, shape, "feature net")
        if _out_shape(feat, shape) != (F,):
            raise UnsupportedModelError(f"ICM feature net: output {_out_shape(feat, shape)}, feature_dim {F}")
        fwd = _model_chain(model.forward_model, F + A, F, "forward model")
        inv = _model_chain(model.inverse_model, 2 * F, A, "inverse model")
        params = list(model.parameters())
        if {id(p) for p in params} != {id(p) for p in layer_params(feat + fwd + inv)}:
            raise UnsupportedModelError("ICM: the module holds parameters outside its three layer chains")
        self.model = model
        self.optim = self._create_optimizer(model, optim)
        self.lr_scale, self.reward_scale, self.forward_loss_weight = lr_scale, reward_scale, forward_loss_weight
        self._icm_dev, self._icm_shape, self._icm_F, self._icm_A = dev, shape, F, A
        self._icm_group = FlatGroup(params, dev)
        bind_optimizer(self.optim, self._icm_group)
        self._icm_feat = FusedStack(feat, self._icm_group, "icm_feature")
        self._icm_fwd = FusedStack(fwd, self._icm_group, "icm_forward")
        self._icm_inv = FusedStack(inv, self._icm_group, "icm_inverse")
        # the feature net's output activation: a Flatten's backward masks its producer, a Linear's is folded in by the combine
        self._icm_out_act = feat[-1].act if feat[-1].kind == "linear" else ACT_NONE
        self._icm_scratch = DeviceScratch(dev)
        self._icm_buf = self._icm_scratch.tensor
        self._icm_state: dict[str, Any] | None = None

    # ------------------------------------------------------------------ inputs
    def _icm_off_policy_input(self, buffer: ReplayBuffer, indices: np.ndarray) -> tuple[torch.Tensor | None, tuple | None, int]:
        """The feature net's 2B input rows from the buffer's raw observations (denominator 1: the ICM's feature net reads them
        as stored, whatever the wrapped network divides by)."""
        srcs: list[DeviceObsSource] = [device_obs_source(buffer, indices, key, self._icm_shape, 1.0, self._icm_dev, self._icm_buf)
                                       for key in ("obs", "obs_next")]
        B = srcs[0].rows
        if srcs[0].frames is not None:
            f0, s0, _ = srcs[0].frames
            f1, s1, _ = srcs[1].frames
            if f0.data_ptr() != f1.data_ptr():
                raise UnsupportedModelError("ICM: image observations need obs_next read from the obs frames (ignore_obs_next)")
            sidx = self._icm_buf("sidx2", (2 * B, s0.shape[1]), torch.int64)
            sidx[:B].copy_(s0)
            sidx[B:].copy_(s1)
            return None, (f0, sidx, 1.0), B
        x = self._icm_buf("x2", (2 * B, srcs[0].x.shape[1]))
        x[:B].copy_(srcs[0].x)
        x[B:].copy_(srcs[1].x)
        return x, None, B

    def _icm_on_policy_input(self, batch: Batch, buffer: ReplayBuffer) -> tuple[torch.Tensor, int]:
        act = np.asarray(buffer.act)[: buffer.maxsize]
        if act.size and (act.min() < 0 or act.max() >= self._icm_A):
            raise ValueError(f"the buffer holds actions in [{act.min()}, {act.max()}], the ICM has {self._icm_A} actions")
        B = batch.obs.shape[0]
        D = batch.obs.reshape(B, -1).shape[1]
        if (D,) != self._icm_shape:
            raise UnsupportedModelError(f"ICM feature net reads {self._icm_shape}, the rollout holds rows of {D} features")
        x = self._icm_buf("x2", (2 * B, D))
        x[:B].copy_(batch.obs.reshape(B, D))
        x[B:].copy_(batch.obs_next.reshape(B, D))
        return x, B

    # ------------------------------------------------------------------ forward (preprocess)
    def _icm_forward(self, x: torch.Tensor | None, frames: tuple | None, B: int, act: torch.Tensor, act_f32: bool,
                     rew_in: torch.Tensor) -> torch.Tensor:
        """phi, the two models' outputs, the per-row losses and gradients; returns the reward with the curiosity term."""
        F, A, st, buf = self._icm_F, self._icm_A, stream_ptr(self._icm_dev), self._icm_buf
        fa = self._icm_feat.forward(x, 2 * B, "icm", frames=frames)
        phi = fa[-1]
        fwd_in, inv_in = buf("fwd_in", (B, F + A)), buf("inv_in", (B, 2 * F))
        call("ts_icm_inputs", ptr(phi), ptr(act), int(act_f32), B, F, A, ptr(fwd_in), ptr(inv_in), st)
        aa = self._icm_fwd.forward(fwd_in, B, "icm")
        ia = self._icm_inv.forward(inv_in, B, "icm")
        dphi, dfh, dah = buf("dphi", (2 * B, F)), buf("dphi2_hat", (B, F)), buf("dact_hat", (B, A))
        rows, losses = buf("rows", (2, B)), buf("losses", 3)
        rew = buf("rew", B, torch.float64)
        rew_in = rew_in.reshape(-1)
        if rew_in.dtype != torch.float64:
            rew_in = rew_in.to(torch.float64)
        call("ts_icm_rows", ptr(phi), ptr(aa[-1]), ptr(ia[-1]), ptr(act), int(act_f32), B, F, A, float(self.lr_scale),
             float(self.forward_loss_weight), ptr(rew_in), float(self.reward_scale), ptr(rew), ptr(dphi), ptr(dfh), ptr(dah),
             ptr(rows), ptr(losses), st)
        self._icm_state = dict(B=B, fa=fa, aa=aa, ia=ia, dphi=dphi, dfh=dfh, dah=dah, losses=losses, rew=rew)
        return rew

    # ------------------------------------------------------------------ update
    def _icm_update(self, original_stats: TrainingStats) -> ICMTrainingStats:
        s = self._icm_state
        assert s is not None, "the ICM update runs after its preprocess"
        B, F = s["B"], self._icm_F
        st = stream_ptr(self._icm_dev)
        dfwd = self._icm_fwd.backward(s["aa"], s["dfh"], B, "icm", input_grad=True, input_cols=(0, F))
        dinv = self._icm_inv.backward(s["ia"], s["dah"], B, "icm", input_grad=True)
        phi = s["fa"][-1]
        call("ts_icm_feature_grad", ptr(s["dphi"]), ptr(dinv), ptr(dfwd), ptr(phi), int(self._icm_out_act), B, F, st)
        self._icm_feat.backward(s["fa"], s["dphi"], 2 * B, "icm", dy_preact=self._icm_out_act != ACT_NONE)
        self._icm_group.adam_step(self.optim._optim, self.optim._max_grad_norm)
        loss, fwd, inv = (float(v) for v in s["losses"].cpu().tolist())       # the only host read of the ICM
        self._icm_state = None
        return ICMTrainingStats(original_stats, icm_loss=loss, icm_forward_loss=fwd, icm_inverse_loss=inv)

    @property
    def icm_reward(self) -> torch.Tensor | None:
        """The reward with the curiosity term of the last preprocess (float64 device rows), kept until the next one."""
        return self._icm_scratch.get("rew_last")


class ICMOffPolicyWrapper(_ICMMixin, OffPolicyWrapperAlgorithm):
    """ICM around an off-policy algorithm (icm.py:112-178)."""

    _on_policy = False

    def __init__(self, *, wrapped_algorithm: OffPolicyAlgorithm, model: IntrinsicCuriosityModule, optim: OptimizerFactory,
                 lr_scale: float, reward_scale: float, forward_loss_weight: float) -> None:
        OffPolicyWrapperAlgorithm.__init__(self, wrapped_algorithm=wrapped_algorithm)
        self._icm_init(model, optim, lr_scale, reward_scale, forward_loss_weight)

    def _preprocess_batch(self, batch: Batch, buffer: ReplayBuffer, indices: Any) -> Batch:
        x, frames, B = self._icm_off_policy_input(buffer, indices)
        idx = ops._idx(np.asarray(indices), self._icm_dev)
        rew_in = ops.gather_rows(buffer.device_array("rew").contiguous(), idx)
        rew = self._icm_forward(x, frames, B, batch.act, False, rew_in)
        self._icm_scratch["rew_last"] = rew
        self._icm_orig_rew = batch.__dict__.get("rew")
        batch.__dict__["rew"] = rew         # never read: the n-step return reads the buffer's rewards (quirk of the reference)
        return super()._preprocess_batch(batch, buffer, indices)

    def _postprocess_batch(self, batch: Batch, buffer: ReplayBuffer, indices: Any) -> None:
        super()._postprocess_batch(batch, buffer, indices)
        if self._icm_orig_rew is None:
            batch.__dict__.pop("rew", None)
        else:
            batch.__dict__["rew"] = self._icm_orig_rew
        self._icm_orig_rew = None

    def _wrapper_update_with_batch(self, batch: Batch, original_stats: TrainingStats) -> ICMTrainingStats:
        return self._icm_update(original_stats)


class ICMOnPolicyWrapper(_ICMMixin, OnPolicyWrapperAlgorithm):
    """ICM around an on-policy algorithm (icm.py:181-248).  The reward GAE reads carries the curiosity term; it is a new tensor,
    never the buffer's device reward column the rollout batch may hold."""

    _on_policy = True

    def __init__(self, *, wrapped_algorithm: OnPolicyAlgorithm, model: IntrinsicCuriosityModule, optim: OptimizerFactory,
                 lr_scale: float, reward_scale: float, forward_loss_weight: float) -> None:
        OnPolicyWrapperAlgorithm.__init__(self, wrapped_algorithm=wrapped_algorithm)
        self._icm_init(model, optim, lr_scale, reward_scale, forward_loss_weight)

    def _preprocess_batch(self, batch: Batch, buffer: ReplayBuffer, indices: Any) -> Batch:
        x, B = self._icm_on_policy_input(batch, buffer)
        act = batch.act.reshape(-1)
        if act.dtype != torch.float32 or not act.is_contiguous():
            act = act.to(torch.float32).contiguous()
        rew = self._icm_forward(x, None, B, act, True, batch.rew)
        self._icm_scratch["rew_last"] = rew
        self._icm_orig_rew = batch.rew
        batch.__dict__["rew"] = rew
        return super()._preprocess_batch(batch, buffer, indices)

    def _postprocess_batch(self, batch: Batch, buffer: ReplayBuffer, indices: Any) -> None:
        super()._postprocess_batch(batch, buffer, indices)
        batch.__dict__["rew"] = self._icm_orig_rew
        self._icm_orig_rew = None

    def _wrapper_update_with_batch(self, batch: Batch, batch_size: int | None, repeat: int,
                                   original_stats: TrainingStats) -> ICMTrainingStats:
        return self._icm_update(original_stats)
