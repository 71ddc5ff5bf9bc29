"""Deep Q-Network (double DQN, n-step, prioritised replay) with ``update()`` on the device
(SURVEY 8(f) ranks 2-3, BASELINE configs[2]).

Reference: tianshou/algorithm/modelfree/dqn.py (DiscreteQLearningPolicy :36-164, QLearningOffPolicyAlgorithm
:170-283, DQN :286-404), env/atari/atari_network.py:60-122 (DQNet), data/buffer/buffer_base.py:557-603 (frame
stacking), utils/lagged_network.py:83-103 (full target copy every ``target_update_freq`` iterations).

Per ``update(buffer, sample_size)``:
  host : index draw (uniform: numpy RandomState streams; prioritised: ``np.random.rand`` scalars, SURVEY A9/A10),
         one D2H of the loss scalar (+ the TD errors for the priority update, as in the reference).
  GPU  : frame-stack index chains (``ts_stack_prev_indices``) -> the first convolution's im2col reads the uint8 frames
         of the buffer's device mirror directly (no stacked observation is ever materialised) -> conv / linear layers
         as wgmma GEMMs (``ts_net_gemm``) for the online and the lagged network -> ``ts_dqn_target`` ->
         ``ts_nstep_return`` -> ``ts_dqn_loss`` -> backward GEMMs + col2im -> Adam; target copy = one device memcpy.
"""
from __future__ import annotations

from copy import deepcopy
from dataclasses import dataclass
from typing import Any

import numpy as np
import torch
from torch import nn

from ..._cabi import call, ptr, stream_ptr, to_device
from ...data import Batch, ReplayBuffer, to_numpy
from ..base import OffPolicyAlgorithm, Policy, TrainingStats
from ..flat_params import FlatGroup, UnsupportedModelError, bind_optimizer
from ..netgraph import ACT_NONE, FusedStack, compile_sequential, module_layers
from ..obs_source import DeviceObsSource, device_obs_source
from ..optim import OptimizerFactory


@dataclass(kw_only=True)
class SimpleLossTrainingStats(TrainingStats):
    loss: float


class DiscreteQLearningPolicy(Policy):
    """argmax-Q policy with epsilon-greedy exploration (dqn.py:36-164)."""

    def __init__(self, *, model: nn.Module, action_space: Any, observation_space: Any | None = None, eps_training: float = 0.0,
                 eps_inference: float = 0.0) -> None:
        super().__init__(action_space=action_space, observation_space=observation_space, action_scaling=False,
                         action_bound_method=None)
        self.model = model
        self.eps_training = eps_training
        self.eps_inference = eps_inference

    def set_eps_training(self, eps: float) -> None:
        self.eps_training = eps

    def set_eps_inference(self, eps: float) -> None:
        self.eps_inference = eps

    def forward(self, batch: Batch, state: Any = None, model: nn.Module | None = None) -> Batch:
        if model is None:
            model = self.model
        obs = batch.obs
        mask = getattr(obs, "mask", None)
        obs_arr = obs.obs if hasattr(obs, "obs") else obs
        action_values, hidden = model(obs_arr, state=state, info=batch.get("info"))
        q = self.compute_q_value(action_values, mask)
        return Batch(logits=action_values, act=to_numpy(q.argmax(dim=1)), state=hidden)

    def compute_q_value(self, logits: torch.Tensor, mask: np.ndarray | None) -> torch.Tensor:
        if mask is not None:
            min_value = logits.min() - logits.max() - 1.0
            logits = logits + torch.as_tensor(1 - mask, device=logits.device, dtype=logits.dtype) * min_value
        return logits

    def add_exploration_noise(self, act: Any, batch: Any) -> Any:
        eps = self.eps_training if self.is_within_training_step else self.eps_inference
        if np.isclose(eps, 0.0):
            return act
        if isinstance(act, np.ndarray):
            batch_size = len(act)
            rand_mask = np.random.rand(batch_size) < eps
            n = getattr(self.action_space, "n", None)
            q = np.random.rand(batch_size, int(n))
            if hasattr(batch.obs, "mask"):
                q += batch.obs.mask
            rand_act = q.argmax(axis=1)
            act[rand_mask] = rand_act[rand_mask]
            return act
        raise NotImplementedError(f"Currently only numpy array is supported for action, but got {type(act)}")


def describe_q_network(model: Any) -> tuple[Any, tuple[int, ...], float]:
    """(inner module with the layer chain, input shape, input denominator) of a Q-network: ``DQNet`` (optionally behind
    ``ScaledObsInputActionReprNet``) or an MLP ``Net`` on flat observations."""
    scale = 1.0          # the DENOMINATOR the observation is divided by before the network
    inner = model
    if hasattr(model, "denom") and hasattr(model, "module"):
        scale = float(model.denom)
        inner = model.module
    if hasattr(inner, "input_shape"):
        return inner, tuple(inner.input_shape), scale
    first = module_layers(inner)[0]
    if isinstance(first, nn.Linear):
        return inner, (int(first.in_features),), scale
    raise UnsupportedModelError(f"cannot infer the input shape of {type(inner).__name__}")


class DQN(OffPolicyAlgorithm):
    """DQN / double DQN with a periodically copied target network (dqn.py:286-404)."""

    def __init__(self, *, policy: DiscreteQLearningPolicy, optim: OptimizerFactory, gamma: float = 0.99,
                 n_step_return_horizon: int = 1, target_update_freq: int = 0, is_double: bool = True,
                 huber_loss_delta: float | None = None) -> None:
        super().__init__(policy=policy)
        assert 0.0 <= gamma <= 1.0, f"discount factor should be in [0, 1] but got: {gamma}"
        assert n_step_return_horizon > 0, f"n_step_return_horizon should be greater than 0 but got: {n_step_return_horizon}"
        self.gamma = gamma
        self.n_step = n_step_return_horizon
        self.target_update_freq = target_update_freq
        self.is_double = is_double
        self.huber_loss_delta = huber_loss_delta
        self._iter = 0
        dev = next(policy.model.parameters()).device
        if dev.type != "cuda":
            raise UnsupportedModelError(f"networks live on {dev}; tianshou_b200 has no CPU path -- move them to a CUDA device")
        self._dev = dev
        inner, self._in_shape, self._in_scale = describe_q_network(policy.model)
        layers = compile_sequential(module_layers(inner), self._in_shape)
        if layers[-1].kind != "linear" or layers[-1].act != ACT_NONE:
            raise UnsupportedModelError("Q-network must end in a linear layer over the actions")
        self.n_actions = layers[-1].out_dim
        params = [p for L in layers if L.weight is not None for p in (L.weight, L.bias)]
        self._group = FlatGroup(params, dev)
        self._net = FusedStack(layers, self._group, "q")
        self.optim = self._create_optimizer(policy, optim)
        bind_optimizer(self.optim, self._group)
        self.model_old = deepcopy(policy.model).eval() if self.use_target_network else None
        self._target_flat = self._group.flat.clone() if self.use_target_network else None
        self._scratch: dict[str, torch.Tensor] = {}

    @property
    def use_target_network(self) -> bool:
        return self.target_update_freq > 0

    def _buf(self, name: str, shape: tuple[int, ...] | int, dtype: torch.dtype = torch.float32) -> torch.Tensor:
        shape = (shape,) if isinstance(shape, int) else tuple(shape)
        t = self._scratch.get(name)
        if t is None or t.shape != shape or t.dtype != dtype:
            t = self._scratch[name] = torch.empty(shape, dtype=dtype, device=self._dev)
        return t

    # ------------------------------------------------------------------ observations -> first-layer input
    def _obs_source(self, buffer: ReplayBuffer, indices: np.ndarray | torch.Tensor, key: str = "obs") -> DeviceObsSource:
        """How the network reads ``buffer[indices].<key>`` without materialising it on the host (obs_source.py)."""
        return device_obs_source(buffer, indices, key, self._in_shape, self._in_scale, self._dev, self._buf)

    def _q_values(self, src: DeviceObsSource, tag: str, target: bool = False) -> tuple[list[torch.Tensor], torch.Tensor]:
        acts = self._net.forward(src.x, src.rows, tag, frames=src.frames, params=self._target_flat if target else None)
        return acts, acts[-1]

    # ------------------------------------------------------------------ target / n-step
    def _target_q(self, buffer: ReplayBuffer, indices: np.ndarray) -> torch.Tensor:
        """Q_old(s', argmax_a Q(s', a)) (double) or max_a Q_old(s', a)   (dqn.py:365-380)."""
        src = self._obs_source(buffer, indices, "obs_next")
        B = src.rows
        _, q_online = self._q_values(src, "tq_on")
        q_tgt = self._q_values(src, "tq_old", target=True)[1] if self.use_target_network else q_online
        out = self._buf("tq_out", B)
        call("ts_dqn_target", ptr(q_online), ptr(q_tgt), B, self.n_actions, int(self.is_double), ptr(out), stream_ptr(self._dev))
        return out

    def _preprocess_batch(self, batch: Batch, buffer: ReplayBuffer, indices: np.ndarray) -> Batch:
        return self.compute_nstep_return(batch=batch, buffer=buffer, indices=indices, target_q_fn=self._target_q,
                                         gamma=self.gamma, n_step=self.n_step)

    def _sample(self, buffer: ReplayBuffer, sample_size: int | None) -> tuple[Batch, Any]:
        indices = buffer.sample_indices(sample_size)
        batch = Batch()
        batch.__dict__["obs"] = self._obs_source(buffer, indices, "obs")
        act = np.asarray(buffer.act)[indices]
        batch.__dict__["act"] = to_device(np.ascontiguousarray(act.reshape(-1)).astype(np.int64), self._dev)
        if hasattr(buffer, "get_weight"):          # PrioritizedReplayBuffer.__getitem__ adds the IS weight (prio.py:104-106)
            w = buffer.get_weight(indices)
            batch.__dict__["weight"] = to_device(np.asarray(w / np.max(w) if buffer._weight_norm else w, dtype=np.float32), self._dev)
        batch.__dict__["info"] = Batch()
        return batch, indices

    # ------------------------------------------------------------------ update
    def _periodically_update_lagged_network_weights(self) -> None:
        if self.use_target_network and self._iter % self.target_update_freq == 0:
            self._group.ensure_adopted()
            self._target_flat.copy_(self._group.flat)                       # full copy (lagged_network.py:98-103)
            with torch.no_grad():
                for tp, sp in zip(self.model_old.parameters(), self.policy.model.parameters(), strict=True):
                    tp.copy_(sp)
        self._iter += 1

    def _update_with_batch(self, batch: Batch) -> SimpleLossTrainingStats:
        self._periodically_update_lagged_network_weights()
        st = stream_ptr(self._dev)
        src = batch.obs
        B = src.rows
        weight = batch.__dict__.pop("weight", None) if "weight" in batch.__dict__ else None
        if weight is not None and not isinstance(weight, torch.Tensor):
            weight = to_device(np.asarray(weight, dtype=np.float32), self._dev)
        acts, q = self._q_values(src, "up")
        returns = batch.returns.reshape(-1).to(self._dev, torch.float32).contiguous()
        td = self._buf("td", B)
        dq = self._buf("dq", (B, self.n_actions))
        rows = self._buf("loss_rows", B)
        loss = self._buf("loss", 1)
        call("ts_dqn_loss", ptr(q), ptr(batch.act), ptr(returns), ptr(weight), B, self.n_actions,
             float(self.huber_loss_delta or 0.0), ptr(td), ptr(dq), ptr(rows), st)
        call("ts_mean", ptr(rows), B, ptr(loss), st)
        batch.weight = td                      # prio-buffer
        self._net.backward(acts, dq, B, "up")
        self._group.adam_step(self.optim._optim, self.optim._max_grad_norm)
        return SimpleLossTrainingStats(loss=float(loss.item()))
