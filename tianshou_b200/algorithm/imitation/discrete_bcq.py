"""Discrete batch-constrained Q-learning (arXiv:1910.01708) with the whole ``update()`` on the device.

Reference: tianshou/algorithm/imitation/discrete_bcq.py (DiscreteBCQPolicy :37-127, DiscreteBCQ :130-261),
utils/lagged_network.py:81-87 (the full lagged copy), examples/offline/atari_bcq.py:104-122 and
test/offline/test_discrete_bcq.py:73-86 (the Q head and the imitator head on ONE preprocess network).

Per ``update(buffer, sample_size)``:
  host : index draw from the buffer's RNG streams, the range check of the drawn actions, one D2H of the four loss scalars.
  GPU  : observation source of s_{t+n} -> online trunk + both heads, lagged trunk + Q head -> ``ts_discrete_bcq_target`` ->
         value mask + ``ts_nstep_return``; observation source of s -> trunk + both heads -> ``ts_discrete_bcq_rows`` (the three
         losses, d loss / d q, d loss / d logits) -> both heads' backward GEMMs into one trunk gradient -> trunk backward ->
         one Adam step over the whole flat group; the lagged copy is one device memcpy.
Every Linear / Conv2d layer's forward, input gradient and weight gradient is one wgmma GEMM launch (csrc/net_gemm.cu); the two
heads on one trunk are shared_trunk.py's.
"""
from __future__ import annotations

import math
from copy import deepcopy
from dataclasses import dataclass
from typing import Any

import numpy as np
import torch
from torch import nn

from ..._cabi import call, ptr, stream_ptr
from ...data import Batch, ReplayBuffer
from ..base import OfflineAlgorithm
from ..flat_params import DeviceScratch, FlatGroup, UnsupportedModelError, bind_optimizer
from ..modelfree.dqn import DiscreteQLearningPolicy, SimpleLossTrainingStats
from ..obs_source import DeviceObsSource, device_obs_source
from ..optim import OptimizerFactory
from ..shared_trunk import TwoHeadNetwork, two_head_parameters
from ..twin_critic import _EvalModeModule, cuda_device_of, sample_discrete

INF = torch.finfo(torch.float32).max


@dataclass(kw_only=True)
class DiscreteBCQTrainingStats(SimpleLossTrainingStats):
    q_loss: float
    i_loss: float
    reg_loss: float


def check_actions_in_range(buffer: ReplayBuffer, indices: np.ndarray, n_actions: int) -> None:
    """The loss kernels index a row of ``n_actions`` values with the stored action: refuse anything else on the host."""
    act = np.asarray(buffer.act)[indices]
    if act.size and (act.min() < 0 or act.max() >= n_actions):
        raise ValueError(f"the buffer holds actions in [{act.min()}, {act.max()}], the networks have {n_actions} outputs")


class DiscreteBCQPolicy(DiscreteQLearningPolicy):
    """The arg-max of Q over the actions the imitator does not call unlikely (discrete_bcq.py:37-127).  ``forward`` is the
    torch-module path the Collector runs."""

    def __init__(self, *, model: nn.Module, imitator: nn.Module, target_update_freq: int = 8000,
                 unlikely_action_threshold: float = 0.3, action_space: Any, observation_space: Any | None = None,
                 eps_inference: float = 0.0) -> None:
        super().__init__(model=model, action_space=action_space, observation_space=observation_space, eps_training=0.0,
                         eps_inference=eps_inference)       # offline: no training data is collected
        self.imitator = imitator
        assert target_update_freq > 0, f"BCQ needs target_update_freq>0 but got: {target_update_freq}."
        assert 0.0 <= unlikely_action_threshold < 1.0, (
            f"unlikely_action_threshold should be in [0, 1) but got: {unlikely_action_threshold}")
        self._log_tau = math.log(unlikely_action_threshold) if unlikely_action_threshold > 0 else -np.inf

    def forward(self, batch: Batch, state: Any = None, model: nn.Module | None = None) -> Batch:
        if model is None:
            model = self.model
        info = batch.get("info")
        q_value, state = model(batch.obs, state=state, info=info)
        imitation_logits, _ = self.imitator(batch.obs, state=state, info=info)
        ratio = imitation_logits - imitation_logits.max(dim=-1, keepdim=True).values
        mask = (ratio < self._log_tau).float()
        act = (q_value - INF * mask).argmax(dim=-1)
        return Batch(act=act, state=state, q_value=q_value, imitation_logits=imitation_logits, logits=imitation_logits)


class DiscreteBCQ(OfflineAlgorithm):
    """Discrete BCQ, reference API and semantics (discrete_bcq.py:130-261).

    ``policy.model`` and ``policy.imitator`` are ``DiscreteActor(softmax_output=False)`` / ``DiscreteCritic``-shaped networks
    (a preprocess net and a ``last`` MLP) over the same preprocess network, or over one each.  As in the reference the lagged
    copy is refreshed when ``_iter % target_update_freq == 0`` BEFORE the step, the loss takes no importance weight, and a
    prioritised buffer's ``batch.weight`` passes through the update untouched.
    """

    def __init__(self, *, policy: DiscreteBCQPolicy, optim: OptimizerFactory, gamma: float = 0.99, n_step_return_horizon: int = 1,
                 target_update_freq: int = 8000, imitation_logits_penalty: float = 1e-2) -> None:
        super().__init__(policy=policy)
        assert 0.0 <= gamma <= 1.0, f"discount factor should be in [0, 1] but got: {gamma}"
        assert n_step_return_horizon > 0, f"n_step_return_horizon should be greater than 0 but got: {n_step_return_horizon}"
        # the reference reads self.model_old and divides by the frequency unconditionally: 0 fails in its first update
        assert target_update_freq > 0, f"BCQ needs target_update_freq>0 but got: {target_update_freq}."
        self.gamma = gamma
        self.n_step = n_step_return_horizon
        self._target = True
        self.freq = target_update_freq
        self._iter = 0
        self._weight_reg = imitation_logits_penalty
        model, imitator = policy.model, policy.imitator
        for name, net in (("model", model), ("imitator", imitator)):
            if getattr(net, "softmax_output", False):
                raise UnsupportedModelError(f"{name}: DiscreteActor(softmax_output=True) is not supported: the update reads the "
                                            "output as Q-values / logits; build it with softmax_output=False")
        dev = self._dev = cuda_device_of(model, imitator)
        self._group = FlatGroup(two_head_parameters(model, imitator), dev)
        self._net = TwoHeadNetwork(model, imitator, self._group, roles=("model", "imitator"))
        self._in_shape, self._in_scale = self._net.in_shape, self._net.in_scale
        self.n_actions = int(policy.action_space.n)
        for name, n in zip(("model", "imitator"), self._net.n_out):
            if n != self.n_actions:
                raise UnsupportedModelError(f"{name} has {n} outputs for {self.n_actions} actions")
        self.optim = self._create_optimizer(policy, optim)
        bind_optimizer(self.optim, self._group)
        # the model's parameters lead the flat order, so the lagged model's flat buffer is a prefix of the same layout
        self.model_old = _EvalModeModule(deepcopy(model))
        self._g_old = FlatGroup(list(self.model_old.module.parameters()), dev)
        self._scratch = DeviceScratch(dev)
        self._buf = self._scratch.tensor

    # ------------------------------------------------------------------ sampling / target
    def _obs_source(self, buffer: ReplayBuffer, indices: np.ndarray | torch.Tensor, key: str = "obs") -> DeviceObsSource:
        return device_obs_source(buffer, indices, key, self._in_shape, self._in_scale, self._dev, self._buf)

    def _sample(self, buffer: ReplayBuffer, sample_size: int | None) -> tuple[Batch, Any]:
        batch, indices = sample_discrete(buffer, sample_size, self._obs_source, self._dev)
        check_actions_in_range(buffer, indices, self.n_actions)
        return batch, indices

    def _target_q(self, buffer: ReplayBuffer, indices: np.ndarray) -> torch.Tensor:
        """Q_old(s', argmax_a Q(s', a) over the actions the imitator keeps)   (discrete_bcq.py:228-234)."""
        src = self._obs_source(buffer, indices, "obs_next")
        on = self._net.forward(src, "tq")
        self._g_old.ensure_adopted()
        old = self._net.forward(src, "tq_old", params=self._g_old.flat, heads=(True, False))
        out = self._buf("tq_out", src.rows)
        call("ts_discrete_bcq_target", ptr(on.a[-1]), ptr(on.b[-1]), ptr(old.a[-1]), float(self.policy._log_tau), src.rows,
             self.n_actions, ptr(out), None, stream_ptr(self._dev))
        return out

    def _preprocess_batch(self, batch: Batch, buffer: ReplayBuffer, indices: np.ndarray) -> Batch:
        return self.compute_nstep_return(batch=batch, buffer=buffer, indices=indices, target_q_fn=self._target_q,
                                         gamma=self.gamma, n_step=self.n_step)

    # ------------------------------------------------------------------ update
    def _update_lagged_network_weights(self) -> None:
        self._group.ensure_adopted()
        self._g_old.ensure_adopted()
        self._g_old.flat.copy_(self._group.flat[: self._g_old.n])         # full copy (lagged_network.py:81-87)

    def _update_with_batch(self, batch: Batch) -> DiscreteBCQTrainingStats:
        if self._iter % self.freq == 0:
            self._update_lagged_network_weights()
        self._iter += 1
        src = batch.obs
        B, A = src.rows, self.n_actions
        acts = self._net.forward(src, "up")
        returns = batch.returns.reshape(-1).to(self._dev, torch.float32).contiguous()
        dq, dlogits = self._buf("dq", (B, A)), self._buf("dlogits", (B, A))
        rows, losses = self._buf("loss_rows", (3, B)), self._buf("losses", 4)
        call("ts_discrete_bcq_rows", ptr(acts.a[-1]), ptr(acts.b[-1]), ptr(batch.act), ptr(returns), B, A, float(self._weight_reg),
             ptr(dq), ptr(dlogits), ptr(rows), ptr(losses), stream_ptr(self._dev))
        self._net.backward(acts, dq, dlogits, "up")
        self._group.adam_step(self.optim._optim, self.optim._max_grad_norm)
        l = losses.cpu().numpy()                # the only host read of the losses
        return DiscreteBCQTrainingStats(loss=float(l[0]), q_loss=float(l[1]), i_loss=float(l[2]), reg_loss=float(l[3]))
