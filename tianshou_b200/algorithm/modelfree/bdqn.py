"""BDQN (branching dueling Q-network, arXiv:1711.08946) with ``update()`` on the device.

Reference: tianshou/algorithm/modelfree/bdqn.py (BDQNPolicy :29-106, BDQN :109-224), utils/net/common.py:553-674 (BranchingNet),
modelfree/dqn.py:170-283 (the lagged network refreshed when ``_iter % target_update_freq == 0``).

Per ``update(buffer, sample_size)``:
  host : index draw (the reference's streams), the action rows of the sample (width and range checked), one D2H of the loss
         (+ the signed td sums for a prioritised buffer's priority update, as in the reference).
  GPU  : rows of s' -> the trunk (``ts_net_gemm``), the value head, and every branch of a layer in ONE batched launch
         (``ts_net_gemm_batched``, the trunk output shared at stride 0) for the online network (when double, or without a
         lagged network) and the lagged one -> ``ts_bdqn_target``; the same on s -> ``ts_bdqn_rows`` (the dueling combine, the
         loss over each branch's chosen action, the gradients of the combine) -> the branches' and the value head's backward,
         their trunk-input gradients summed in a fixed order -> the trunk's backward -> one Adam step over the whole network;
         the lagged refresh is one device copy.
"""
from __future__ import annotations

from copy import deepcopy
from typing import Any

import numpy as np
import torch
from torch import nn

from ... import ops
from ..._cabi import call, ptr, stream_ptr, to_device
from ...data import Batch, ReplayBuffer, to_numpy
from ...utils.net.common import BranchingNet
from ..base import OffPolicyAlgorithm
from ..discrete_q import DiscreteQCore, lagged_group, sample_discrete
from ..flat_params import FlatGroup, UnsupportedModelError, bind_optimizer
from ..netgraph import ACT_NONE, FusedStack, _Layer, compile_branches, compile_sequential, layer_params, module_layers
from ..optim import OptimizerFactory
from ..twin_critic import _EvalModeModule, cuda_device_of, pop_batch_weight
from .dqn import DiscreteQLearningPolicy, SimpleLossTrainingStats

# The reference's ``_preprocess_batch`` (bdqn.py:177-184) calls ``_compute_return`` without the algorithm's ``gamma``, so that
# method's default discounts every target whatever ``gamma`` was given; the update reproduces it.
TARGET_GAMMA = 0.99


class BDQNPolicy(DiscreteQLearningPolicy):
    """argmax-Q per branch with epsilon-greedy exploration (bdqn.py:29-106): ``act`` is ``[B, num_branches]``."""

    def __init__(self, *, model: BranchingNet, action_space: Any, observation_space: Any | None = None,
                 eps_training: float = 0.0, eps_inference: float = 0.0) -> None:
        super().__init__(model=model, action_space=action_space, observation_space=observation_space, eps_training=eps_training,
                         eps_inference=eps_inference)

    def forward(self, batch: Batch, state: Any = None, model: nn.Module | None = None) -> Batch:
        if model is None:
            model = self.model
        obs = batch.obs
        obs_next_BO = obs.obs if hasattr(obs, "obs") else obs      # the reference's unwrap (bdqn.py:75-76)
        action_values_BA, hidden_BH = model(obs_next_BO, state=state, info=batch.info)
        return Batch(logits=action_values_BA, act=to_numpy(action_values_BA.argmax(dim=-1)), state=hidden_BH)

    def add_exploration_noise(self, act: Any, batch: Any) -> Any:
        eps = self.eps_training if self.is_within_training_step else self.eps_inference
        if np.isclose(eps, 0.0):
            return act
        if isinstance(act, np.ndarray):
            bsz = len(act)
            rand_mask = np.random.rand(bsz) < eps
            rand_act = np.random.randint(low=0, high=self.model.action_per_branch, size=(bsz, act.shape[-1]))
            if hasattr(batch.obs, "mask"):
                rand_act += batch.obs.mask
            act[rand_mask] = rand_act[rand_mask]
            return act
        raise NotImplementedError(f"Currently only numpy arrays are supported, got {type(act)=}.")


def describe_branching_net(model: Any) -> tuple[list[_Layer], list[_Layer], list[_Layer]]:
    """A ``BranchingNet`` as three chains on one flat group: the trunk, the value head (one output) and the branches as one
    ensemble chain of ``num_branches`` members.  Norm layers, activations other than ReLU / Tanh and branches of different shapes
    are refused."""
    if not all(hasattr(model, k) for k in ("common", "value", "branches", "num_branches", "action_per_branch")):
        raise UnsupportedModelError(f"BDQN needs a BranchingNet, got {type(model).__name__}")
    try:
        trunk_mods = module_layers(model.common)
        first = trunk_mods[0] if trunk_mods else None
        if not isinstance(first, nn.Linear):
            raise UnsupportedModelError("the trunk must start with a Linear layer")
        common = compile_sequential(trunk_mods, (int(first.in_features),))
        H = common[-1].out_dim
        value = compile_sequential(module_layers(model.value), (H,))
        branches = compile_branches(model.branches, H)
    except UnsupportedModelError as e:
        raise UnsupportedModelError(f"BDQN BranchingNet: {e}") from e
    if any(L.kind != "linear" for L in common + value):
        raise UnsupportedModelError("BDQN BranchingNet: the trunk and the value head must be MLPs of Linear layers")
    if value[-1].out_dim != 1 or value[-1].act != ACT_NONE:
        raise UnsupportedModelError("BDQN BranchingNet: the value head must end in one linear output")
    if branches[-1].out_dim != model.action_per_branch or branches[-1].act != ACT_NONE:
        raise UnsupportedModelError(f"BDQN BranchingNet: the branches must end in {model.action_per_branch} linear outputs")
    if len(model.branches) != model.num_branches:
        raise UnsupportedModelError(f"BDQN BranchingNet: {len(model.branches)} branches, num_branches={model.num_branches}")
    return common, value, branches


class BDQN(DiscreteQCore, OffPolicyAlgorithm):
    """BDQN, reference API (bdqn.py:109-224).

    The update reproduces what ``BDQN._update_with_batch`` computes:

    * the target is ``r + 0.99 * mean_k Q'_k(s', a*_k) * (1 - end)`` (``TARGET_GAMMA``: the reference's target ignores
      ``gamma``) with ``a*_k`` the per-branch arg-max of the online network (``is_double``) or of the lagged one, ``end`` the
      buffer's ``done`` (terminated or truncated) and True at every unfinished episode's last slot; 1-step only;
    * the loss is ``mean_b w_b mean_k (y_b - Q_k(s_b, a_bk))^2`` with one Adam step over the whole network, and ``batch.weight =
      sum_k (y_b - Q_k)`` (signed) feeds a prioritised buffer;
    * at B = 1 the reported loss also carries the reference's broadcast term, the population variance over branches of the
      per-branch targets; a prioritised buffer with more than one branch at B = 1 is refused (the reference fails in its priority
      update after stepping).
    """

    def __init__(self, *, policy: BDQNPolicy, optim: OptimizerFactory, gamma: float = 0.99, target_update_freq: int = 0,
                 is_double: bool = True) -> None:
        super().__init__(policy=policy)
        assert 0.0 <= gamma <= 1.0, f"discount factor should be in [0, 1] but got: {gamma}"
        self.gamma = gamma
        self.n_step = 1
        self.target_update_freq = target_update_freq
        self.is_double = is_double
        dev = cuda_device_of(policy.model)
        common, value, branches = describe_branching_net(policy.model)
        self.num_branches, self.action_per_branch = len(policy.model.branches), int(policy.model.action_per_branch)
        self._init_discrete(dev, (common[0].in_dim,), 1.0, self.action_per_branch)
        self._group = FlatGroup(layer_params(common) + layer_params(value) + layer_params(branches), dev)
        self._common = FusedStack(common, self._group, "common")
        self._value = FusedStack(value, self._group, "value")
        self._branches = FusedStack(branches, self._group, "branches")
        self.optim = self._create_optimizer(policy, optim)
        bind_optimizer(self.optim, self._group)
        self.model_old: _EvalModeModule | None = None
        self._g_old: FlatGroup | None = None
        if self.use_target_network:
            self.model_old = _EvalModeModule(deepcopy(policy.model))
            oc, ov, ob = describe_branching_net(self.model_old.module)
            self._g_old = lagged_group(self._group, layer_params(oc) + layer_params(ov) + layer_params(ob))

    @property
    def use_target_network(self) -> bool:
        return self.target_update_freq > 0

    # ------------------------------------------------------------------ rows
    def _sample(self, buffer: ReplayBuffer, sample_size: int | None) -> tuple[Batch, Any]:
        if self.num_branches > 1 and hasattr(buffer, "update_weight") and (sample_size if sample_size else len(buffer)) == 1:
            raise ValueError("BDQN with a prioritised buffer needs a batch of more than one row when num_branches > 1: the "
                             "reference's priority update fails at B = 1 (its td sums broadcast to num_branches values)")
        return sample_discrete(buffer, sample_size, self._obs_source, self._dev, self.n_actions, branches=self.num_branches)

    def _q_parts(self, x: torch.Tensor, rows: int, tag: str, target: bool = False
                 ) -> tuple[list[torch.Tensor], list[torch.Tensor], list[torch.Tensor]]:
        """Activation lists of the trunk, the value head ([rows, 1]) and the branches ([nb, rows, A]) on ``x``."""
        params = None
        if target:
            self._g_old.ensure_adopted()
            params = self._g_old.flat
        acts_c = self._common.forward(x, rows, tag, params=params)
        h = acts_c[-1]
        return acts_c, self._value.forward(h, rows, tag, params=params), self._branches.forward(h, rows, tag, params=params)

    # ------------------------------------------------------------------ target
    def _preprocess_batch(self, batch: Batch, buffer: ReplayBuffer, indices: np.ndarray) -> Batch:
        """The 1-step target of ``_compute_return`` (bdqn.py:144-175) into ``batch.returns`` [B]."""
        src = self._obs_source(buffer, indices, "obs_next")
        B = src.rows
        on = tg = None
        if self.is_double or not self.use_target_network:      # the online pass on s', once (the reference runs it twice)
            _, v, s = self._q_parts(src.x, B, "tq_on")
            on = (v[-1], s[-1])
        if self.use_target_network:
            _, v, s = self._q_parts(src.x, B, "tq_old", target=True)
            tg = (v[-1], s[-1])
        else:
            tg = on
        sel = on if self.is_double else tg
        rew = buffer.device_array("rew")
        if rew.dtype != torch.float64:
            rew = rew.to(torch.float64)
        end = ops.buffer_end_flags(buffer.device_meta())
        idx = to_device(np.asarray(indices, dtype=np.int64), self._dev)
        y = self._buf("y", B)
        y_branch = self._buf("y_branch", (1, self.num_branches)) if B == 1 and self.num_branches > 1 else None
        call("ts_bdqn_target", ptr(sel[0]), ptr(sel[1]), ptr(tg[0]), ptr(tg[1]), B, self.num_branches, self.action_per_branch,
             TARGET_GAMMA, ptr(rew), ptr(end), ptr(idx), ptr(y), ptr(y_branch),
             stream_ptr(self._dev))
        batch.returns = y
        batch.__dict__["returns_branch"] = y_branch
        return batch

    # ------------------------------------------------------------------ update
    def _update_with_batch(self, batch: Batch) -> SimpleLossTrainingStats:
        self._tick_lagged(self.target_update_freq)
        dev, st = self._dev, stream_ptr(self._dev)
        B, nb, A = batch.obs.rows, self.num_branches, self.action_per_branch
        weight = pop_batch_weight(batch, dev)
        y_branch = batch.__dict__.pop("returns_branch", None)
        acts_c, acts_v, acts_s = self._q_parts(batch.obs.x, B, "up")
        h = acts_c[-1]
        td, rows, td_sum = self._buf("td", (B, nb)), self._buf("loss_rows", B), self._buf("td_sum", B)
        ds, dv, loss = self._buf("ds", (nb, B, A)), self._buf("dv", (B, 1)), self._buf("loss", 1)
        call("ts_bdqn_rows", ptr(acts_v[-1]), ptr(acts_s[-1]), ptr(batch.act), ptr(batch.returns), ptr(weight),
             ptr(y_branch), B, nb, A, ptr(td), ptr(rows), ptr(td_sum), ptr(ds), ptr(dv), ptr(loss),
             st)
        # d loss / d trunk output = sum_k (branch k's input gradient), in branch order, + the value head's
        dh = self._buf("dh", tuple(h.shape))
        trunk_act = (self._common.layers[-1].act, h)
        self._branches.backward(acts_s, ds, B, "up", input_grad=True, input_act=trunk_act, dx_out=dh)
        self._value.backward(acts_v, dv, B, "up", input_grad=True, input_act=trunk_act, dx_out=dh, dx_accumulate=True)
        self._common.backward(acts_c, dh, B, "up", dy_preact=True)
        self._group.adam_step(self.optim._optim, self.optim._max_grad_norm)
        batch.weight = td_sum                   # prio-buffer: the signed sum over branches
        return SimpleLossTrainingStats(loss=float(loss.item()))
