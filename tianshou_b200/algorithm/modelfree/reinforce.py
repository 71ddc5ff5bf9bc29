"""Stochastic actor policy (API of tianshou/algorithm/modelfree/reinforce.py:62-192)."""
from __future__ import annotations

import warnings
from collections.abc import Callable
from dataclasses import dataclass
from typing import Any, Literal

import numpy as np
import torch

from ...data import Batch, SequenceSummaryStats
from ..base import Policy, TrainingStats

TDistFn = Callable[..., torch.distributions.Distribution]


@dataclass(kw_only=True)
class LossSequenceTrainingStats(TrainingStats):
    """The loss of an update (reinforce.py:58-60); C51 fills it with a float, as the reference does."""

    loss: SequenceSummaryStats


class ProbabilisticActorPolicy(Policy):
    """actor(obs) -> dist_fn(...) -> sampled (or modal) action."""

    def __init__(self, *, actor: torch.nn.Module, dist_fn: TDistFn, deterministic_eval: bool = False,
                 action_space: Any, observation_space: Any | None = None, action_scaling: bool = True,
                 action_bound_method: Literal["clip", "tanh"] | None = "clip") -> None:
        super().__init__(action_space=action_space, observation_space=observation_space,
                         action_scaling=action_scaling, action_bound_method=action_bound_method)
        if action_scaling:
            try:
                if np.isclose(float(actor.max_action), 1.0) and not getattr(actor, "_unbounded", False):
                    warnings.warn(
                        "action_scaling and action_bound_method are only intended to deal with unbounded "
                        "model action space; consider unbounded=True for the actor.")
            except BaseException:
                pass
        self.actor = actor
        self.dist_fn = dist_fn
        self._eps = 1e-8
        self.deterministic_eval = deterministic_eval
        # set by the owning algorithm when the actor belongs to the fused kernel family: (FlatGroup, desc).
        # Inference under torch.no_grad() then runs ONE kernel (the update path's forward kernel) instead of the
        # module-by-module torch forward (SURVEY 8(f) rank 4: Collector._compute_action_policy_hidden).
        self._fused_inference: Any = None
        self.use_fused_inference = True

    def forward(self, batch: Batch, state: Any = None) -> Batch:
        """Batch(logits, act, state, dist); samples unless deterministic evaluation applies
        (reinforce.py:167-192)."""
        dist_input = self._fused_dist_input(batch.obs) if state is None else None
        hidden = None
        if dist_input is None:
            dist_input, hidden = self.actor(batch.obs, state=state, info=batch.get("info"))
        dist = self.dist_fn(dist_input)
        if self.deterministic_eval and not self.is_within_training_step:
            act = dist.mode
        else:
            act = dist.sample()
        return Batch(logits=dist_input, act=act, state=hidden, dist=dist)


# fused inference path of ProbabilisticActorPolicy (kept outside the class body for readability)
def _fused_dist_input(self: ProbabilisticActorPolicy, obs: Any) -> Any:
    """Actor output for ``obs`` from the fused forward kernel, or None when the torch modules must run (autograd
    needed, unsupported actor, non-array observations)."""
    if self._fused_inference is None or not self.use_fused_inference or torch.is_grad_enabled():
        return None
    if not isinstance(obs, np.ndarray | torch.Tensor):
        return None
    from ... import ops
    from ..._cabi import AC_CATEGORICAL
    flat, desc = self._fused_inference
    obs_t = torch.as_tensor(obs, device=flat.device, dtype=torch.float32)
    if obs_t.dim() < 2 or obs_t[0].numel() != desc.obs_dim:
        return None
    obs_t = obs_t.reshape(obs_t.shape[0], -1).contiguous()
    flat.ensure_adopted()
    n = obs_t.shape[0]
    categorical = bool(desc.flags & AC_CATEGORICAL)
    dummy = getattr(self, "_fused_dummy_act", None)
    width = 1 if categorical else desc.act_dim
    if dummy is None or dummy.shape[0] < n or dummy.shape[1] != width:
        dummy = self._fused_dummy_act = torch.zeros((n, width), dtype=torch.float32, device=flat.device)
    _, out = ops.actor_logp(flat.flat, desc, obs_t, dummy[:n], want_mu=True)
    if categorical:
        return out                                            # probabilities (DiscreteActor(softmax_output=True))
    sigma = (self.actor.sigma_param.view(1, -1) + torch.zeros_like(out)).exp()    # continuous.py:232-237
    return out, sigma


ProbabilisticActorPolicy._fused_dist_input = _fused_dist_input  # type: ignore[attr-defined]


class DiscreteActorPolicy(ProbabilisticActorPolicy):
    """Categorical policy over a Discrete action space (reinforce.py:195-243): no action scaling / bounding."""

    def __init__(self, *, actor: torch.nn.Module, dist_fn: TDistFn | None = None, deterministic_eval: bool = False,
                 action_space: Any, observation_space: Any | None = None) -> None:
        if not (type(action_space).__name__ == "Discrete" or hasattr(action_space, "n")):
            raise ValueError(f"Action space must be an instance of Discrete; got {action_space}")
        if dist_fn is None:
            from ...utils.net.discrete import dist_fn_categorical_from_logits
            dist_fn = dist_fn_categorical_from_logits
        super().__init__(actor=actor, dist_fn=dist_fn, deterministic_eval=deterministic_eval, action_space=action_space,
                         observation_space=observation_space, action_scaling=False, action_bound_method=None)
