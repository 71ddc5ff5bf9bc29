"""The deterministic continuous policies of DDPG / TD3 / TD3+BC (API of tianshou/algorithm/modelfree/ddpg.py:45-190).  Only the
policy classes live here, at the reference's import path; the algorithms are in td3.py and imitation/td3_bc.py.  ``forward`` is
the torch path the Collector runs."""
from __future__ import annotations

import warnings
from abc import ABC
from typing import Any, Literal

import numpy as np
import torch

from ...data import Batch
from ...exploration import BaseNoise, GaussianNoise
from ..base import Policy


class ContinuousPolicyWithExplorationNoise(Policy, ABC):
    """A continuous policy that adds ``exploration_noise`` to its numpy actions (ddpg.py:45-111); ``"default"`` is
    ``GaussianNoise(sigma=0.1)``."""

    def __init__(self, *, exploration_noise: BaseNoise | Literal["default"] | None = None, action_space: Any,
                 observation_space: Any | None = None, action_scaling: bool = True,
                 action_bound_method: Literal["clip"] | None = "clip") -> None:
        super().__init__(action_space=action_space, observation_space=observation_space, action_scaling=action_scaling,
                         action_bound_method=action_bound_method)
        if exploration_noise == "default":
            exploration_noise = GaussianNoise(sigma=0.1)
        self.exploration_noise = exploration_noise

    def set_exploration_noise(self, noise: BaseNoise | None) -> None:
        """Set the exploration noise."""
        self.exploration_noise = noise

    def add_exploration_noise(self, act: Any, batch: Any) -> Any:
        if self.exploration_noise is None:
            return act
        if isinstance(act, np.ndarray):
            return act + self.exploration_noise(act.shape)
        warnings.warn("Cannot add exploration noise to non-numpy_array action.")
        return act


class ContinuousDeterministicPolicy(ContinuousPolicyWithExplorationNoise):
    """A policy whose actor maps states to actions directly (ddpg.py:114-190)."""

    def __init__(self, *, actor: torch.nn.Module, exploration_noise: BaseNoise | Literal["default"] | None = None,
                 action_space: Any, observation_space: Any | None = None, action_scaling: bool = True,
                 action_bound_method: Literal["clip"] | None = "clip") -> None:
        if action_scaling and not np.isclose(actor.max_action, 1.0):
            warnings.warn(
                "action_scaling and action_bound_method are only intended to deal"
                "with unbounded model action space, but find actor model bound"
                f"action space with max_action={actor.max_action}."
                "Consider using unbounded=True option of the actor model,"
                "or set action_scaling to False and action_bound_method to None.",
            )
        super().__init__(exploration_noise=exploration_noise, action_space=action_space, observation_space=observation_space,
                         action_scaling=action_scaling, action_bound_method=action_bound_method)
        self.actor = actor

    def forward(self, batch: Batch, state: Any = None, model: torch.nn.Module | None = None, **kwargs: Any) -> Batch:
        """``act`` = the actor's (or ``model``'s) output on ``batch.obs``, ``state`` its hidden state."""
        if model is None:
            model = self.actor
        actions, hidden = model(batch.obs, state=state, info=batch.get("info"))
        return Batch(act=actions, state=hidden)
