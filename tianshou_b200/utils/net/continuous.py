"""Deterministic and Gaussian actors / critic heads (API of tianshou/utils/net/continuous.py:28-238)."""
from __future__ import annotations

import warnings
from collections.abc import Sequence
from typing import Any

import numpy as np
import torch
from torch import nn

from ..torch_utils import torch_device
from .common import MLP, ModuleWithVectorOutput, TLinearLayer

SIGMA_MIN = -20
SIGMA_MAX = 2


class AbstractContinuousActorDeterministic(ModuleWithVectorOutput):
    """Marker interface for continuous deterministic actors (DDPG like), continuous.py:28-29."""


class ContinuousActorDeterministic(AbstractContinuousActorDeterministic):
    """s -> ``max_action * tanh(last(preprocess(s)))`` (continuous.py:32-85): the actor of DDPG / TD3 / TD3+BC.  The submodules
    and their order are the reference's, so ``state_dict()`` keys and seeded initial weights match."""

    def __init__(self, *, preprocess_net: ModuleWithVectorOutput, action_shape: Any, hidden_sizes: Sequence[int] = (),
                 max_action: float = 1.0) -> None:
        output_dim = int(np.prod(action_shape))
        super().__init__(output_dim)
        self.preprocess = preprocess_net
        self.last = MLP(input_dim=preprocess_net.get_output_dim(), output_dim=self.output_dim, hidden_sizes=hidden_sizes)
        self.max_action = max_action

    def get_preprocess_net(self) -> ModuleWithVectorOutput:
        return self.preprocess

    def get_output_dim(self) -> int:
        return self.output_dim

    def forward(self, obs: Any, state: Any = None, info: dict[str, Any] | None = None) -> tuple[torch.Tensor, Any]:
        action_BA, hidden_BH = self.preprocess(obs, state)
        action_BA = self.max_action * torch.tanh(self.last(action_BA))
        return action_BA, hidden_BH


class ContinuousCritic(ModuleWithVectorOutput):
    """V(s) (or Q(s,a) when ``act`` is given): preprocess net -> ``last`` MLP -> 1."""

    def __init__(self, *, preprocess_net: ModuleWithVectorOutput, hidden_sizes: Sequence[int] = (),
                 linear_layer: TLinearLayer = nn.Linear, flatten_input: bool = True,
                 apply_preprocess_net_to_obs_only: bool = False) -> None:
        super().__init__(output_dim=1)
        self.preprocess = preprocess_net
        self.apply_preprocess_net_to_obs_only = apply_preprocess_net_to_obs_only
        self.last = MLP(input_dim=preprocess_net.get_output_dim(), output_dim=1, hidden_sizes=hidden_sizes,
                        linear_layer=linear_layer, flatten_input=flatten_input)

    def forward(self, obs: np.ndarray | torch.Tensor, act: np.ndarray | torch.Tensor | None = None,
                info: dict[str, Any] | None = None) -> torch.Tensor:
        device = torch_device(self)
        obs = torch.as_tensor(obs, device=device, dtype=torch.float32)
        if self.apply_preprocess_net_to_obs_only:
            obs, _ = self.preprocess(obs)
        obs = obs.flatten(1)
        if act is not None:
            act = torch.as_tensor(act, device=device, dtype=torch.float32).flatten(1)
            obs = torch.cat([obs, act], dim=1)
        if not self.apply_preprocess_net_to_obs_only:
            obs, _ = self.preprocess(obs)
        return self.last(obs)


class ContinuousActorProbabilistic(ModuleWithVectorOutput):
    """(mu, sigma) of a diagonal Gaussian; sigma is ``exp(sigma_param)`` (state independent) unless
    ``conditioned_sigma``."""

    def __init__(self, *, preprocess_net: ModuleWithVectorOutput, action_shape: Any,
                 hidden_sizes: Sequence[int] = (), max_action: float = 1.0, unbounded: bool = False,
                 conditioned_sigma: bool = False) -> None:
        output_dim = int(np.prod(action_shape))
        super().__init__(output_dim)
        if unbounded and not np.isclose(max_action, 1.0):
            warnings.warn("Note that max_action input will be discarded when unbounded is True.")
            max_action = 1.0
        self.preprocess = preprocess_net
        input_dim = preprocess_net.get_output_dim()
        self.mu = MLP(input_dim=input_dim, output_dim=output_dim, hidden_sizes=hidden_sizes)
        self._c_sigma = conditioned_sigma
        if conditioned_sigma:
            self.sigma = MLP(input_dim=input_dim, output_dim=output_dim, hidden_sizes=hidden_sizes)
        else:
            self.sigma_param = nn.Parameter(torch.zeros(output_dim, 1))
        self.max_action = max_action
        self._unbounded = unbounded

    def get_preprocess_net(self) -> ModuleWithVectorOutput:
        return self.preprocess

    def forward(self, obs: Any, state: Any = None, info: dict[str, Any] | None = None
                ) -> tuple[tuple[torch.Tensor, torch.Tensor], Any]:
        logits, _hidden = self.preprocess(obs, state)
        mu = self.mu(logits)
        if not self._unbounded:
            mu = self.max_action * torch.tanh(mu)
        if self._c_sigma:
            sigma = torch.clamp(self.sigma(logits), min=SIGMA_MIN, max=SIGMA_MAX).exp()
        else:
            shape = [1] * len(mu.shape)
            shape[1] = -1
            sigma = (self.sigma_param.view(shape) + torch.zeros_like(mu)).exp()
        return (mu, sigma), state


class Perturbation(nn.Module):
    """BCQ's perturbation network (continuous.py:378-412): ``clamp(a + phi * max_action * tanh(logits), +-max_action)`` with
    ``logits = preprocess_net(cat([s, a], -1))[0]``.  As in the reference, that ``[0]`` is the logits of a ``Net`` (which
    returns ``(logits, state)``) but ROW 0 of the output of an ``MLP``, whose perturbation then applies to every row."""

    def __init__(self, *, preprocess_net: nn.Module, max_action: float, phi: float = 0.05):
        super().__init__()
        self.preprocess_net = preprocess_net
        self.max_action = max_action
        self.phi = phi

    def forward(self, state: torch.Tensor, action: torch.Tensor) -> torch.Tensor:
        logits = self.preprocess_net(torch.cat([state, action], -1))[0]
        noise = self.phi * self.max_action * torch.tanh(logits)
        return (noise + action).clamp(-self.max_action, self.max_action)


class VAE(nn.Module):
    """The VAE over actions of BCQ (continuous.py:415-490): the encoder on [s | a] (output width ``hidden_dim``), the ``mean`` and
    ``log_std`` heads (``log_std`` clamped to [-4, 15]), the decoder on [s | z] (output width A) under ``max_action * tanh``.
    ``decode(state)`` without a latent draws it with ``torch.randn`` on torch's CPU generator, clamped to [-0.5, 0.5]."""

    def __init__(self, *, encoder: nn.Module, decoder: nn.Module, hidden_dim: int, latent_dim: int, max_action: float):
        super().__init__()
        self.encoder = encoder
        self.mean = nn.Linear(hidden_dim, latent_dim)
        self.log_std = nn.Linear(hidden_dim, latent_dim)
        self.decoder = decoder
        self.max_action = max_action
        self.latent_dim = latent_dim

    def forward(self, state: torch.Tensor, action: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        latent_z = self.encoder(torch.cat([state, action], -1))
        mean = self.mean(latent_z)
        log_std = self.log_std(latent_z).clamp(-4, 15)
        std = torch.exp(log_std)
        latent_z = mean + std * torch.randn_like(std)
        reconstruction = self.decode(state, latent_z)
        return reconstruction, mean, std

    def decode(self, state: torch.Tensor, latent_z: torch.Tensor | None = None) -> torch.Tensor:
        if latent_z is None:
            device = torch_device(self)
            latent_z = torch.randn(state.shape[:-1] + (self.latent_dim,)).to(device).clamp(-0.5, 0.5)
        return self.max_action * torch.tanh(self.decoder(torch.cat([state, latent_z], -1)))
