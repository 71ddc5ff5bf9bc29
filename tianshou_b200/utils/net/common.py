"""MLP / Net building blocks (API of tianshou/utils/net/common.py:76-369, :457-470).

These are ordinary ``nn.Module``s: the Collector runs them for action inference and
``state_dict()`` round-trips unchanged.  The device updates do not call them -- they read the very
same parameter storage through the flat view of a ``FlatGroup`` (tianshou_b200/algorithm/flat_params.py).
"""
from __future__ import annotations

from collections.abc import Callable, Sequence
from typing import Any

import numpy as np
import torch
from torch import nn

from ..torch_utils import torch_device

ModuleType = type[nn.Module]
TLinearLayer = Callable[[int, int], nn.Module]


def _per_layer(spec: Any, args: Any, n: int) -> tuple[list, list]:
    if not spec:
        return [None] * n, [None] * n
    if isinstance(spec, list):
        assert len(spec) == n
        if isinstance(args, list):
            assert len(args) == n
            return spec, args
        return spec, [args] * n
    return [spec] * n, [args] * n


def _instantiate(cls: ModuleType, args: Any, *lead: Any) -> nn.Module:
    if isinstance(args, tuple):
        return cls(*lead, *args)
    if isinstance(args, dict):
        return cls(*lead, **args)
    return cls(*lead)


def miniblock(input_size: int, output_size: int = 0, norm_layer: ModuleType | None = None,
              norm_args: Any = None, activation: ModuleType | None = None, act_args: Any = None,
              linear_layer: TLinearLayer = nn.Linear) -> list[nn.Module]:
    """linear -> [norm] -> [activation]."""
    layers: list[nn.Module] = [linear_layer(input_size, output_size)]
    if norm_layer is not None:
        layers.append(_instantiate(norm_layer, norm_args, output_size))
    if activation is not None:
        layers.append(_instantiate(activation, act_args))
    return layers


class ModuleWithVectorOutput(nn.Module):
    def __init__(self, output_dim: int) -> None:
        super().__init__()
        self.output_dim = output_dim

    def get_output_dim(self) -> int:
        return self.output_dim


class MLP(ModuleWithVectorOutput):
    """Stack of miniblocks + optional output Linear; modules live in ``self.model`` (Sequential)."""

    def __init__(self, *, input_dim: int, output_dim: int = 0, hidden_sizes: Sequence[int] = (),
                 norm_layer: Any = None, norm_args: Any = None, activation: Any = nn.ReLU,
                 act_args: Any = None, linear_layer: TLinearLayer = nn.Linear,
                 flatten_input: bool = True) -> None:
        n = len(hidden_sizes)
        norms, nargs = _per_layer(norm_layer, norm_args, n)
        acts, aargs = _per_layer(activation, act_args, n)
        dims = [input_dim, *hidden_sizes]
        model: list[nn.Module] = []
        for i in range(n):
            model += miniblock(dims[i], dims[i + 1], norms[i], nargs[i], acts[i], aargs[i], linear_layer)
        if output_dim > 0:
            model.append(linear_layer(dims[-1], output_dim))
        super().__init__(output_dim or dims[-1])
        self.model = nn.Sequential(*model)
        self.flatten_input = flatten_input

    def forward(self, obs: np.ndarray | torch.Tensor) -> torch.Tensor:
        obs = torch.as_tensor(obs, device=torch_device(self), dtype=torch.float32)
        if self.flatten_input:
            obs = obs.flatten(1)
        return self.model(obs)


class Net(ModuleWithVectorOutput):
    """obs -> MLP features (``(logits, state)`` tuple like the reference, common.py:223-369).
    ``num_atoms > 1`` widens the last layer to ``prod(action_shape) * num_atoms`` outputs and returns them as
    ``[B, actions, num_atoms]`` (the distributional heads of QR-DQN, common.py:298-369); the dueling head is not provided."""

    def __init__(self, *, state_shape: int | Sequence[int], action_shape: Any = 0,
                 hidden_sizes: Sequence[int] = (), norm_layer: Any = None, norm_args: Any = None,
                 activation: Any = nn.ReLU, act_args: Any = None, softmax: bool = False,
                 concat: bool = False, num_atoms: int = 1, linear_layer: TLinearLayer = nn.Linear) -> None:
        input_dim = int(np.prod(state_shape))
        action_dim = int(np.prod(action_shape)) * num_atoms
        if concat:
            input_dim += action_dim
        model = MLP(input_dim=input_dim, output_dim=action_dim if not concat else 0,
                    hidden_sizes=hidden_sizes, norm_layer=norm_layer, norm_args=norm_args,
                    activation=activation, act_args=act_args, linear_layer=linear_layer)
        super().__init__(model.output_dim)
        self.softmax = softmax
        self.num_atoms = num_atoms
        self.model = model

    def forward(self, obs: Any, state: Any = None, info: dict | None = None) -> tuple[torch.Tensor, Any]:
        logits = self.model(obs)
        if self.num_atoms > 1:
            logits = logits.view(logits.shape[0], -1, self.num_atoms)
        if self.softmax:
            logits = torch.softmax(logits, dim=-1)
        return logits, state


class EnsembleLinear(nn.Module):
    """``ensemble_size`` Linear layers applied side by side (common.py:518-550): ``x @ weight + bias_weights`` with
    ``weight [E, in, out]`` and ``bias_weights [E, 1, out]``, so a ``[B, in]`` input gives ``[E, B, out]`` and an
    ``[E, B, in]`` input maps member by member.  Initialised like the reference, uniform in +-sqrt(1 / in)."""

    def __init__(self, ensemble_size: int, in_feature: int, out_feature: int, bias: bool = True) -> None:
        super().__init__()
        k = np.sqrt(1.0 / in_feature)
        weight_data = torch.rand((ensemble_size, in_feature, out_feature)) * 2 * k - k
        self.weight = nn.Parameter(weight_data, requires_grad=True)
        self.bias_weights: nn.Parameter | None = None
        if bias:
            bias_data = torch.rand((ensemble_size, 1, out_feature)) * 2 * k - k
            self.bias_weights = nn.Parameter(bias_data, requires_grad=True)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        x = torch.matmul(x, self.weight)
        if self.bias_weights is not None:
            x = x + self.bias_weights
        return x


class ActorCritic(nn.Module):
    """Parameter holder so one optimizer covers actor and critic (common.py:457-470)."""

    def __init__(self, actor: nn.Module, critic: nn.Module) -> None:
        super().__init__()
        self.actor = actor
        self.critic = critic
