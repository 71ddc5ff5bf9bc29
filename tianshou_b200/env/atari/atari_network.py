"""NatureCNN Q-networks (API of tianshou/env/atari/atari_network.py:26-235).

Ordinary ``nn.Module``s: the Collector runs them for action selection; ``DQN.update`` reads the same parameter
storage through a flat view and runs the conv stack as implicit GEMM on the tensor cores (algorithm/netgraph.py).
"""
from __future__ import annotations

from collections.abc import Callable, Sequence
from typing import Any

import numpy as np
import torch
from torch import nn

from ...utils.net.common import ModuleWithVectorOutput
from ...utils.net.discrete import NoisyLinear
from ...utils.torch_utils import torch_device


class ScaledObsInputActionReprNet(ModuleWithVectorOutput):
    """obs / denom before the wrapped network (atari_network.py:26-55)."""

    def __init__(self, module: ModuleWithVectorOutput, denom: float = 255.0) -> None:
        super().__init__(module.get_output_dim())
        self.module = module
        self.denom = denom

    def forward(self, obs: Any, state: Any = None, info: dict | None = None) -> tuple[torch.Tensor, Any]:
        if info is None:
            info = {}
        scaled = obs / self.denom        # numpy uint8 / float -> float64, cast to f32 by the wrapped net (as in the reference)
        return self.module.forward(scaled, state, info)


def scale_obs(module: ModuleWithVectorOutput, denom: float = 255.0) -> ScaledObsInputActionReprNet:
    return ScaledObsInputActionReprNet(module, denom=denom)


class DQNet(ModuleWithVectorOutput):
    """Human-level control through deep reinforcement learning (atari_network.py:60-122): conv 8x8/4 -> 4x4/2 -> 3x3/1,
    Linear(3136, 512), Linear(512, actions), ReLU between."""

    def __init__(self, c: int, h: int, w: int, action_shape: Sequence[int] | int, features_only: bool = False,
                 output_dim_added_layer: int | None = None,
                 layer_init: Callable[[nn.Module], nn.Module] = lambda x: x) -> None:
        if not features_only and output_dim_added_layer is not None:
            raise ValueError("Should not provide explicit output dimension using `output_dim_added_layer` when "
                             "`features_only` is true.")
        net = nn.Sequential(
            layer_init(nn.Conv2d(c, 32, kernel_size=8, stride=4)), nn.ReLU(inplace=True),
            layer_init(nn.Conv2d(32, 64, kernel_size=4, stride=2)), nn.ReLU(inplace=True),
            layer_init(nn.Conv2d(64, 64, kernel_size=3, stride=1)), nn.ReLU(inplace=True),
            nn.Flatten())
        with torch.no_grad():
            base_cnn_output_dim = int(np.prod(net(torch.zeros(1, c, h, w)).shape[1:]))
        if not features_only:
            action_dim = int(np.prod(action_shape))
            net = nn.Sequential(net, layer_init(nn.Linear(base_cnn_output_dim, 512)), nn.ReLU(inplace=True),
                                layer_init(nn.Linear(512, action_dim)))
            output_dim = action_dim
        elif output_dim_added_layer is not None:
            net = nn.Sequential(net, layer_init(nn.Linear(base_cnn_output_dim, output_dim_added_layer)), nn.ReLU(inplace=True))
            output_dim = output_dim_added_layer
        else:
            output_dim = base_cnn_output_dim
        super().__init__(output_dim)
        self.net = net
        self.input_shape = (c, h, w)

    def forward(self, obs: Any, state: Any = None, info: dict | None = None) -> tuple[torch.Tensor, Any]:
        obs = torch.as_tensor(obs, device=torch_device(self), dtype=torch.float32)
        return self.net(obs), state


class QRDQNet(DQNet):
    """Distributional Reinforcement Learning with Quantile Regression (atari_network.py:211-235): a ``DQNet`` whose last Linear
    has ``actions * num_quantiles`` outputs, returned as ``[B, actions, num_quantiles]``."""

    def __init__(self, *, c: int, h: int, w: int, action_shape: Sequence[int] | int, num_quantiles: int = 200) -> None:
        self.action_num = int(np.prod(action_shape))
        super().__init__(c=c, h=h, w=w, action_shape=[self.action_num * num_quantiles])
        self.num_quantiles = num_quantiles

    def forward(self, obs: Any, state: Any = None, info: dict | None = None) -> tuple[torch.Tensor, Any]:
        obs, state = super().forward(obs)
        return obs.view(-1, self.action_num, self.num_quantiles), state


class C51Net(DQNet):
    """A distributional perspective on reinforcement learning (atari_network.py:125-151): a ``DQNet`` whose last Linear has
    ``actions * num_atoms`` outputs, a softmax over each action's atoms, returned as ``[B, actions, num_atoms]``."""

    def __init__(self, *, c: int, h: int, w: int, action_shape: Sequence[int] | int, num_atoms: int = 51) -> None:
        self.action_num = int(np.prod(action_shape))
        super().__init__(c=c, h=h, w=w, action_shape=[self.action_num * num_atoms])
        self.num_atoms = num_atoms

    def forward(self, obs: Any, state: Any = None, info: dict | None = None) -> tuple[torch.Tensor, Any]:
        obs, state = super().forward(obs)
        obs = obs.view(-1, self.num_atoms).softmax(dim=-1)
        return obs.view(-1, self.action_num, self.num_atoms), state


class RainbowNet(DQNet):
    """Rainbow: Combining Improvements in Deep Reinforcement Learning (atari_network.py:154-208): the ``DQNet`` convolutions
    (``features_only``), then a Q head ``Linear(features, 512), ReLU, Linear(512, actions * num_atoms)`` and, when
    ``is_dueling``, a V head ``Linear(features, 512), ReLU, Linear(512, num_atoms)``; the Linear layers are ``NoisyLinear(.,
    ., noisy_std)`` when ``is_noisy``.  ``forward`` returns ``softmax(q - q.mean(1) + v)`` (or ``softmax(q)``) over each action's
    atoms, ``[B, actions, num_atoms]``."""

    def __init__(self, *, c: int, h: int, w: int, action_shape: Sequence[int] | int, num_atoms: int = 51,
                 noisy_std: float = 0.5, is_dueling: bool = True, is_noisy: bool = True) -> None:
        super().__init__(c=c, h=h, w=w, action_shape=action_shape, features_only=True)
        self.action_num = int(np.prod(action_shape))
        self.num_atoms = num_atoms

        def linear(x: int, y: int) -> NoisyLinear | nn.Linear:
            if is_noisy:
                return NoisyLinear(x, y, noisy_std)
            return nn.Linear(x, y)

        self.Q = nn.Sequential(linear(self.output_dim, 512), nn.ReLU(inplace=True), linear(512, self.action_num * self.num_atoms))
        self._is_dueling = is_dueling
        if self._is_dueling:
            self.V = nn.Sequential(linear(self.output_dim, 512), nn.ReLU(inplace=True), linear(512, self.num_atoms))
        self.output_dim = self.action_num * self.num_atoms

    def forward(self, obs: Any, state: Any = None, info: dict | None = None) -> tuple[torch.Tensor, Any]:
        obs, state = super().forward(obs)
        q = self.Q(obs).view(-1, self.action_num, self.num_atoms)
        if self._is_dueling:
            v = self.V(obs).view(-1, 1, self.num_atoms)
            logits = q - q.mean(dim=1, keepdim=True) + v
        else:
            logits = q
        return logits.softmax(dim=2), state
