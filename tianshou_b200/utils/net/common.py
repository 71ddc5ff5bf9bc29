"""MLP / Net building blocks (API of tianshou/utils/net/common.py:76-369, :457-470, :553-674).

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
    ``[B, actions, num_atoms]`` (the distributional heads of QR-DQN, common.py:298-369).  ``dueling_param = (q_kwargs, v_kwargs)``
    ends the MLP trunk at its last hidden layer and puts two MLPs on it, built from those keyword dicts: ``Q`` with
    ``prod(action_shape) * num_atoms`` outputs and ``V`` with ``num_atoms``; the output is ``q - q.mean(1) + v`` over
    ``[B, actions, num_atoms]`` (``[B, actions]`` when ``num_atoms == 1``).  Only RainbowDQN runs a network with these heads on
    the device."""

    def __init__(self, *, state_shape: int | Sequence[int], action_shape: Any = 0,
                 hidden_sizes: Sequence[int] = (), norm_layer: Any = None, norm_args: Any = None,
                 activation: Any = nn.ReLU, act_args: Any = None, softmax: bool = False,
                 concat: bool = False, num_atoms: int = 1,
                 dueling_param: tuple[dict[str, Any], dict[str, Any]] | None = None,
                 linear_layer: TLinearLayer = nn.Linear) -> None:
        input_dim = int(np.prod(state_shape))
        action_dim = int(np.prod(action_shape)) * num_atoms
        if concat:
            input_dim += action_dim
        use_dueling = dueling_param is not None
        model = MLP(input_dim=input_dim, output_dim=action_dim if not use_dueling and not concat else 0,
                    hidden_sizes=hidden_sizes, norm_layer=norm_layer, norm_args=norm_args,
                    activation=activation, act_args=act_args, linear_layer=linear_layer)
        Q: MLP | None = None
        V: MLP | None = None
        if use_dueling:
            q_kwargs = {**dueling_param[0], "input_dim": model.output_dim}
            v_kwargs = {**dueling_param[1], "input_dim": model.output_dim}
            q_kwargs["output_dim"] = 0 if concat else action_dim
            v_kwargs["output_dim"] = 0 if concat else num_atoms
            Q, V = MLP(**q_kwargs), MLP(**v_kwargs)
            output_dim = Q.output_dim
        else:
            output_dim = model.output_dim
        super().__init__(output_dim)
        self.use_dueling = use_dueling
        self.softmax = softmax
        self.num_atoms = num_atoms
        self.model = model
        self.Q = Q
        self.V = V

    def forward(self, obs: Any, state: Any = None, info: dict | None = None) -> tuple[torch.Tensor, Any]:
        logits = self.model(obs)
        if self.use_dueling:
            q, v = self.Q(logits), self.V(logits)
            if self.num_atoms > 1:
                q = q.view(logits.shape[0], -1, self.num_atoms)
                v = v.view(logits.shape[0], -1, self.num_atoms)
            logits = q - q.mean(dim=1, keepdim=True) + v
        elif self.num_atoms > 1:
            logits = logits.view(logits.shape[0], -1, self.num_atoms)
        if self.softmax:
            logits = torch.softmax(logits, dim=-1)
        return logits, state


class Recurrent(ModuleWithVectorOutput):
    """LSTM Q-network of DRQN (common.py:372-453): ``fc1`` (no activation) -> ``nn.LSTM(layer_num, batch_first)`` -> ``fc2`` on the
    last step.  ``obs`` is ``[B, len, D]`` (a stacked sample) or ``[B, D]`` (one step, read as a length-1 sequence); ``state`` is
    None or ``{hidden, cell}`` as ``[B, layer_num, H]``.  Returns ``(logits, {hidden, cell})``.  ``DQN.update`` runs this network on
    the device (algorithm/recurrent.py); this torch forward is the Collector's path."""

    def __init__(self, *, layer_num: int, state_shape: int | Sequence[int], action_shape: Any,
                 hidden_layer_size: int = 128) -> None:
        output_dim = int(np.prod(action_shape))
        super().__init__(output_dim)
        self.nn = nn.LSTM(input_size=hidden_layer_size, hidden_size=hidden_layer_size, num_layers=layer_num, batch_first=True)
        self.fc1 = nn.Linear(int(np.prod(state_shape)), hidden_layer_size)
        self.fc2 = nn.Linear(hidden_layer_size, output_dim)

    def forward(self, obs: Any, state: Any = None, info: dict | None = None) -> tuple[torch.Tensor, Any]:
        from ...data import Batch
        if state is not None and not {"hidden", "cell"}.issubset(state.keys()):
            raise ValueError(f"Expected to find keys 'hidden' and 'cell' but instead found {state.keys()}")
        obs = torch.as_tensor(obs, device=torch_device(self), dtype=torch.float32)
        if len(obs.shape) == 2:
            obs = obs.unsqueeze(-2)
        obs = self.fc1(obs)
        self.nn.flatten_parameters()
        if state is None:
            obs, (hidden, cell) = self.nn(obs)
        else:
            obs, (hidden, cell) = self.nn(obs, (state["hidden"].transpose(0, 1).contiguous(),
                                                state["cell"].transpose(0, 1).contiguous()))
        obs = self.fc2(obs[:, -1])
        return obs, Batch({"hidden": hidden.transpose(0, 1).detach(), "cell": cell.transpose(0, 1).detach()})


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


class BranchingNet(nn.Module):
    """Branching dueling Q-network of BDQN (common.py:553-674, arXiv:1711.08946): a shared trunk ``common`` (an MLP ending in
    its last hidden layer's activation), a state-value MLP ``value`` with one output, and ``num_branches`` identical action MLPs
    ``branches`` with ``action_per_branch`` outputs each, all reading the trunk.  ``forward`` gives ``[B, num_branches,
    action_per_branch]`` Q-values ``value + (scores - scores.mean(2))``.  An empty ``common_hidden_sizes`` fails here, as in the
    reference."""

    def __init__(self, *, state_shape: int | Sequence[int], num_branches: int = 0, action_per_branch: int = 2,
                 common_hidden_sizes: list[int] | None = None, value_hidden_sizes: list[int] | None = None,
                 action_hidden_sizes: list[int] | None = None, norm_layer: ModuleType | None = None, norm_args: Any = None,
                 activation: ModuleType | None = nn.ReLU, act_args: Any = None) -> None:
        super().__init__()
        common_hidden_sizes = common_hidden_sizes or []
        value_hidden_sizes = value_hidden_sizes or []
        action_hidden_sizes = action_hidden_sizes or []
        self.num_branches = num_branches
        self.action_per_branch = action_per_branch
        kw = dict(norm_layer=norm_layer, norm_args=norm_args, activation=activation, act_args=act_args)
        self.common = MLP(input_dim=int(np.prod(state_shape)), output_dim=0, hidden_sizes=common_hidden_sizes, **kw)
        self.value = MLP(input_dim=common_hidden_sizes[-1], output_dim=1, hidden_sizes=value_hidden_sizes, **kw)
        self.branches = nn.ModuleList([
            MLP(input_dim=common_hidden_sizes[-1], output_dim=action_per_branch, hidden_sizes=action_hidden_sizes, **kw)
            for _ in range(self.num_branches)])

    def forward(self, obs: Any, state: Any = None, info: dict | None = None) -> tuple[torch.Tensor, Any]:
        common_out = self.common(obs)
        value_out = torch.unsqueeze(self.value(common_out), 1)
        action_scores = torch.stack([b(common_out) for b in self.branches], 1)
        action_scores = action_scores - torch.mean(action_scores, 2, keepdim=True)
        return value_out + action_scores, state


class ActorCritic(nn.Module):
    """Parameter holder so one optimizer covers actor and critic (common.py:457-470)."""

    def __init__(self, actor: nn.Module, critic: nn.Module) -> None:
        super().__init__()
        self.actor = actor
        self.critic = critic
