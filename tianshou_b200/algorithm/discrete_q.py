"""What the discrete-action value-based updates share: DQN, QR-DQN, discrete CQL, discrete BCQ and discrete CRR stand on
``DiscreteQCore``; discrete SAC reads its networks and draws its batches with the same functions.

Reference: modelfree/dqn.py:170-283 (QLearningOffPolicyAlgorithm: the n-step return, the lagged network refreshed when
``_iter % target_update_freq == 0``), :384-401 (``q[np.arange(len(q)), batch.act]``: an action outside the network's outputs
raises), utils/lagged_network.py:21-41 and :81-103 (the lagged copy under ``.module``, its full copy), utils/net/discrete.py:29-123
(``DiscreteActor`` / ``DiscreteCritic``: a preprocess net, then the ``last`` MLP).
"""
from __future__ import annotations

from collections.abc import Callable
from typing import Any

import numpy as np
import torch
from torch import nn

from .._cabi import to_device
from ..data import Batch, ReplayBuffer
from ..utils.net.discrete import NoisyLinear
from .base import Algorithm
from .flat_params import DeviceScratch, FlatGroup, UnsupportedModelError
from .netgraph import ACT_NONE, _Layer, _out_shape, compile_sequential, module_layers, network_heads
from .obs_source import DeviceObsSource, device_obs_source
from .twin_critic import per_weight


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
    if isinstance(first, (nn.Linear, NoisyLinear)):
        return inner, (int(first.in_features),), scale
    raise UnsupportedModelError(f"cannot infer the input shape of {type(inner).__name__}")


def atom_chain(inner: Any, in_shape: tuple[int, ...], n_actions: int, n_atoms: int, kind: str, atom_name: str,
               noisy: bool = False) -> list:
    """The layer chain of a distributional Q-network (QR-DQN's quantiles, C51's atoms): ``inner`` read as a plain chain ending in
    ``Linear(., n_actions * n_atoms)`` with no activation, the output viewed as ``[B, n_actions, n_atoms]``; anything else is
    refused.  ``kind`` names the network, ``atom_name`` the per-action outputs (``num_<atom_name>`` is the keyword).
    ``noisy``: ``NoisyLinear`` layers join the chain (Rainbow)."""
    return _check_head(compile_sequential(module_layers(inner), in_shape, noisy=noisy), n_actions * n_atoms,
                       f"{n_actions} actions x {n_atoms} {atom_name}", f"the {kind} network", f"actions * num_{atom_name}")


def _check_head(layers: list[_Layer], width: int, what: str, name: str, over: str) -> list[_Layer]:
    if not layers or layers[-1].kind != "linear" or layers[-1].act != ACT_NONE:
        raise UnsupportedModelError(f"{name} must end in a linear layer over {over}")
    if layers[-1].out_dim != width:
        raise UnsupportedModelError(f"the network has {layers[-1].out_dim} outputs, not {what}")
    return layers


def dueling_atom_chains(model: Any, n_actions: int, n_atoms: int) -> tuple[Any, tuple[int, ...], float, list[list[_Layer]]]:
    """(inner module, input shape, input denominator, chains) of a categorical network whose Linear layers may be
    ``NoisyLinear`` (Rainbow), optionally behind ``ScaledObsInputActionReprNet``.  A network with a V head (``Net(dueling_param=
    ...)``, ``RainbowNet(is_dueling=True)``) gives three chains: the trunk, the Q head over ``n_actions * n_atoms`` outputs and the
    V head over ``n_atoms``, both reading the trunk's output.  ``RainbowNet(is_dueling=False)`` gives its trunk and Q head as one
    chain, any other network its plain chain (``atom_chain``)."""
    heads = network_heads(model.module if hasattr(model, "denom") and hasattr(model, "module") else model)
    if heads is None:
        inner, in_shape, scale = describe_q_network(model)
        return inner, in_shape, scale, [atom_chain(inner, in_shape, n_actions, n_atoms, "categorical", "atoms", noisy=True)]
    scale, inner = (float(model.denom), model.module) if hasattr(model, "denom") and hasattr(model, "module") else (1.0, model)
    trunk_m, q_m, v_m = heads
    if hasattr(inner, "input_shape"):
        in_shape = tuple(inner.input_shape)
    elif trunk_m and hasattr(trunk_m[0], "in_features"):
        in_shape = (int(trunk_m[0].in_features),)
    else:
        raise UnsupportedModelError(f"{type(inner).__name__}: the heads need a trunk that starts with a linear layer (hidden_sizes)")
    what, over = f"{n_actions} actions x {n_atoms} atoms", "actions * num_atoms"
    if v_m is None:
        return inner, in_shape, scale, [_check_head(compile_sequential(trunk_m + q_m, in_shape, noisy=True), n_actions * n_atoms, what,
                                                    "the Q head", over)]
    trunk = compile_sequential(trunk_m, in_shape, noisy=True)
    feat = _out_shape(trunk, in_shape)
    q = _check_head(compile_sequential(q_m, feat, noisy=True), n_actions * n_atoms, what, "the Q head", over)
    v = _check_head(compile_sequential(v_m, feat, noisy=True), n_atoms, f"{n_atoms} atoms", "the V head", "num_atoms")
    return inner, in_shape, scale, [trunk, q, v]


def describe_discrete_head(net: Any, role: str) -> tuple[Any, Any, tuple[int, ...], float]:
    """``DiscreteActor`` / ``DiscreteCritic`` -> (the preprocess net's inner module, the ``last`` MLP, input shape, input
    denominator).  The preprocess net is anything ``describe_q_network`` reads; a softmax output of it is refused."""
    pre, last = getattr(net, "preprocess", None), getattr(net, "last", None)
    if pre is None or last is None:
        raise UnsupportedModelError(f"{role}: expected a DiscreteActor / DiscreteCritic (preprocess net + last MLP), got "
                                    f"{type(net).__name__}")
    try:
        inner, shape, scale = describe_q_network(pre)
    except UnsupportedModelError as e:
        raise UnsupportedModelError(f"{role}: {e}") from e
    if getattr(pre, "softmax", False) or getattr(inner, "softmax", False):
        raise UnsupportedModelError(f"{role}: a softmax preprocess output is not supported")
    return inner, last, shape, scale


def sample_discrete(buffer: ReplayBuffer, sample_size: int | None, obs_source: Callable[..., DeviceObsSource],
                    device: torch.device, n_actions: int, branches: int | None = None) -> tuple[Batch, Any]:
    """Indices from the buffer's host RNG streams (identical to the reference's draws); the observations as
    ``obs_source(buffer, indices, "obs")`` reads them on the device, the actions as int64 device rows, the importance weight
    of a prioritised buffer.  The loss kernels index a row of ``n_actions`` values with each drawn action: an action outside
    ``[0, n_actions)`` is refused here, before anything is launched.  ``branches``: multi-discrete actions, one per branch, as
    ``[B, branches]`` rows; a buffer whose action rows have another shape is refused before the index draw."""
    if branches is not None:
        shape = np.shape(buffer.act)[1:]
        if shape != (branches,):
            raise ValueError(f"the buffer holds action rows of shape {shape}, the network has {branches} branches: rows of "
                             f"{branches} actions expected")
    indices = buffer.sample_indices(sample_size)
    act = np.asarray(buffer.act)[indices]
    if act.size and (act.min() < 0 or act.max() >= n_actions):
        raise ValueError(f"the buffer holds actions in [{act.min()}, {act.max()}], the networks have {n_actions} outputs")
    batch = Batch()
    batch.__dict__["obs"] = obs_source(buffer, indices, "obs")
    act = act.reshape(-1) if branches is None else act.reshape(len(act), branches)
    batch.__dict__["act"] = to_device(np.ascontiguousarray(act).astype(np.int64), device)
    weight = per_weight(buffer, indices, device)
    if weight is not None:
        batch.__dict__["weight"] = weight
    batch.__dict__["info"] = Batch()
    return batch, indices


def lagged_group(online: FlatGroup, lagged_params: list[nn.Parameter]) -> FlatGroup:
    """The flat group of a lagged copy whose parameters match the first ``len(lagged_params)`` of ``online``'s, shape by
    shape: its flat buffer is a prefix of the online layout, so the online chains run on it as ``params=`` and one copy
    refreshes it.  A copy of the whole network is the trivial prefix.  The lagged modules' parameters become views of it."""
    shapes = [tuple(p.shape) for p in lagged_params]
    if shapes != [tuple(p.shape) for p in online.params[: len(shapes)]]:
        raise UnsupportedModelError(f"the lagged network's parameter shapes {shapes} are not a prefix of the online network's "
                                    f"{[tuple(p.shape) for p in online.params]}")
    return FlatGroup(lagged_params, online.device)


def refresh_lagged(online: FlatGroup, lagged: FlatGroup) -> None:
    """The full copy of the lagged network (lagged_network.py:81-103): one device copy of the online prefix."""
    online.ensure_adopted()
    lagged.ensure_adopted()
    lagged.flat.copy_(online.flat[: lagged.n])


class DiscreteQCore(Algorithm):
    """A discrete-action value-based update on one CUDA device.  The subclass builds its networks, calls ``_init_discrete``
    and sets ``gamma``, ``n_step``, ``_target_q``, ``_group`` and (with a lagged network) ``_g_old``; the core reads the
    observations, draws the batch (refusing actions outside ``[0, n_actions)``), computes the n-step return and refreshes
    the lagged copy on its tick."""

    def _init_discrete(self, dev: torch.device, in_shape: tuple[int, ...], in_scale: float, n_actions: int, seq: bool = False) -> None:
        """``seq``: the network reads each sample's stacked observations as a sequence (a ``Recurrent`` network)."""
        self._dev, self._in_shape, self._in_scale, self.n_actions, self._seq = dev, in_shape, in_scale, n_actions, seq
        self._iter = 0
        self._scratch = DeviceScratch(dev)
        self._buf = self._scratch.tensor

    def _obs_source(self, buffer: ReplayBuffer, indices: np.ndarray | torch.Tensor, key: str = "obs") -> DeviceObsSource:
        """How the network reads ``buffer[indices].<key>`` without materialising it on the host (obs_source.py)."""
        return device_obs_source(buffer, indices, key, self._in_shape, self._in_scale, self._dev, self._buf, seq=self._seq)

    def _sample(self, buffer: ReplayBuffer, sample_size: int | None) -> tuple[Batch, Any]:
        return sample_discrete(buffer, sample_size, self._obs_source, self._dev, self.n_actions)

    def _preprocess_batch(self, batch: Batch, buffer: ReplayBuffer, indices: np.ndarray) -> Batch:
        return self.compute_nstep_return(batch=batch, buffer=buffer, indices=indices, target_q_fn=self._target_q,
                                         gamma=self.gamma, n_step=self.n_step)

    def _tick_lagged(self, freq: int) -> None:
        """Before the step: the lagged copy is refreshed when ``freq > 0 and _iter % freq == 0``, then ``_iter`` advances."""
        if freq > 0 and self._iter % freq == 0:
            self._refresh_lagged()
        self._iter += 1

    def _refresh_lagged(self) -> None:
        refresh_lagged(self._group, self._g_old)
