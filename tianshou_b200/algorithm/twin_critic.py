"""What the twin-critic algorithms (SAC, discrete SAC, CQL, TD3, TD3+BC) share: one actor (with an optional lagged copy) and
two (critic, lagged critic) pairs as flat groups on one CUDA device, their three optimisers, the scratch, the one Adam seam,
the lagged forwards and Polyak; plus the sampling helpers the off-policy algorithms share with DQN.

Reference: modelfree/td3.py:40-92 (dual critics, ``critic2=None`` deep-copies the critic), :183 (TD3's lagged actor),
utils/lagged_network.py:8-80 (Polyak, the lagged copy under ``.module``), data/buffer/prio.py:104-106 (the importance weight of
a prioritised sample).
"""
from __future__ import annotations

from collections.abc import Callable
from typing import Any

import numpy as np
import torch
from torch import nn

from .._cabi import to_device
from ..data import Batch, ReplayBuffer
from .base import Algorithm
from .flat_params import DeviceScratch, FlatGroup, UnsupportedModelError, bind_optimizer
from .netgraph import FusedStack, _Layer, polyak_update
from .obs_source import DeviceObsSource
from .optim import OptimizerFactory

Describe = Callable[..., tuple[list[_Layer], list[nn.Parameter]]]


def cuda_device_of(*nets: nn.Module) -> torch.device:
    """The one CUDA device all parameters of ``nets`` live on; anything else is refused."""
    devs = {p.device for net in nets for p in net.parameters()}
    if len(devs) != 1 or next(iter(devs)).type != "cuda":
        raise UnsupportedModelError(f"networks live on {sorted(map(str, devs))}; tianshou_b200 has no CPU path -- move them to "
                                    "one CUDA device")
    return next(iter(devs))


def per_weight(buffer: ReplayBuffer, indices: np.ndarray, device: torch.device) -> torch.Tensor | None:
    """The importance weight ``PrioritizedReplayBuffer.__getitem__`` adds to a sample, as fp32 on ``device``; None for a
    uniform buffer."""
    if not hasattr(buffer, "get_weight"):
        return None
    w = buffer.get_weight(indices)
    return to_device(np.asarray(w / np.max(w) if buffer._weight_norm else w, dtype=np.float32), device)


def pop_batch_weight(batch: Batch, device: torch.device) -> torch.Tensor | None:
    """``batch.weight`` removed from the batch, as a flat contiguous fp32 tensor on ``device`` (None when it has none)."""
    weight = batch.__dict__.pop("weight", None)
    if weight is None:
        return None
    if not isinstance(weight, torch.Tensor):
        weight = to_device(np.asarray(weight, dtype=np.float32), device)
    return weight.reshape(-1).to(device, torch.float32).contiguous()


def sample_discrete(buffer: ReplayBuffer, sample_size: int | None, obs_source: Callable[..., DeviceObsSource],
                    device: torch.device) -> tuple[Batch, Any]:
    """Indices from the buffer's host RNG streams (identical to the reference's draws); the observations as
    ``obs_source(buffer, indices, "obs")`` reads them on the device, the actions as int64 device rows, the importance weight
    of a prioritised buffer."""
    indices = buffer.sample_indices(sample_size)
    batch = Batch()
    batch.__dict__["obs"] = obs_source(buffer, indices, "obs")
    act = np.asarray(buffer.act)[indices]
    batch.__dict__["act"] = to_device(np.ascontiguousarray(act.reshape(-1)).astype(np.int64), device)
    weight = per_weight(buffer, indices, device)
    if weight is not None:
        batch.__dict__["weight"] = weight
    batch.__dict__["info"] = Batch()
    return batch, indices


class _EvalModeModule(nn.Module):
    """A lagged network as the reference holds it (utils/lagged_network.py:21-41): the copy under ``.module``, always in eval
    mode, so ``state_dict()`` has the reference's ``critic_old.module.*`` keys."""

    def __init__(self, module: nn.Module) -> None:
        super().__init__()
        self.module = module.eval()

    def train(self, mode: bool = True) -> "_EvalModeModule":
        super().train(False)
        return self

    def forward(self, *args: Any, **kwargs: Any) -> Any:
        return self.module(*args, **kwargs)


def _group_adam_step(group: FlatGroup, optimizer: torch.optim.Optimizer, max_grad_norm: float | None) -> None:
    """The default Adam seam: the group's own ``adam_step``, looked up on the instance, so a step replaced on one group (to
    record its gradient, say) is the one the update takes."""
    group.adam_step(optimizer, max_grad_norm)


class TwinCriticAlgorithm(Algorithm):
    """An actor and two critics with a lagged copy each (and optionally a lagged actor), stepped on the device.  The subclass
    assigns ``critic``, ``critic2``, their lagged modules ``critic_old`` / ``critic2_old`` and ``tau``, then calls
    ``_build_twin_critic``."""

    def _build_twin_critic(self, *, describe_actor: Describe, describe_critic: Describe, lagged: tuple[nn.Module, nn.Module],
                           policy_optim: OptimizerFactory, critic_optim: OptimizerFactory,
                           critic2_optim: OptimizerFactory | None, max_grad_norm: float | None = None,
                           lagged_actor: nn.Module | None = None) -> None:
        """``describe_actor(actor)`` and ``describe_critic(net, role)`` return (layer chain, parameters in flat order);
        ``lagged`` are the lagged critics as ``describe_critic`` reads them, ``lagged_actor`` (None: there is none) the lagged
        actor as ``describe_actor`` reads it.  ``critic2_optim`` defaults to ``critic_optim``; ``max_grad_norm`` clips both
        critics' steps."""
        dev = self._dev = cuda_device_of(self.policy.actor, self.critic, self.critic2)
        a_layers, a_params = describe_actor(self.policy.actor)
        self._g_actor = FlatGroup(a_params, dev)
        self._actor = FusedStack(a_layers, self._g_actor, "actor")
        self._g_at = None if lagged_actor is None else FlatGroup(describe_actor(lagged_actor)[1], dev)
        self._g_c, self._c, self._g_ct = [], [], []
        for name, src, tgt in (("critic", self.critic, lagged[0]), ("critic2", self.critic2, lagged[1])):
            layers, params = describe_critic(src, name)
            _, tparams = describe_critic(tgt, name)
            g = FlatGroup(params, dev)
            self._g_c.append(g)
            self._c.append(FusedStack(layers, g, name))
            self._g_ct.append(FlatGroup(tparams, dev))
        self.policy_optim = self._create_optimizer(self.policy, policy_optim)
        self.critic_optim = self._create_optimizer(self.critic, critic_optim, max_grad_norm=max_grad_norm)
        self.critic2_optim = self._create_optimizer(self.critic2, critic2_optim or critic_optim, max_grad_norm=max_grad_norm)
        for o, g in ((self.policy_optim, self._g_actor), (self.critic_optim, self._g_c[0]), (self.critic2_optim, self._g_c[1])):
            bind_optimizer(o, g)
        self._scratch = DeviceScratch(dev)
        self._buf = self._scratch.tensor
        self._adam = _group_adam_step           # every Adam step of the update: ``self._adam(group, torch_optimizer, max_grad_norm)``

    def _lagged_forward(self, k: int, x: torch.Tensor | None, rows: int, tag: str, frames: tuple | None = None) -> list[torch.Tensor]:
        """Lagged critic ``k`` on ``x`` (or ``frames``): its activation list."""
        self._g_ct[k].ensure_adopted()
        return self._c[k].forward(x, rows, tag, frames=frames, params=self._g_ct[k].flat)

    def _lagged_actor_forward(self, x: torch.Tensor, rows: int, tag: str) -> list[torch.Tensor]:
        """The lagged actor on ``x``: its activation list."""
        self._g_at.ensure_adopted()
        return self._actor.forward(x, rows, tag, params=self._g_at.flat)

    def _polyak(self) -> None:
        """``_update_lagged_network_weights``: both lagged critics (and the lagged actor, when there is one) toward their
        networks by ``tau``."""
        for k in range(2):
            polyak_update(self._g_ct[k], self._g_c[k], self.tau)
        if self._g_at is not None:
            polyak_update(self._g_at, self._g_actor, self.tau)
