"""Rainbow DQN (arXiv:1710.02298) with ``update()`` on the device: C51 on noisy layers and dueling categorical heads.

Reference: tianshou/algorithm/modelfree/rainbow.py (RainbowDQN: C51 whose ``_update_with_batch`` first redraws the noise of the
online and then of the lagged network, whose lagged network is not held in eval mode), utils/net/discrete.py (``NoisyLinear``),
utils/net/common.py:300-369 (``Net(dueling_param=...)``), env/atari/atari_network.py:154-208 (``RainbowNet``),
utils/lagged_network.py:99-110 (the full lagged copy: every parameter, the noise included).

Per ``update(buffer, sample_size)``, in the reference's order:
  1. ``_sample_noise`` of the online network, then of the lagged one: ``NoisyLinear.sample()`` per noisy layer in
     ``modules()`` order, torch's ``randn`` on the model's device, written in place into the flat noise buffers the kernels read;
  2. the lagged tick (C51's), one device copy of the parameters and one of the noise: on a tick the lagged network's fresh
     noise is overwritten by the online network's;
  3. the target at s' (C51's ``ts_c51_target``), 4. the forward at s, 5. ``ts_c51_rows``, 6. ``ts_dueling_atoms_bwd``,
  7. the heads' and the trunk's backward GEMMs, 8. one Adam step, 9. one host read of the loss.
Every forward uses the train-mode weights ``mu + sigma * noise`` (``ts_noisy_weight``), as the reference runs its update in
train mode.  A dueling network is three chains on one flat group -- trunk, Q head (``A * N`` outputs), V head (``N``) -- combined
by ``ts_dueling_atoms`` into the ``[B, A, N]`` logits C51's kernels read; the trunk's input gradient is the Q head's plus the V
head's, in that order.  ``eps_p`` / ``eps_q`` stay out of the Adam group: the optimiser lists them, as the reference's does, and
never steps them.
"""
from __future__ import annotations

from copy import deepcopy
from dataclasses import dataclass
from typing import Any

import torch
from torch import nn

from ..._cabi import call, ptr, stream_ptr
from ...env.atari.atari_network import C51Net, RainbowNet
from ...utils.net.discrete import NoisyLinear
from ..discrete_q import dueling_atom_chains, lagged_group, refresh_lagged
from ..flat_params import FlatGroup, UnsupportedModelError
from ..netgraph import FusedStack, layer_params, noise_params
from ..optim import OptimizerFactory
from .c51 import C51, C51Policy
from .reinforce import LossSequenceTrainingStats


@dataclass(kw_only=True)
class RainbowTrainingStats:
    """rainbow.py's stats class; ``update()`` returns C51's ``LossSequenceTrainingStats``, as the reference's does."""

    loss: float


class RainbowDQN(C51):
    """Rainbow DQN, reference API and semantics (rainbow.py).

    ``policy.model`` is anything C51 reads, and its Linear layers may be ``NoisyLinear``; or a ``Net(softmax=True, num_atoms=N,
    dueling_param=...)`` or a ``RainbowNet`` (optionally behind ``ScaledObsInputActionReprNet``).  ``model_old`` is the plain
    lagged copy (``state_dict()`` keys ``model_old.*``).  ``_sample_noise(model)`` is the noise draw; replace it on the instance
    to inject noise."""

    def __init__(self, *, policy: C51Policy, optim: OptimizerFactory, gamma: float = 0.99, n_step_return_horizon: int = 1,
                 target_update_freq: int = 0) -> None:
        super().__init__(policy=policy, optim=optim, gamma=gamma, n_step_return_horizon=n_step_return_horizon,
                         target_update_freq=target_update_freq)

    def _build_network(self, policy: C51Policy, dev: torch.device) -> None:
        N = policy.num_atoms
        n_actions = int(policy.action_space.n)
        inner, in_shape, in_scale, chains = dueling_atom_chains(policy.model, n_actions, N)
        per_action_softmax = (isinstance(inner, (C51Net, RainbowNet)) and inner.num_atoms == N) or \
            (getattr(inner, "softmax", False) and getattr(inner, "num_atoms", 1) == N)
        if not per_action_softmax:
            raise UnsupportedModelError(f"RainbowDQN reads the network output as probabilities over {N} atoms per action: build "
                                        f"Net(softmax=True, num_atoms={N}), C51Net or RainbowNet(num_atoms={N}), got "
                                        f"{type(inner).__name__} without that softmax")
        self._init_discrete(dev, in_shape, in_scale, n_actions)
        layers = [L for c in chains for L in c]
        self._group = FlatGroup(layer_params(layers), dev)
        self._eps = FlatGroup(noise_params(layers), dev)
        self._eps_old: FlatGroup | None = None
        names = ("trunk", "q", "v") if len(chains) == 3 else ("rainbow",)
        stacks = [FusedStack(c, self._group, n, noise=self._eps) for c, n in zip(chains, names)]
        self._net, self._q, self._v = (stacks[0], None, None) if len(stacks) == 1 else stacks

    def _frozen_params(self) -> tuple[nn.Parameter, ...]:
        return tuple(self._eps.params)

    def _build_lagged(self, policy: C51Policy) -> None:
        """The lagged copy, unwrapped (rainbow.py: its noise must be drawn in train mode), its parameters and noise on flat
        buffers of the online layout."""
        self.model_old = deepcopy(policy.model)
        chains = dueling_atom_chains(self.model_old, self.n_actions, policy.num_atoms)[3]
        layers = [L for c in chains for L in c]
        self._g_old = lagged_group(self._group, layer_params(layers))
        self._eps_old = lagged_group(self._eps, noise_params(layers))

    def _refresh_lagged(self) -> None:
        """``full_parameter_update`` copies every parameter, the noise included (lagged_network.py:99-110)."""
        refresh_lagged(self._group, self._g_old)
        refresh_lagged(self._eps, self._eps_old)

    @staticmethod
    def _sample_noise(model: nn.Module) -> bool:
        """Redraw the noise of every ``NoisyLinear`` of ``model`` in ``modules()`` order; True if there was one."""
        sampled_any_noise = False
        for m in model.modules():
            if isinstance(m, NoisyLinear):
                m.sample()
                sampled_any_noise = True
        return sampled_any_noise

    # ------------------------------------------------------------------ network
    def _logits(self, src: Any, tag: str, lagged: bool = False) -> tuple[torch.Tensor, Any]:
        params = noise = None
        if lagged:
            self._g_old.ensure_adopted()
            self._eps_old.ensure_adopted()
            params, noise = self._g_old.flat, self._eps_old.flat
        B = src.rows
        if self._v is None:
            acts = self._net.forward(src.x, B, tag, frames=src.frames, params=params, noise=noise)
            return acts[-1], acts
        at = self._net.forward(src.x, B, tag, frames=src.frames, params=params, noise=noise)
        aq = self._q.forward(at[-1], B, tag, params=params, noise=noise)
        av = self._v.forward(at[-1], B, tag, params=params, noise=noise)
        A, N = self.n_actions, self.policy.num_atoms
        logits = self._buf(f"logits_{tag}", (B, A * N))
        call("ts_dueling_atoms", ptr(aq[-1]), ptr(av[-1]), B, A, N, ptr(logits), stream_ptr(self._dev))
        return logits, (at, aq, av)

    def _backward(self, acts: Any, dlogits: torch.Tensor, rows: int) -> None:
        if self._v is None:
            self._net.backward(acts, dlogits, rows, "up")
            return
        at, aq, av = acts
        A, N = self.n_actions, self.policy.num_atoms
        dq, dv = self._buf("dq", (rows, A * N)), self._buf("dv", (rows, N))
        call("ts_dueling_atoms_bwd", ptr(dlogits), rows, A, N, ptr(dq), ptr(dv), stream_ptr(self._dev))
        # d loss / d trunk output = the Q head's input gradient + the V head's, masked by the trunk's last activation
        h = at[-1]
        dh = self._buf("dh", tuple(h.shape))
        trunk_act = (self._net._producer_act(len(self._net.layers)), h)
        self._q.backward(aq, dq, rows, "up", input_grad=True, input_act=trunk_act, dx_out=dh)
        self._v.backward(av, dv, rows, "up", input_grad=True, input_act=trunk_act, dx_out=dh, dx_accumulate=True)
        self._net.backward(at, dh, rows, "up", dy_preact=True)

    # ------------------------------------------------------------------ update
    def _update_with_batch(self, batch: Any) -> LossSequenceTrainingStats:
        self._sample_noise(self.policy.model)
        if self.use_target_network:
            self._sample_noise(self.model_old)
        return super()._update_with_batch(batch)
