"""Two ``DiscreteActor`` / ``DiscreteCritic`` heads on ONE preprocess network, stepped by one optimiser over one loss: the trunk
runs once, both ``last`` chains run on its output, and the trunk's gradient is the sum of what comes down from both heads.

Reference: every use of discrete BCQ and discrete CRR (examples/offline/atari_bcq.py:104-122, atari_crr.py:105-124,
test/offline/test_discrete_bcq.py:73-86, test_discrete_crr.py:69-84) builds both networks on one ``DQNet(features_only=True)`` or
one ``Net``; utils/net/discrete.py:29-123 (preprocess net, then the ``last`` MLP).  Two networks that share nothing are the same
thing without a trunk: two full chains in the same flat group.
"""
from __future__ import annotations

from typing import Any, NamedTuple

import torch
from torch import nn

from .flat_params import FlatGroup, UnsupportedModelError
from .modelfree.dqn import describe_q_network
from .netgraph import ACT_NONE, FusedStack, _Layer, compile_sequential, module_layers, _out_shape
from .obs_source import DeviceObsSource


class TwoHeadActs(NamedTuple):
    """Activation lists of one ``TwoHeadNetwork.forward``: the trunk's (None without a shared trunk) and each head's (None for
    a head that was not asked for).  ``a[-1]`` / ``b[-1]`` are the heads' outputs ``[rows, outputs]``."""

    trunk: list[torch.Tensor] | None
    a: list[torch.Tensor] | None
    b: list[torch.Tensor] | None


def two_head_parameters(a: nn.Module, b: nn.Module) -> list[nn.Parameter]:
    """``a.parameters()`` then ``b.parameters()``, a shared parameter once: the order torch gives an optimiser built over a
    module that holds ``a`` before ``b``."""
    seen: set[int] = set()
    out = []
    for p in [*a.parameters(), *b.parameters()]:
        if id(p) not in seen:
            seen.add(id(p))
            out.append(p)
    return out


def _parts(net: Any, role: str) -> tuple[Any, Any, tuple[int, ...], float]:
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


def _layer_params(layers: list[_Layer]) -> list[nn.Parameter]:
    return [p for L in layers if L.weight is not None for p in (L.weight, L.bias)]


class TwoHeadNetwork:
    """Heads ``a`` and ``b`` (each ``preprocess`` + ``last``) in one ``FlatGroup`` built over ``two_head_parameters(a, b)``.
    ``shared``: both hold the same preprocess parameters, so the trunk is compiled and evaluated once."""

    def __init__(self, a: nn.Module, b: nn.Module, group: FlatGroup, roles: tuple[str, str] = ("a", "b")) -> None:
        self.group = group
        self.device = group.device
        pre_a, last_a, shape, scale = _parts(a, roles[0])
        pre_b, last_b, shape_b, scale_b = _parts(b, roles[1])
        ids_a, ids_b = {id(p) for p in a.preprocess.parameters()}, {id(p) for p in b.preprocess.parameters()}
        own_a, own_b = {id(p) for p in a.parameters()}, {id(p) for p in b.parameters()}
        self.shared = bool(ids_a) and ids_a == ids_b
        if (own_a & own_b) != (ids_a if self.shared else set()):
            raise UnsupportedModelError(f"{roles[0]} and {roles[1]} share some parameters but not one whole preprocess network; "
                                        "share the preprocess network or nothing")
        if (shape, scale) != (shape_b, scale_b):
            raise UnsupportedModelError(f"{roles[1]} reads the observation as shape {shape_b} / denominator {scale_b}, {roles[0]} "
                                        f"as {shape} / {scale}: the networks must read it the same way")
        self.in_shape, self.in_scale = shape, scale
        try:
            if self.shared:
                trunk = compile_sequential(module_layers(pre_a), shape)
                if not trunk:
                    raise UnsupportedModelError("the shared preprocess network has no layers")
                feat = _out_shape(trunk, shape)
                chains = [compile_sequential(module_layers(last), feat) for last in (last_a, last_b)]
            else:
                trunk = []
                chains = [compile_sequential(module_layers(pre) + module_layers(last), shape)
                          for pre, last in ((pre_a, last_a), (pre_b, last_b))]
        except UnsupportedModelError as e:
            raise UnsupportedModelError(f"{roles[0]} / {roles[1]}: {e}") from e
        for role, chain in zip(roles, chains):
            if not chain or chain[-1].kind != "linear" or chain[-1].act != ACT_NONE:
                raise UnsupportedModelError(f"{role}: must end in a linear layer (with a bias, without activation) over its outputs")
            if chain[0].kind != "linear" and self.shared:
                raise UnsupportedModelError(f"{role}: the head on a shared trunk must start with a linear layer")
        covered = {id(p) for p in _layer_params(trunk + chains[0] + chains[1])}
        if covered != {id(p) for p in group.params}:
            raise UnsupportedModelError("the flat group's parameters differ from the parameters of the compiled layers")
        self.n_out = (chains[0][-1].out_dim, chains[1][-1].out_dim)
        self._trunk = FusedStack(trunk, group, "trunk") if self.shared else None
        self._heads = (FusedStack(chains[0], group, roles[0]), FusedStack(chains[1], group, roles[1]))
        # what the heads' input gradient still has to be multiplied by: the derivative of the activation that produced the trunk's
        # output.  A trunk ending in Flatten applies its producer's ReLU mask in its own backward.
        self._trunk_act = ACT_NONE
        if self.shared and trunk[-1].kind != "flatten":
            self._trunk_act = trunk[-1].act

    # ------------------------------------------------------------------ forward
    def forward(self, src: DeviceObsSource, tag: str, params: torch.Tensor | None = None,
                heads: tuple[bool, bool] = (True, True)) -> TwoHeadActs:
        """The trunk once on ``src`` (dense rows or the frame source of the first convolution), then the asked-for heads on its
        output; ``params``: another flat buffer of the group's layout (the lagged copy)."""
        rows = src.rows
        if not self.shared:
            out = [h.forward(src.x, rows, tag, frames=src.frames, params=params) if want else None
                   for h, want in zip(self._heads, heads)]
            return TwoHeadActs(None, out[0], out[1])
        t = self._trunk.forward(src.x, rows, tag, frames=src.frames, params=params)
        out = [h.forward(t[-1], rows, tag, params=params) if want else None for h, want in zip(self._heads, heads)]
        return TwoHeadActs(t, out[0], out[1])

    # ------------------------------------------------------------------ backward
    def backward(self, acts: TwoHeadActs, d_a: torch.Tensor, d_b: torch.Tensor, tag: str) -> None:
        """Every parameter's gradient of the loss whose gradients w.r.t. the two head outputs are ``d_a`` / ``d_b``, stored into
        the group's gradient buffer: head a writes its input gradient, head b adds its own into the same buffer, the trunk runs
        backward once on the sum."""
        rows = d_a.shape[0]
        ha, hb = self._heads
        if not self.shared:
            ha.backward(acts.a, d_a, rows, tag)
            hb.backward(acts.b, d_b, rows, tag)
            return
        feat = acts.trunk[-1]
        dfeat = self._trunk._buf((tag, "dfeat"), feat.numel())[: feat.numel()].view(feat.shape)
        input_act = (self._trunk_act, feat) if self._trunk_act != ACT_NONE else None
        ha.backward(acts.a, d_a, rows, tag, input_grad=True, input_act=input_act, dx_out=dfeat)
        hb.backward(acts.b, d_b, rows, tag, input_grad=True, input_act=input_act, dx_out=dfeat, dx_accumulate=True)
        self._trunk.backward(acts.trunk, dfeat, rows, tag, dy_preact=True)
