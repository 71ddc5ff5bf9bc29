"""Discrete-action actor / critic heads and IQN's quantile network (API of tianshou/utils/net/discrete.py:22-216)."""
from __future__ import annotations

from collections.abc import Sequence
from typing import Any

import numpy as np
import torch
import torch.nn.functional as F
from torch import nn

from .common import MLP, ModuleWithVectorOutput


def dist_fn_categorical_from_logits(logits: torch.Tensor) -> torch.distributions.Categorical:
    """Default distribution function for categorical actors (discrete.py:22-26)."""
    return torch.distributions.Categorical(logits=logits)


class DiscreteActor(ModuleWithVectorOutput):
    """preprocess net -> ``last`` MLP -> action values; probabilities when ``softmax_output``
    (discrete.py:29-92)."""

    def __init__(self, *, preprocess_net: ModuleWithVectorOutput, action_shape: Any,
                 hidden_sizes: Sequence[int] = (), softmax_output: bool = True) -> None:
        output_dim = int(np.prod(action_shape))
        super().__init__(output_dim)
        self.preprocess = preprocess_net
        self.last = MLP(input_dim=preprocess_net.get_output_dim(), output_dim=self.output_dim,
                        hidden_sizes=hidden_sizes)
        self.softmax_output = softmax_output

    def get_preprocess_net(self) -> ModuleWithVectorOutput:
        return self.preprocess

    def forward(self, obs: Any, state: Any = None, info: dict[str, Any] | None = None) -> tuple[torch.Tensor, Any]:
        x, hidden = self.preprocess(obs, state)
        x = self.last(x)
        if self.softmax_output:
            x = F.softmax(x, dim=-1)
        return x, hidden


class DiscreteCritic(ModuleWithVectorOutput):
    """V(s): preprocess net -> ``last`` MLP -> ``last_size`` (discrete.py:94-123)."""

    def __init__(self, *, preprocess_net: ModuleWithVectorOutput, hidden_sizes: Sequence[int] = (),
                 last_size: int = 1) -> None:
        super().__init__(output_dim=last_size)
        self.preprocess = preprocess_net
        self.last = MLP(input_dim=preprocess_net.get_output_dim(), output_dim=last_size, hidden_sizes=hidden_sizes)

    def forward(self, obs: Any, state: Any = None, info: dict[str, Any] | None = None) -> torch.Tensor:
        logits, _ = self.preprocess(obs, state=state)
        return self.last(logits)


class CosineEmbeddingNetwork(nn.Module):
    """Fractions ``taus [B, S]`` -> ``ReLU(Linear(num_cosines, embedding_dim)(cos(tau * pi * i)))`` for i = 1 .. num_cosines,
    shape ``[B, S, embedding_dim]`` (discrete.py:126-160).  ``pi * i`` is formed in the fractions' dtype, as ``np.pi`` times an
    arange of that dtype."""

    def __init__(self, num_cosines: int, embedding_dim: int) -> None:
        super().__init__()
        self.net = nn.Sequential(nn.Linear(num_cosines, embedding_dim), nn.ReLU())
        self.num_cosines = num_cosines
        self.embedding_dim = embedding_dim

    def forward(self, taus: torch.Tensor) -> torch.Tensor:
        B, S = taus.shape[0], taus.shape[1]
        i_pi = np.pi * torch.arange(1, self.num_cosines + 1, dtype=taus.dtype, device=taus.device)
        cos = torch.cos(taus.view(B, S, 1) * i_pi.view(1, 1, -1)).view(B * S, self.num_cosines)
        return self.net(cos).view(B, S, self.embedding_dim)


class ImplicitQuantileNetwork(DiscreteCritic):
    """IQN's quantile network (discrete.py:163-216): the preprocess net's features ``[B, D]`` times the cosine embedding of
    ``sample_size`` uniform fractions per row, then the ``last`` MLP on the ``B * sample_size`` products.  ``forward`` returns
    ``((q [B, actions, sample_size], taus [B, sample_size]), hidden)``; the fractions are drawn with ``torch.rand`` in the
    features' dtype on their device."""

    def __init__(self, *, preprocess_net: ModuleWithVectorOutput, action_shape: Any, hidden_sizes: Sequence[int] = (),
                 num_cosines: int = 64) -> None:
        super().__init__(preprocess_net=preprocess_net, hidden_sizes=hidden_sizes, last_size=int(np.prod(action_shape)))
        self.input_dim = preprocess_net.get_output_dim()
        self.embed_model = CosineEmbeddingNetwork(num_cosines, self.input_dim)

    def forward(self, obs: Any, sample_size: int, **kwargs: Any) -> tuple[Any, Any]:  # type: ignore[override]
        feat, hidden = self.preprocess(obs, state=kwargs.get("state"))
        B = feat.size(0)
        taus = torch.rand(B, sample_size, dtype=feat.dtype, device=feat.device)
        h = (feat.unsqueeze(1) * self.embed_model(taus)).view(B * sample_size, -1)
        q = self.last(h).view(B, sample_size, -1).transpose(1, 2)
        return (q, taus), hidden
