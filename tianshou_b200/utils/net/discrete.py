"""Discrete-action actor / critic heads, IQN's quantile network, FQF's fraction proposal and full quantile function and Rainbow's
noisy layer and the intrinsic curiosity module (API of tianshou/utils/net/discrete.py:22-428)."""
from __future__ import annotations

from collections.abc import Sequence
from typing import Any

import numpy as np
import torch
import torch.nn.functional as F
from torch import nn

from ...data import Batch
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


class FractionProposalNetwork(nn.Module):
    """FQF's fraction proposal (discrete.py:219-252): ``Linear(embedding_dim, num_fractions)`` (Xavier-uniform weight at gain
    0.01, zero bias) on the trunk's features, read as the logits of a ``Categorical``.  ``forward`` returns ``taus [B, N + 1]``
    (0, then the cumulative sum of the probabilities), ``tau_hats [B, N]`` (the midpoints, detached) and the entropies ``[B]``."""

    def __init__(self, num_fractions: int, embedding_dim: int) -> None:
        super().__init__()
        self.net = nn.Linear(embedding_dim, num_fractions)
        torch.nn.init.xavier_uniform_(self.net.weight, gain=0.01)
        torch.nn.init.constant_(self.net.bias, 0)
        self.num_fractions = num_fractions
        self.embedding_dim = embedding_dim

    def forward(self, obs_embeddings: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        dist = torch.distributions.Categorical(logits=self.net(obs_embeddings))
        taus = F.pad(torch.cumsum(dist.probs, dim=1), (1, 0))
        tau_hats = (taus[:, :-1] + taus[:, 1:]).detach() / 2.0
        return taus, tau_hats, dist.entropy()


class FullQuantileFunction(ImplicitQuantileNetwork):
    """FQF's quantile network (discrete.py:255-314): IQN's network evaluated at the fractions a ``FractionProposalNetwork``
    proposes from the trunk's detached features.  ``forward`` returns ``((quantiles [B, actions, N] at tau_hats, fractions,
    quantiles_tau), hidden)`` with ``fractions = Batch(taus, tau_hats, entropies)`` (or the ``fractions`` passed in, whose
    ``tau_hats`` are then used); in training mode ``quantiles_tau [B, actions, N - 1]`` are the quantiles at ``taus[:, 1:-1]``,
    computed without gradient, else None."""

    def __init__(self, *, preprocess_net: ModuleWithVectorOutput, action_shape: Any, hidden_sizes: Sequence[int] = (),
                 num_cosines: int = 64) -> None:
        super().__init__(preprocess_net=preprocess_net, action_shape=action_shape, hidden_sizes=hidden_sizes,
                         num_cosines=num_cosines)

    def _compute_quantiles(self, obs: torch.Tensor, taus: torch.Tensor) -> torch.Tensor:
        B, S = taus.shape
        h = (obs.unsqueeze(1) * self.embed_model(taus)).view(B * S, -1)
        return self.last(h).view(B, S, -1).transpose(1, 2)

    def forward(self, obs: Any, propose_model: FractionProposalNetwork, fractions: Batch | None = None,  # type: ignore[override]
                **kwargs: Any) -> tuple[Any, Any]:
        feat, hidden = self.preprocess(obs, state=kwargs.get("state"))
        if fractions is None:
            taus, tau_hats, entropies = propose_model(feat.detach())
            fractions = Batch(taus=taus, tau_hats=tau_hats, entropies=entropies)
        else:
            taus, tau_hats = fractions.taus, fractions.tau_hats
        quantiles = self._compute_quantiles(feat, tau_hats)
        quantiles_tau = None
        if self.training:
            with torch.no_grad():
                quantiles_tau = self._compute_quantiles(feat, taus[:, 1:-1])
        return (quantiles, fractions, quantiles_tau), hidden


class NoisyLinear(nn.Module):
    """Noisy network layer with factorised Gaussian noise (arXiv:1706.10295, discrete.py:317-364).  In training mode ``forward``
    uses ``mu_W + sigma_W * ger(eps_q, eps_p)`` and ``mu_bias + sigma_bias * eps_q``, in eval mode ``mu_W`` and ``mu_bias``.
    ``eps_p [in]`` and ``eps_q [out]`` are parameters with ``requires_grad=False``, so they are in ``state_dict()`` and in an
    optimiser built from ``parameters()``; ``sample()`` redraws them in place as sign(x) sqrt|x| of ``torch.randn``, ``in``
    values then ``out``, on the module's device.  Initialised as the reference: mu uniform in +-1/sqrt(in), sigma
    ``noisy_std / sqrt(in)``, then one ``sample()``."""

    def __init__(self, in_features: int, out_features: int, noisy_std: float = 0.5) -> None:
        super().__init__()
        self.mu_W = nn.Parameter(torch.FloatTensor(out_features, in_features))
        self.sigma_W = nn.Parameter(torch.FloatTensor(out_features, in_features))
        self.mu_bias = nn.Parameter(torch.FloatTensor(out_features))
        self.sigma_bias = nn.Parameter(torch.FloatTensor(out_features))
        self.eps_p = nn.Parameter(torch.FloatTensor(in_features), requires_grad=False)
        self.eps_q = nn.Parameter(torch.FloatTensor(out_features), requires_grad=False)
        self.in_features = in_features
        self.out_features = out_features
        self.sigma = noisy_std
        self.reset()
        self.sample()

    def reset(self) -> None:
        bound = 1 / np.sqrt(self.in_features)
        self.mu_W.data.uniform_(-bound, bound)
        self.mu_bias.data.uniform_(-bound, bound)
        self.sigma_W.data.fill_(self.sigma / np.sqrt(self.in_features))
        self.sigma_bias.data.fill_(self.sigma / np.sqrt(self.in_features))

    def f(self, x: torch.Tensor) -> torch.Tensor:
        x = torch.randn(x.size(0), device=x.device)
        return x.sign().mul_(x.abs().sqrt_())

    def sample(self) -> None:
        """Redraw ``eps_p`` then ``eps_q`` in place (the device updates read these very tensors)."""
        self.eps_p.copy_(self.f(self.eps_p))
        self.eps_q.copy_(self.f(self.eps_q))

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if self.training:
            weight = self.mu_W + self.sigma_W * (self.eps_q.ger(self.eps_p))
            bias = self.mu_bias + self.sigma_bias * self.eps_q.clone()
        else:
            weight = self.mu_W
            bias = self.mu_bias
        return F.linear(x, weight, bias)


class IntrinsicCuriosityModule(nn.Module):
    """Intrinsic curiosity module (arXiv:1705.05363, discrete.py:377-428): a feature net, a forward model predicting the next
    state's features from ``[phi1 | one_hot(act)]`` and an inverse model predicting the action from ``[phi1 | phi2]``.  ``forward``
    is the reference's torch path; the wrappers of algorithm/modelbased/icm.py run the same computation on the device."""

    def __init__(self, *, feature_net: nn.Module, feature_dim: int, action_dim: int, hidden_sizes: Sequence[int] = ()) -> None:
        super().__init__()
        self.feature_net = feature_net
        self.forward_model = MLP(input_dim=feature_dim + action_dim, output_dim=feature_dim, hidden_sizes=hidden_sizes)
        self.inverse_model = MLP(input_dim=feature_dim * 2, output_dim=action_dim, hidden_sizes=hidden_sizes)
        self.feature_dim = feature_dim
        self.action_dim = action_dim

    def forward(self, s1: np.ndarray | torch.Tensor, act: np.ndarray | torch.Tensor, s2: np.ndarray | torch.Tensor,
                **kwargs: Any) -> tuple[torch.Tensor, torch.Tensor]:
        """s1, act, s2 -> (mse_loss, act_hat)."""
        device = next(self.parameters()).device
        s1 = torch.as_tensor(s1, dtype=torch.float32, device=device)
        s2 = torch.as_tensor(s2, dtype=torch.float32, device=device)
        phi1, phi2 = self.feature_net(s1), self.feature_net(s2)
        act = torch.as_tensor(act, dtype=torch.long, device=device)
        phi2_hat = self.forward_model(torch.cat([phi1, F.one_hot(act, num_classes=self.action_dim)], dim=1))
        mse_loss = 0.5 * F.mse_loss(phi2_hat, phi2, reduction="none").sum(1)
        act_hat = self.inverse_model(torch.cat([phi1, phi2], dim=1))
        return mse_loss, act_hat
