"""Soft Actor-Critic with the whole ``update()`` on the device (SURVEY 8(f) rank 2, BASELINE configs[3]).

Reference: tianshou/algorithm/modelfree/sac.py (SACPolicy :55-131, Alpha :133-215, SAC :218-336),
modelfree/td3.py:31-102 (dual critics, ``min`` target), modelfree/ddpg.py:196-339 (n-step target, critic
squared loss), utils/lagged_network.py:8-80 (Polyak).

Per ``update(buffer, sample_size)``:
  host : index draw (``buffer.sample_indices``: numpy RandomState streams, SURVEY A9 -- kept so the sampled
         transitions are the reference's), the two ``rsample`` noise draws (torch generator), one D2H of 3 loss scalars.
  GPU  : row gathers from the buffer's device mirror (or one upload of the sampled rows), target actor + lagged critics
         forward -> ``ts_sac_target`` -> ``ts_nstep_return``; per critic forward / loss / backward (``ts_net_gemm``) + Adam;
         actor forward, critics' input-gradient GEMMs (the second accumulating into the first), tanh-Gaussian head backward,
         actor backward + Adam; Polyak axpy.
Every Linear layer's forward / input gradient / weight gradient is one wgmma GEMM launch (csrc/net_gemm.cu).  The critic pair,
the row reads, the critic step and the n-step target are ``ContinuousTwinCritic``'s, shared with CQL and TD3; the actor forward
and the actor step are ``SquashedGaussianTwinCritic``'s, shared with CQL (imitation/cql.py); both stand on the twin-critic core
of twin_critic.py.
"""
from __future__ import annotations

from abc import ABC, abstractmethod
from copy import deepcopy
from dataclasses import dataclass
from typing import Any, Union

import numpy as np
import torch
from torch import nn
from torch.distributions import Independent, Normal

from ..._cabi import call, ptr, stream_ptr
from ...data import Batch, ReplayBuffer
from ..base import OffPolicyAlgorithm, Policy, TrainingStats
from ..flat_params import FlatGroup, UnsupportedModelError
from ..netgraph import ACT_NONE, _Layer, compile_sequential, module_layers
from ..optim import OptimizerFactory
from ..twin_critic import TwinCriticAlgorithm, per_weight, pop_batch_weight

SIGMA_MIN, SIGMA_MAX = -20.0, 2.0          # utils/net/continuous.py:17-18
_F32_EPS = float(np.finfo(np.float32).eps)


def correct_log_prob_gaussian_tanh(log_prob: torch.Tensor, tanh_squashed_action: torch.Tensor,
                                   eps: float = _F32_EPS) -> torch.Tensor:
    """Equation 21 of arXiv:1801.01290 (sac.py:25-39)."""
    return log_prob - torch.log(1 - tanh_squashed_action.pow(2) + eps).sum(-1, keepdim=True)


@dataclass(kw_only=True)
class SACTrainingStats(TrainingStats):
    actor_loss: float
    critic1_loss: float
    critic2_loss: float
    alpha: float | None = None
    alpha_loss: float | None = None


class SACPolicy(Policy):
    """Tanh-squashed Gaussian policy (sac.py:55-131).  ``forward`` is the torch-module path the Collector runs."""

    def __init__(self, *, actor: nn.Module, exploration_noise: Any = None, deterministic_eval: bool = True,
                 action_scaling: bool = True, action_space: Any, observation_space: Any | None = None) -> None:
        super().__init__(action_space=action_space, observation_space=observation_space, action_scaling=action_scaling,
                         action_bound_method=None)
        if exploration_noise == "default":
            raise UnsupportedModelError("exploration_noise='default' (GaussianNoise) is not provided; pass a callable or None")
        self.actor = actor
        self.exploration_noise = exploration_noise
        self.deterministic_eval = deterministic_eval

    def add_exploration_noise(self, act: Any, batch: Any) -> Any:
        if self.exploration_noise is None:
            return act
        if isinstance(act, np.ndarray):
            return act + self.exploration_noise(act.shape)
        return act

    def forward(self, batch: Batch, state: Any = None, **kwargs: Any) -> Batch:
        (loc, scale), hidden = self.actor(batch.obs, state=state, info=batch.get("info"))
        dist = Independent(Normal(loc=loc, scale=scale), 1)
        act = dist.mode if (self.deterministic_eval and not self.is_within_training_step) else dist.rsample()
        log_prob = dist.log_prob(act).unsqueeze(-1)
        squashed = torch.tanh(act)
        log_prob = correct_log_prob_gaussian_tanh(log_prob, squashed)
        return Batch(logits=(loc, scale), act=squashed, state=hidden, dist=dist, log_prob=log_prob)


class Alpha(ABC):
    """Entropy regularisation coefficient (sac.py:133-165)."""

    @staticmethod
    def from_float_or_instance(alpha: Union[float, "Alpha"]) -> "Alpha":
        if isinstance(alpha, float):
            return FixedAlpha(alpha)
        if isinstance(alpha, Alpha):
            return alpha
        raise ValueError(f"Expected float or Alpha instance, but got {alpha=}")

    @property
    @abstractmethod
    def value(self) -> float: ...

    @abstractmethod
    def update(self, entropy: torch.Tensor) -> float | None: ...


class FixedAlpha(Alpha):
    def __init__(self, alpha: float):
        self._value = alpha

    @property
    def value(self) -> float:
        return self._value

    def update(self, entropy: torch.Tensor) -> float | None:
        return None


class AutoAlpha(nn.Module, Alpha):
    """Auto-tuned alpha (sac.py:168-215): a single scalar parameter; its three-flop update stays in torch."""

    def __init__(self, target_entropy: float, log_alpha: float, optim: OptimizerFactory):
        super().__init__()
        self._target_entropy = target_entropy
        self._log_alpha = nn.Parameter(torch.tensor(log_alpha))
        self._optim, lr_scheduler = optim.create_instances(self)
        if lr_scheduler is not None:
            raise ValueError(f"Learning rate schedulers are not supported by {self.__class__.__name__}")

    @property
    def value(self) -> float:
        return self._log_alpha.detach().exp().item()

    def update(self, entropy: torch.Tensor) -> float:
        entropy_deficit = self._target_entropy - entropy.to(self._log_alpha.device)
        alpha_loss = -(self._log_alpha * entropy_deficit).mean()
        self._optim.zero_grad()
        alpha_loss.backward()
        self._optim.step()
        return alpha_loss.item()


# ------------------------------------------------------------------------------------------------ module -> kernel views
def _linear_relu_chain(mod: Any, in_dim: int, what: str) -> list[_Layer]:
    try:
        return compile_sequential(module_layers(mod), (in_dim,))
    except UnsupportedModelError as e:
        raise UnsupportedModelError(f"{what}: {e}") from e


def describe_q_critic(critic: Any, obs_dim: int, act_dim: int) -> tuple[list[_Layer], list[nn.Parameter]]:
    """ContinuousCritic(preprocess_net=Net(concat=True), ...) -> Linear/ReLU chain on concat(obs, act) ending in 1 output."""
    if getattr(critic, "apply_preprocess_net_to_obs_only", False):
        raise UnsupportedModelError("critic: apply_preprocess_net_to_obs_only unsupported")
    layers = _linear_relu_chain(critic.preprocess, obs_dim + act_dim, "critic.preprocess")
    if getattr(critic.preprocess, "softmax", False):
        raise UnsupportedModelError("critic: softmax trunk output unsupported")
    layers += _linear_relu_chain(critic.last, layers[-1].out_dim, "critic.last")
    if layers[-1].out_dim != 1 or layers[-1].act != ACT_NONE:
        raise UnsupportedModelError("critic must end in a single linear Q output")
    params: list[nn.Parameter] = []
    for L in layers:
        params += [L.weight, L.bias]
    return layers, params


def describe_gaussian_actor(actor: Any, obs_dim: int) -> tuple[list[_Layer], list[nn.Parameter], int]:
    """ContinuousActorProbabilistic(conditioned_sigma=True, unbounded=True): trunk + ONE virtual head layer whose rows are
    (mu.weight ; sigma.weight) -- adjacent in the flat buffer, so the head is a single [2A, H] GEMM."""
    if not getattr(actor, "_c_sigma", False):
        raise UnsupportedModelError("SAC actor: conditioned_sigma=True expected (examples/mujoco/mujoco_sac.py:97-104)")
    if not getattr(actor, "_unbounded", False):
        raise UnsupportedModelError("SAC actor: only unbounded=True (mu without tanh) is supported")
    trunk = _linear_relu_chain(actor.preprocess, obs_dim, "actor.preprocess")
    mu = _linear_relu_chain(actor.mu, trunk[-1].out_dim, "actor.mu")
    sg = _linear_relu_chain(actor.sigma, trunk[-1].out_dim, "actor.sigma")
    if len(mu) != 1 or len(sg) != 1 or mu[0].out_dim != sg[0].out_dim:
        raise UnsupportedModelError("SAC actor: mu / sigma heads must be single Linear layers of equal width")
    A = mu[0].out_dim
    params: list[nn.Parameter] = []
    for L in trunk:
        params += [L.weight, L.bias]
    params += [mu[0].weight, sg[0].weight, mu[0].bias, sg[0].bias]     # adjacency = the virtual [2A, H] layer
    head = _Layer("linear", mu[0].weight, mu[0].bias, ACT_NONE, mu[0].in_dim, 2 * A)
    return [*trunk, head], params, A


class ContinuousTwinCritic(TwinCriticAlgorithm):
    """What the continuous twin-critic algorithms (SAC, CQL, TD3, TD3+BC) share: two Q(s, a) critics on concat(obs, act), the
    row reads, the critics' squared-loss step and the n-step target.  The subclass supplies ``_describe_actor(actor, obs_dim)``
    (layer chain, parameters in flat order, action width) and, for the n-step target, ``_target_q``."""

    _cols_override: Any = None          # the mirror's columns while a graphed body runs (no cross-stream wait inside a capture)

    def _describe_actor(self, actor: nn.Module, obs_dim: int) -> tuple[list[_Layer], list[nn.Parameter], int]:
        raise NotImplementedError

    def _build_networks(self, *, lagged: tuple[nn.Module, nn.Module], policy_optim: OptimizerFactory,
                        critic_optim: OptimizerFactory, critic2_optim: OptimizerFactory | None,
                        max_grad_norm: float | None = None, lagged_actor: nn.Module | None = None) -> None:
        def describe_actor(actor: nn.Module) -> tuple[list[_Layer], list[nn.Parameter]]:
            self.obs_dim = int(module_layers(actor.preprocess)[0].in_features)
            layers, params, self.act_dim = self._describe_actor(actor, self.obs_dim)
            return layers, params

        self._build_twin_critic(describe_actor=describe_actor,
                                describe_critic=lambda net, _: describe_q_critic(net, self.obs_dim, self.act_dim), lagged=lagged,
                                policy_optim=policy_optim, critic_optim=critic_optim, critic2_optim=critic2_optim,
                                max_grad_norm=max_grad_norm, lagged_actor=lagged_actor)

    def _rows(self, buffer: ReplayBuffer, key: str, indices: np.ndarray | torch.Tensor) -> torch.Tensor:
        """buffer[key][indices] as a dense fp32 [I, width] device tensor: gathered from the device mirror when the
        buffer keeps one (no host traffic), else a host gather of the sampled rows + one upload."""
        from ... import ops
        return ops.buffer_rows(buffer, key, indices, self._dev, cols=self._cols_override)

    def _obs_next_rows(self, buffer: ReplayBuffer, indices: np.ndarray | torch.Tensor) -> torch.Tensor:
        """``buffer[indices].obs_next``: the stored column, or ``obs`` at ``buffer.next(indices)``."""
        if buffer._save_obs_next:
            obs_next = self._rows(buffer, "obs_next", indices)
        else:
            obs_next = self._rows(buffer, "obs", buffer.next(indices))
        return obs_next.contiguous()

    def _sample(self, buffer: ReplayBuffer, sample_size: int | None) -> tuple[Batch, Any]:
        """Indices from the buffer's host RNG streams (identical to the reference's draws); rows stay on the device."""
        indices = buffer.sample_indices(sample_size)
        batch = Batch()
        batch.__dict__["obs"] = self._rows(buffer, "obs", indices).contiguous()
        batch.__dict__["act"] = self._rows(buffer, "act", indices).contiguous()
        weight = per_weight(buffer, indices, self._dev)
        if weight is not None:
            batch.__dict__["weight"] = weight
        batch.__dict__["info"] = Batch()
        return batch, indices

    def _preprocess_batch(self, batch: Batch, buffer: ReplayBuffer, indices: np.ndarray) -> Batch:
        """The n-step return of ``_target_q`` into ``batch.returns`` (ddpg.py:287-302)."""
        return self.compute_nstep_return(batch=batch, buffer=buffer, indices=indices, target_q_fn=self._target_q,
                                         gamma=self.gamma, n_step=self.n_step_return_horizon)

    def _concat(self, obs: torch.Tensor, act: torch.Tensor, out: torch.Tensor) -> None:
        call("ts_concat2", ptr(obs), self.obs_dim, ptr(act), self.act_dim, obs.shape[0], ptr(out), stream_ptr(self._dev))

    def _q_pair(self, obs: torch.Tensor, act: torch.Tensor, tag: str, target: bool = False) -> list[list[torch.Tensor]]:
        """Both critics (or both lagged critics) on concat(obs, act): their activation lists."""
        B = obs.shape[0]
        x = self._buf(f"{tag}_x", (B, self.obs_dim + self.act_dim))
        self._concat(obs, act, x)
        return [self._lagged_forward(k, x, B, tag) if target else self._c[k].forward(x, B, tag) for k in range(2)]

    def _critic_step(self, k: int, x: torch.Tensor, returns: torch.Tensor, weight: torch.Tensor | None, optim: Any,
                     out_loss: torch.Tensor) -> torch.Tensor:
        """``_minimize_critic_squared_loss`` (ddpg.py:267-285) on the critic input x = concat(obs, act): forward, weighted
        MSE, backward, Adam."""
        B = x.shape[0]
        st = stream_ptr(self._dev)
        acts = self._c[k].forward(x, B, "cu")
        td = self._buf(f"td{k}", B)
        dq = self._buf("dq", (B, 1))
        rows = self._buf("loss_rows", B)
        call("ts_critic_mse", ptr(acts[-1]), ptr(returns), ptr(weight), B, ptr(td), ptr(dq), ptr(rows), st)
        call("ts_mean", ptr(rows), B, ptr(out_loss), st)
        self._c[k].backward(acts, dq, B, "cu")
        self._adam(self._g_c[k], optim._optim, optim._max_grad_norm)
        return td


class SquashedGaussianTwinCritic(ContinuousTwinCritic):
    """The tanh-squashed Gaussian actor SAC and CQL share: its description, its forward and SAC's actor step."""

    def _describe_actor(self, actor: nn.Module, obs_dim: int) -> tuple[list[_Layer], list[nn.Parameter], int]:
        return describe_gaussian_actor(actor, obs_dim)

    def _actor_forward(self, obs: torch.Tensor, tag: str) -> tuple[list[torch.Tensor], torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
        """policy(batch) on the device (sac.py:108-131): returns (activations, act, log_prob, sigma, noise)."""
        B, A = obs.shape[0], self.act_dim
        acts = self._actor.forward(obs, B, tag)
        noise = self._noise_fn((B, A)).to(self._dev, torch.float32).contiguous()
        act, logp, sigma = self._buf(tag + "_act", (B, A)), self._buf(tag + "_logp", B), self._buf(tag + "_sigma", (B, A))
        call("ts_squashed_gaussian", ptr(acts[-1]), 2 * A, ptr(noise), B, A, SIGMA_MIN, SIGMA_MAX, _F32_EPS, ptr(act), ptr(logp),
             ptr(sigma), stream_ptr(self._dev))
        return acts, act, logp, sigma, noise

    def _actor_step(self, obs: torch.Tensor, alpha: float, out_loss: torch.Tensor) -> torch.Tensor:
        """SAC's actor step against the current critics: L = mean(alpha * log pi(a|s) - min(Q1, Q2)(s, a)) with
        a = tanh(mu + sigma * eps) into ``out_loss``, backward through both critics' input gradients and the tanh-Gaussian
        head, Adam.  Returns log pi(a|s)."""
        B, A = obs.shape[0], self.act_dim
        st = stream_ptr(self._dev)
        a_acts, act, logp, sigma, noise = self._actor_forward(obs, "au")
        c_acts = self._q_pair(obs, act, "aq")
        dq1, dq2, rows = self._buf("adq1", (B, 1)), self._buf("adq2", (B, 1)), self._buf("actor_rows", B)
        call("ts_sac_actor_q_grad", ptr(c_acts[0][-1]), ptr(c_acts[1][-1]), ptr(logp), alpha, B, ptr(dq1), ptr(dq2), ptr(rows), st)
        call("ts_mean", ptr(rows), B, ptr(out_loss), st)
        cols = (self.obs_dim, self.obs_dim + A)
        dact = self._buf("dact", (B, A))            # d loss / d act of both critics, the second one accumulated
        for k, d in enumerate((dq1, dq2)):
            self._c[k].backward(c_acts[k], d, B, "aq", param_grads=False, input_grad=True, input_cols=cols, dx_out=dact,
                                dx_accumulate=k == 1)
        dhead = self._buf("dhead", (B, 2 * A))
        call("ts_squashed_gaussian_bwd", ptr(a_acts[-1]), 2 * A, ptr(noise), ptr(act), ptr(sigma), ptr(dact), B, A,
             SIGMA_MIN, SIGMA_MAX, _F32_EPS, alpha / B, ptr(dhead), st)
        self._actor.backward(a_acts, dhead, B, "au")
        self._adam(self._g_actor, self.policy_optim._optim, self.policy_optim._max_grad_norm)
        return logp


class SAC(SquashedGaussianTwinCritic, OffPolicyAlgorithm):
    """Soft Actor-Critic (arXiv:1801.01290 / 1812.05905), reference API (sac.py:218-336)."""

    def __init__(self, *, policy: SACPolicy, policy_optim: OptimizerFactory, critic: nn.Module, critic_optim: OptimizerFactory,
                 critic2: nn.Module | None = None, critic2_optim: OptimizerFactory | None = None, tau: float = 0.005,
                 gamma: float = 0.99, alpha: float | Alpha = 0.2, n_step_return_horizon: int = 1,
                 deterministic_eval: bool = True, cuda_graph: bool = False) -> None:
        assert 0.0 <= tau <= 1.0, f"tau should be in [0, 1] but got: {tau}"
        assert 0.0 <= gamma <= 1.0, f"gamma should be in [0, 1] but got: {gamma}"
        super().__init__(policy=policy)
        if _space_name(policy.action_space) != "continuous":
            raise ValueError(f"SACPolicy only supports Box action spaces, but got {policy.action_space=}.")
        self.tau = tau
        self.gamma = gamma
        self.n_step_return_horizon = n_step_return_horizon
        self.deterministic_eval = deterministic_eval
        self.alpha = Alpha.from_float_or_instance(alpha)
        self.critic = critic
        self.critic2 = critic2 or deepcopy(critic)
        self.critic_old = deepcopy(self.critic).eval()
        self.critic2_old = deepcopy(self.critic2).eval()
        self._build_networks(lagged=(self.critic_old, self.critic2_old), policy_optim=policy_optim, critic_optim=critic_optim,
                             critic2_optim=critic2_optim)
        # opt-in: the device work of one update() (~80 launches) captured once into a CUDA graph and replayed -- the eager call
        # sequence is Python-launch bound.  Needs a buffer with a device mirror, uniform replay and a fixed alpha.
        self.cuda_graph = bool(cuda_graph)
        self._graph: dict[str, Any] = {}
        # rsample noise source: torch's generator on the networks' device (what the reference draws when it runs there)
        dev = self._dev
        self._noise_fn = lambda shape: torch.normal(torch.zeros(shape, device=dev), torch.ones(shape, device=dev))

    # ------------------------------------------------------------------ target
    def _target_q(self, buffer: ReplayBuffer, indices: np.ndarray) -> torch.Tensor:
        """min(Q1', Q2')(s', a') - alpha * log pi(a'|s') with a' ~ pi(.|s')   (ddpg.py:327-339, td3.py:94-102, sac.py:298-302)"""
        obs_next = self._obs_next_rows(buffer, indices)
        B = obs_next.shape[0]
        _, act, logp, _, _ = self._actor_forward(obs_next, "tq")
        t_acts = self._q_pair(obs_next, act, "tq", target=True)
        out = self._buf("tq_out", (B, 1))
        call("ts_sac_target", ptr(t_acts[0][-1]), ptr(t_acts[1][-1]), ptr(logp), float(self.alpha.value), B, ptr(out),
             stream_ptr(self._dev))
        return out

    def _update_with_batch(self, batch: Batch) -> SACTrainingStats:
        dev = self._dev
        obs, act = batch.obs, batch.act
        B = obs.shape[0]
        returns = batch.returns.reshape(-1).to(dev, torch.float32).contiguous()
        weight = pop_batch_weight(batch, dev)
        losses = self._buf("losses", 3)
        x = self._buf("cu_x", (B, self.obs_dim + self.act_dim))
        self._concat(obs, act, x)
        td1 = self._critic_step(0, x, returns, weight, self.critic_optim, losses[0:1])
        td2 = self._critic_step(1, x, returns, weight, self.critic2_optim, losses[1:2])
        batch.weight = (td1 + td2) / 2.0       # prio-buffer

        logp = self._actor_step(obs, float(self.alpha.value), losses[2:3])
        alpha_loss = None if self._in_graph_body else self.alpha.update(-logp.detach().unsqueeze(-1))
        self._polyak()
        if self._in_graph_body:
            return None                         # the losses stay on the device; update() reads them after the replay
        l = losses.cpu().numpy()                # the only host sync of the update
        return SACTrainingStats(actor_loss=float(l[2]), critic1_loss=float(l[0]), critic2_loss=float(l[1]),
                                alpha=float(self.alpha.value), alpha_loss=alpha_loss)

    # ------------------------------------------------------------------ CUDA-graph mode
    _in_graph_body = False

    def _graph_usable(self, buffer: ReplayBuffer) -> bool:
        cols = buffer.device_columns() if hasattr(buffer, "device_columns") else None
        # (a learning-rate schedule would change a constant baked into the captured launches every update: eager then)
        return (self.cuda_graph and isinstance(self.alpha, FixedAlpha) and not hasattr(buffer, "update_weight") and cols is not None
                and not self.lr_schedulers
                and buffer._save_obs_next and all(k in cols for k in ("obs", "act", "rew", "terminated", "done", "obs_next")))

    def _device_body(self, buffer: ReplayBuffer, g: dict[str, Any]) -> None:
        """Everything of one update() after the index / noise draws, with no host synchronisation: n-step chain, target,
        both critic steps, the actor step, Polyak.  Runs eagerly once, then inside the capture, then as graph replays."""
        from ... import ops
        idx, meta, cols = g["idx"], g["meta"], g["cols"]
        noise_iter = iter((g["noise"][0], g["noise"][1]))
        saved_fn, self._noise_fn = self._noise_fn, lambda shape: next(noise_iter)
        saved_adam, self._adam = self._adam, FlatGroup.adam_step_device
        self._in_graph_body, self._cols_override = True, cols
        try:
            B = idx.numel()
            n = self.n_step_return_horizon
            stacked = ops.stack_next_indices(meta, idx, n)
            last = stacked[-1].contiguous()
            tq = self._target_q(buffer, last).reshape(B, -1).clone()
            ops.value_mask_rows(tq, cols["terminated"].view(torch.uint8), last)
            rew = cols["rew"] if cols["rew"].dtype == torch.float64 else cols["rew"].to(torch.float64)
            returns = ops.nstep_return(rew, ops.buffer_end_flags(meta), tq, stacked, self.gamma, n, out_dtype=torch.float64)
            batch = Batch()
            batch.__dict__["obs"] = self._rows(buffer, "obs", idx).contiguous()
            batch.__dict__["act"] = self._rows(buffer, "act", idx).contiguous()
            batch.__dict__["returns"] = returns.to(torch.float32)
            self._update_with_batch(batch)
            g["h_losses"].copy_(self._buf("losses", 3), non_blocking=True)
        finally:
            self._noise_fn, self._adam, self._in_graph_body, self._cols_override = saved_fn, saved_adam, False, None

    def update(self, buffer: ReplayBuffer, sample_size: int | None) -> TrainingStats:
        """``OffPolicyAlgorithm.update`` (algorithm_base.py:868-903); with ``cuda_graph=True`` the device work is one graph replay."""
        if buffer is None or not self.policy.is_within_training_step or not self._graph_usable(buffer):
            return super().update(buffer, sample_size)
        import time

        from ...ops import DeviceBufferMeta
        from ...utils.torch_utils import torch_train_mode
        start = time.time()
        dev = self._dev
        indices = np.asarray(buffer.sample_indices(sample_size), dtype=np.int64)
        B, A = len(indices), self.act_dim
        cols = buffer.device_columns()                       # also orders this stream after the mirror's pending copies
        E = int(buffer.buffer_num)
        g = self._graph
        key = (B, E, tuple(int(cols[k].data_ptr()) for k in sorted(cols)), float(self.policy_optim._optim.param_groups[0]["lr"]),
               float(self.critic_optim._optim.param_groups[0]["lr"]), float(self.critic2_optim._optim.param_groups[0]["lr"]))
        if g.get("key") != key:                              # (re)build the persistent inputs; the next call captures
            g.clear()
            g.update(key=key, calls=0, graph=None, cols=dict(cols),
                     h_idx=torch.empty(B, dtype=torch.int64, pin_memory=True), idx=torch.empty(B, dtype=torch.int64, device=dev),
                     h_meta=torch.empty((3, E), dtype=torch.int64, pin_memory=True), d_meta=torch.empty((3, E), dtype=torch.int64, device=dev),
                     noise=torch.empty((2, B, A), dtype=torch.float32, device=dev), h_losses=torch.empty(3, dtype=torch.float32, pin_memory=True))
            off = torch.from_numpy(np.asarray(buffer._extend_offset, dtype=np.int64)).to(dev)
            g["meta"] = DeviceBufferMeta(off, cols["done"].view(torch.uint8), g["d_meta"][0], g["d_meta"][1], g["d_meta"][2])
        g["h_idx"].numpy()[...] = indices
        hm = g["h_meta"].numpy()
        hm[0], hm[1], hm[2] = buffer.last_index, buffer._sizes, buffer._ins
        g["idx"].copy_(g["h_idx"], non_blocking=True)
        g["d_meta"].copy_(g["h_meta"], non_blocking=True)
        g["noise"][0].copy_(self._noise_fn((B, A)).to(dev, torch.float32))      # the two rsample draws, in the reference's order
        g["noise"][1].copy_(self._noise_fn((B, A)).to(dev, torch.float32))
        with torch_train_mode(self):
            if g["graph"] is not None:
                g["graph"].replay()
            elif g["calls"] == 0:                            # first update with these shapes: eager (allocates every scratch buffer)
                self._device_body(buffer, g)
            else:                                            # second: capture, then replay it as this update
                graph = torch.cuda.CUDAGraph()
                torch.cuda.synchronize(dev)
                with torch.cuda.graph(graph):
                    self._device_body(buffer, g)
                g["graph"] = graph
                graph.replay()
        g["calls"] += 1
        torch.cuda.current_stream(dev).synchronize()         # the one host sync: the three loss scalars
        l = g["h_losses"].numpy()
        for sched in self.lr_schedulers:
            sched.step()
        stat = SACTrainingStats(actor_loss=float(l[2]), critic1_loss=float(l[0]), critic2_loss=float(l[1]), alpha=float(self.alpha.value),
                                alpha_loss=None)
        stat.train_time = time.time() - start
        return stat


def _space_name(space: Any) -> str:
    from ..base import _space_kind
    return _space_kind(space)
