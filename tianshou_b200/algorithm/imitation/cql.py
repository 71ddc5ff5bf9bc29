"""Conservative Q-learning (arXiv:2006.04779, CalQL calibration arXiv:2303.05479) with the whole ``update()`` on the device.

Reference: tianshou/algorithm/imitation/cql.py (CQLTrainingStats :23-28, CQL :32-400), algorithm_base.py:906-951
(OfflineAlgorithm), modelfree/sac.py (SACPolicy, Alpha), utils/lagged_network.py:8-80 (Polyak).

Per ``update(buffer, sample_size)``:
  host : index draw (numpy RandomState streams -- the reference's transitions), the four ``rsample`` draws through ``_noise_fn``
         (actor step, target, current-pi, next-pi), the ``uniform_`` draw of the random actions on torch's CPU generator between
         the target and the current-pi draw (where the reference makes it), one D2H of the losses at the end.
  GPU  : row gathers (device mirror or one upload); actor forward -> ``ts_squashed_gaussian`` -> both critics -> actor backward
         -> Adam; the alpha update; actor + lagged critics on s' -> ``ts_cql_target``; actor on the repeated s and s' (B * R rows
         each); ONE forward per critic over [data B | random N | current-pi N | next-pi N] rows (``ts_concat2``) ->
         ``ts_cql_rows`` (both critics) -> ``ts_cql_losses`` -> Lagrange multiplier Adam -> per critic one parameter-gradient
         backward + clipped Adam; Polyak.
The gradients the reference computes and then discards (the critic losses into the actor through the pi actions, the
multiplier's loss into the critics) are zeroed by each ``Optimizer.step`` before use, so they are not computed here.
"""
from __future__ import annotations

from copy import deepcopy
from dataclasses import dataclass
from typing import Any

import numpy as np
import torch
from torch import nn

from ..._cabi import call, ptr, stream_ptr
from ...data import Batch, ReplayBuffer
from ..base import OfflineAlgorithm
from ..flat_params import FlatGroup
from ..modelfree.sac import Alpha, ContinuousTwinCritic, SACPolicy, SACTrainingStats
from ..optim import OptimizerFactory


@dataclass(kw_only=True)
class CQLTrainingStats(SACTrainingStats):
    """Loss statistics of the CQL learn step (cql.py:23-28)."""

    cql_alpha: float | None = None
    cql_alpha_loss: float | None = None


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


class CQL(ContinuousTwinCritic, OfflineAlgorithm):
    """Conservative Q-learning (arXiv:2006.04779), reference API and semantics (cql.py:32-400).

    The update reproduces what ``CQL._update_with_batch`` computes:

    * the actor step first (SAC's actor loss against the current critics), then ``alpha.update``; the target and both pi-value
      blocks use the updated actor and alpha; the critic steps last, then Polyak;
    * the target is ``rew + logical_not(done) * gamma * (min(Q1', Q2')(s', a') - alpha log pi(a'|s'))``: one step, ``done``
      (terminated or truncated), plain MSE without importance weights;
    * the random actions are ``torch.FloatTensor(B * R, A).uniform_(-min_action, max_action)`` on torch's CPU generator, as in
      the reference (with the defaults every random action is exactly 1.0);
    * the next-pi block evaluates the critics on the repeated ``obs``, not ``obs_next``;
    * the penalty is ``mean_i logsumexp_j(v_ij / T) * w * T - mean(Q(s, a)) * w`` where the log-sum-exp runs over the THREE
      values (random, current-pi, next-pi) of each of the B * R rows: the reference concatenates three (B * R, 1) blocks along
      dim 1;
    * calibrated: each block value is ``max(value, calibration return)``, half the gradient to each side at a tie.

    ``process_buffer`` stores the Monte-Carlo returns of ``buffer.sample(0)`` POSITIONALLY, as the reference does: element i of
    the sampled order goes to slot i of ``calibration_returns``; in a buffer that has wrapped around this is not the return of
    slot i itself.

    The Lagrange multiplier (``with_lagrange``): ``cql_alpha = clamp(exp(cql_log_alpha), alpha_min, alpha_max)`` scales both
    penalties, ``cql_alpha_loss = -0.5 (c1 + c2)`` takes one ``torch.optim.Adam(lr=cql_alpha_lr)`` step on ``cql_log_alpha``
    (an fp32 one-element Adam on the device with torch's defaults; the clamp passes the gradient inside its bounds).  This is
    the behaviour of the reference on the CPU.  On a CUDA device the reference's multiplier never moves: its
    ``cql_log_alpha.to(device)`` is a non-leaf copy that its optimiser does not hold, so ``cql_alpha`` stays ``clamp(1, ...)``
    there.  This implementation trains the multiplier wherever it runs.  As in the reference, ``cql_log_alpha`` and
    ``cql_alpha_optim`` are not part of ``state_dict()``: carry them over by hand (``cql_log_alpha.data.copy_(...)`` and
    ``cql_alpha_optim.load_state_dict(...)``).

    With a fixed alpha the update synchronises with the host once, to read the losses at its end (``AutoAlpha`` reads its
    value and loss as in SAC).
    """

    def __init__(self, *, policy: SACPolicy, policy_optim: OptimizerFactory, critic: nn.Module, critic_optim: OptimizerFactory,
                 critic2: nn.Module | None = None, critic2_optim: OptimizerFactory | None = None, cql_alpha_lr: float = 1e-4,
                 cql_weight: float = 1.0, tau: float = 0.005, gamma: float = 0.99, alpha: float | Alpha = 0.2,
                 temperature: float = 1.0, with_lagrange: bool = True, lagrange_threshold: float = 10.0, min_action: float = -1.0,
                 max_action: float = 1.0, num_repeat_actions: int = 10, alpha_min: float = 0.0, alpha_max: float = 1e6,
                 max_grad_norm: float = 1.0, calibrated: bool = True) -> None:
        super().__init__(policy=policy)
        self.tau = tau
        self.critic = critic
        self.critic2 = critic2 or deepcopy(critic)
        self.critic_old = _EvalModeModule(deepcopy(self.critic))
        self.critic2_old = _EvalModeModule(deepcopy(self.critic2))
        self.gamma = gamma
        self.alpha = Alpha.from_float_or_instance(alpha)
        self.temperature = temperature
        self.with_lagrange = with_lagrange
        self.lagrange_threshold = lagrange_threshold
        self.cql_weight = cql_weight
        self.min_action = min_action
        self.max_action = max_action
        self.num_repeat_actions = num_repeat_actions
        self.alpha_min = alpha_min
        self.alpha_max = alpha_max
        self.calibrated = calibrated
        if int(num_repeat_actions) < 1:
            raise ValueError(f"num_repeat_actions must be at least 1, got {num_repeat_actions}")
        self._build_networks(lagged=(self.critic_old.module, self.critic2_old.module), policy_optim=policy_optim,
                             critic_optim=critic_optim, critic2_optim=critic2_optim, max_grad_norm=max_grad_norm)
        dev = self._dev
        # the Lagrange multiplier: a plain tensor (not a module attribute, so not in state_dict(), as in the reference) whose
        # storage is a one-element flat group on the device
        self.cql_log_alpha = torch.tensor([0.0], requires_grad=True)
        self.cql_alpha_optim = torch.optim.Adam([self.cql_log_alpha], lr=cql_alpha_lr)
        self._g_la = FlatGroup([self.cql_log_alpha], dev)
        self._g_la.export_state(self.cql_alpha_optim)
        # rsample noise source: torch's generator on the networks' device, the standard-normal draw Normal.rsample makes there
        # (randn: no host-side validity check, so no synchronisation)
        self._noise_fn = lambda shape: torch.randn(shape, device=dev)

    # ------------------------------------------------------------------ helpers
    def _repeat_rows(self, x: torch.Tensor, R: int, tag: str) -> torch.Tensor:
        """x.unsqueeze(1).repeat(1, R, 1).view(B * R, -1) (cql.py:309-313): row b * R + j is x[b]."""
        from ... import ops
        B = x.shape[0]
        idx = self._scratch.get("rep_idx")
        if idx is None or idx.numel() != B * R or self._scratch.get("rep_R") != R:
            idx = self._scratch["rep_idx"] = torch.arange(B * R, device=self._dev) // R
            self._scratch["rep_R"] = R
        return ops.gather_rows(x, idx, out=self._buf(tag, (B * R, x.shape[1])))

    # ------------------------------------------------------------------ buffer
    def process_buffer(self, buffer: ReplayBuffer) -> ReplayBuffer:
        """``calibrated``: the Monte-Carlo returns of ``buffer.sample(0)`` (``compute_episodic_return`` with ``gae_lambda=1``,
        ``ts_gae`` on the device) become the ``_meta`` key ``calibration_returns``, stored positionally (cql.py:243-266)."""
        if self.calibrated:
            assert isinstance(buffer, ReplayBuffer)
            batch, indices = buffer.sample(0)
            returns, _ = self.compute_episodic_return(batch=batch, buffer=buffer, indices=indices, gamma=self.gamma, gae_lambda=1.0)
            buffer._meta = Batch(**buffer._meta.__dict__, calibration_returns=returns)
            buffer.__dict__.get("_dev_cache", {}).pop("calibration_returns", None)     # device_array() uploads the new key
        return buffer

    def _sample(self, buffer: ReplayBuffer, sample_size: int | None) -> tuple[Batch, Any]:
        """Indices from the buffer's host RNG streams (identical to the reference's draws); rows stay on the device."""
        from ... import ops
        indices = np.asarray(buffer.sample_indices(sample_size), dtype=np.int64)
        dev = self._dev
        idx = torch.from_numpy(indices).pin_memory().to(dev, non_blocking=True)
        cols = buffer.device_columns() if hasattr(buffer, "device_columns") else None
        at = idx if cols is not None else indices       # mirror: a device gather; else a host gather + one upload
        rows = lambda key, where: ops.buffer_rows(buffer, key, where, dev, cols=cols).contiguous()
        batch = Batch()
        d = batch.__dict__
        d["obs"], d["act"] = rows("obs", at), rows("act", at)
        d["obs_next"] = rows("obs_next", at) if buffer._save_obs_next else rows("obs", buffer.next(indices))
        d["rew"], d["done"] = rows("rew", at).view(-1), rows("done", at).view(-1)
        if self.calibrated:
            if "calibration_returns" not in buffer._meta.get_keys():
                raise AttributeError("calibrated=True reads the buffer's calibration_returns: pass the buffer through "
                                     "process_buffer() first")
            n_ret = len(buffer._meta["calibration_returns"])
            if len(indices) and int(indices.max()) >= n_ret:
                raise IndexError(f"index {int(indices.max())} is out of bounds for the {n_ret} calibration returns")
            d["calibration_returns"] = ops.gather_rows(buffer.device_array("calibration_returns"), idx).to(torch.float32)
        d["info"] = Batch()
        return batch, indices

    # ------------------------------------------------------------------ update
    def _update_with_batch(self, batch: Batch) -> CQLTrainingStats:
        losses, alpha_loss = self._device_update(batch)
        l = losses.cpu().numpy()                # the only host read of the losses
        lag = self.with_lagrange
        return CQLTrainingStats(actor_loss=float(l[0]), critic1_loss=float(l[1]), critic2_loss=float(l[2]),
                                alpha=float(self.alpha.value), alpha_loss=alpha_loss,
                                cql_alpha=float(l[3]) if lag else None, cql_alpha_loss=float(l[4]) if lag else None)

    def _device_update(self, batch: Batch) -> tuple[torch.Tensor, float | None]:
        """Everything of one update after the sampling; returns the device losses (actor, critic1, critic2, cql_alpha,
        cql_alpha_loss) and alpha's loss."""
        dev, st = self._dev, stream_ptr(self._dev)
        obs, act, obs_next = batch.obs, batch.act, batch.obs_next
        B, A, R = obs.shape[0], self.act_dim, int(self.num_repeat_actions)
        N = B * R
        losses = self._buf("losses", 5)

        # actor: mean(alpha log pi - min(Q1, Q2)) against the current critics (cql.py:208-216, 275-276)
        logp = self._actor_step(obs, float(self.alpha.value), losses[0:1])
        alpha_loss = self.alpha.update(-logp.detach().unsqueeze(-1))

        # target with the updated actor and alpha (cql.py:282-292)
        alpha = float(self.alpha.value)
        _, act_n, logp_n, _, _ = self._actor_forward(obs_next, "tq")
        t_acts = self._q_pair(obs_next, act_n, "tq", target=True)
        y = self._buf("target", B)
        call("ts_cql_target", ptr(t_acts[0][-1]), ptr(t_acts[1][-1]), ptr(logp_n), alpha, ptr(batch.rew), ptr(batch.done), float(self.gamma), B, ptr(y), st)

        # random actions on torch's CPU generator (cql.py:303-307), uploaded without blocking the host
        rand = torch.empty((N, A), dtype=torch.float32, pin_memory=True).uniform_(-self.min_action, self.max_action)
        rand = rand.to(dev, non_blocking=True)

        # current-pi on the repeated obs, next-pi on the repeated obs_next (cql.py:309-317)
        tmp_obs = self._repeat_rows(obs, R, "tmp_obs")
        tmp_obs_next = self._repeat_rows(obs_next, R, "tmp_obs_next")
        _, act_c, logp_c, _, _ = self._actor_forward(tmp_obs, "pc")
        _, act_x, logp_x, _, _ = self._actor_forward(tmp_obs_next, "px")

        # one critic input over [data | random | current-pi | next-pi]; the next-pi block reads the repeated obs (cql.py:317)
        x = self._buf("cq_x", (B + 3 * N, self.obs_dim + A))
        self._concat(obs, act, x[:B])
        for j, a in enumerate((rand, act_c, act_x)):
            self._concat(tmp_obs, a, x[B + j * N:B + (j + 1) * N])
        q = [self._c[k].forward(x, B + 3 * N, "cq") for k in range(2)]
        cal = batch.calibration_returns if self.calibrated else None
        log_alpha = self._g_la.flat if self.with_lagrange else None
        if log_alpha is not None:
            self._g_la.ensure_adopted()
            self._sync_multiplier_state()
        dq = [self._buf(f"cq_dq{k}", (B + 3 * N, 1)) for k in range(2)]
        sq_rows, lse_rows = self._buf("cq_sq", 2 * B), self._buf("cq_lse", 2 * N)
        rand_logp = float(np.log(0.5 ** A))                 # cql.py:236 (a float64 numpy scalar; subtracted in fp32)
        call("ts_cql_rows", ptr(q[0][-1]), ptr(q[1][-1]), ptr(y), B, R, ptr(logp_c), ptr(logp_x), rand_logp, ptr(cal),
             float(self.temperature), float(self.cql_weight), ptr(log_alpha), float(self.alpha_min), float(self.alpha_max),
             ptr(dq[0]), ptr(dq[1]), ptr(sq_rows), ptr(lse_rows), st)
        call("ts_cql_losses", ptr(q[0][-1]), ptr(q[1][-1]), ptr(sq_rows), ptr(lse_rows), B, N, float(self.temperature),
             float(self.cql_weight), ptr(log_alpha), float(self.alpha_min), float(self.alpha_max), float(self.lagrange_threshold),
             ptr(self._g_la.grad) if log_alpha is not None else None, ptr(losses[1:5]), st)
        if log_alpha is not None:                           # cql.py:378-381
            self._adam(self._g_la, self.cql_alpha_optim, None)
            self._g_la.export_state(self.cql_alpha_optim)

        # critics: parameter gradients only (cql.py:383-388), clipped Adam
        for k, optim in enumerate((self.critic_optim, self.critic2_optim)):
            self._c[k].backward(q[k], dq[k], B + 3 * N, "cq")
            self._adam(self._g_c[k], optim._optim, optim._max_grad_norm)
        self._polyak()
        return losses, alpha_loss

    def _sync_multiplier_state(self) -> None:
        """``cql_alpha_optim``'s state IS the flat group's (views); after a ``load_state_dict`` replaced it, pull it in."""
        st = self.cql_alpha_optim.state.get(self.cql_log_alpha)
        if st and st.get("exp_avg") is not None and st["exp_avg"].data_ptr() == self._g_la.exp_avg.data_ptr():
            return
        self._g_la.import_state(self.cql_alpha_optim)
