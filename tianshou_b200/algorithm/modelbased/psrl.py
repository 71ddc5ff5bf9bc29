"""Posterior sampling reinforcement learning (PSRL, Strens 2000) with the posterior update and value iteration on the device.

Reference: tianshou/algorithm/modelbased/psrl.py (PSRLTrainingStats :18-21, PSRLModel :24-160, PSRLPolicy :163-214, PSRL :217-276).

The model's state (the Dirichlet counts over transitions and the normal posterior over rewards) lives on the device in float64.

  update       : the rows in ``np.random.permutation(len(batch))`` order, drawn on the host from numpy's global stream exactly as
                 ``batch.split(size=1)`` draws it -> ``ts_psrl_update``: one pass checks every index, the batch's sums run per
                 (s, a) in that order in float64 (a stable sort groups the rows), the counts are exact, and observe's formula is
                 applied with explicitly rounded operations, so the posterior is bit-for-bit the reference's.  One device-to-host
                 copy per update brings back the error flag and the two stat means.  An index out of range (or negative, which
                 numpy would wrap) raises ``IndexError`` and changes nothing.
  solve_policy : at the first call after an update: a Dirichlet draw of P and a normal draw of the rewards on torch's device
                 generator, then ``ts_psrl_value_iteration``, one cooperative kernel that sweeps until np.allclose's test holds,
                 adds the tie-break noise and takes the first argmax.  One copy brings back the policy, the sweep count and the
                 converged flag; ``forward`` then indexes the host policy with no further synchronise.

Value iteration that does not converge in ``max_iterations`` sweeps (the reference loops forever, e.g. on NaN rewards) raises
``RuntimeError`` and keeps the previous policy and value.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Any

import numpy as np
import torch

from ... import ops
from ..._cabi import to_device
from ...data import Batch, ReplayBuffer
from ..base import OnPolicyAlgorithm, Policy, TrainingStats
from ..flat_params import UnsupportedModelError

DEFAULT_MAX_ITERATIONS = 100_000
_IDX_KEYS = ("obs", "act", "obs_next")


@dataclass(kw_only=True)
class PSRLTrainingStats(TrainingStats):
    psrl_rew_mean: float = 0.0
    psrl_rew_std: float = 0.0


def _index_column(a: Any, key: str) -> np.ndarray:
    a = np.asarray(a)
    if a.dtype.kind not in "iu":
        raise IndexError(f"PSRL: '{key}' must hold integer indices, got dtype {a.dtype}")
    return a.reshape(-1)


@dataclass
class _Rows:
    """The rollout's columns on the device: int64 indices (host path) or the device mirror's float32 ones, float32 or float64
    rewards, ``sq_f32`` when the buffer's rewards are float32 (squared in float32, as numpy does)."""

    obs: torch.Tensor
    act: torch.Tensor
    obs_next: torch.Tensor
    rew: torch.Tensor
    done: torch.Tensor
    sq_f32: bool

    def __len__(self) -> int:
        return self.obs.numel()

    def check(self) -> None:
        """Every column holds one value per row (the kernels read each of them at every row)."""
        n = len(self)
        for k in ("act", "obs_next", "rew", "done"):
            if getattr(self, k).numel() != n:
                raise ValueError(f"PSRL: '{k}' has {getattr(self, k).numel()} entries for {n} rows")

    @staticmethod
    def from_batch(batch: Batch, device: torch.device) -> "_Rows":
        """One upload of the sampled batch's columns."""
        idx = [_index_column(batch[k], k) for k in _IDX_KEYS]
        rew = np.asarray(batch.rew).reshape(-1)
        sq_f32 = rew.dtype == np.float32
        if not sq_f32 and rew.dtype != np.float64:
            rew = rew.astype(np.float64)
        done = batch.done if "done" in batch.get_keys() else np.logical_or(batch.terminated, batch.truncated)
        cols = [to_device(c.astype(np.int64, copy=False), device) for c in idx]
        return _Rows(*cols, to_device(rew, device), to_device(np.asarray(done, dtype=bool).reshape(-1), device), sq_f32)

    @staticmethod
    def from_mirror(buffer: ReplayBuffer, indices: np.ndarray, device: torch.device) -> "_Rows | None":
        """The rows gathered from the buffer's device mirror at ``indices``, or None when the buffer keeps no usable mirror."""
        cols = buffer.device_columns()
        need = (*_IDX_KEYS, "rew", "done")
        if cols is None or not all(k in cols for k in need) or cols["obs"].device != device:
            return None
        if any(cols[k].dtype != torch.float32 for k in _IDX_KEYS) or cols["rew"].dtype not in (torch.float32, torch.float64):
            return None     # e.g. uint8 observations, which the mirror keeps as uint8: the upload path reads them
        meta = buffer._meta
        for k in _IDX_KEYS:
            _index_column(meta[k][:0], k)
        idx = to_device(np.asarray(indices, dtype=np.int64), device)
        g = {k: ops.gather_rows(cols[k].reshape(cols[k].shape[0], -1), idx).reshape(-1) for k in need}
        return _Rows(g["obs"], g["act"], g["obs_next"], g["rew"], g["done"].view(torch.uint8),
                     np.asarray(meta.rew).dtype == np.float32)


class PSRLModel:
    """Posterior sampling RL model (psrl.py:24-160) with its state on the device.

    ``trans_count``, ``rew_mean``, ``rew_std``, ``rew_square_sum``, ``rew_count``, ``value`` and ``policy`` read as numpy arrays:
    each read is a copy to the host and synchronises, so they are not for the hot path.
    """

    def __init__(self, trans_count_prior: np.ndarray, rew_mean_prior: np.ndarray, rew_std_prior: np.ndarray, gamma: float,
                 epsilon: float, *, max_iterations: int = DEFAULT_MAX_ITERATIONS, device: torch.device | str | None = None) -> None:
        self.device = ops._dev(device)
        self.n_state, self.n_action = np.shape(rew_mean_prior)
        shape = (self.n_state, self.n_action)
        if np.shape(trans_count_prior) != (*shape, self.n_state) or np.shape(rew_std_prior) != shape:
            raise ValueError(f"PSRL priors: trans_count_prior must be {(*shape, self.n_state)} and rew_std_prior {shape}")
        _check_states(self.n_state)
        if max_iterations < 1:
            raise ValueError("max_iterations must be at least 1")

        def f64(a: Any) -> torch.Tensor:     # a copy: the caller's prior is never aliased
            return to_device(np.array(a, dtype=np.float64), self.device)

        self._trans_count = f64(trans_count_prior)
        self._rew_mean = f64(rew_mean_prior)
        self._rew_std_prior = f64(rew_std_prior)
        self._rew_std = self._rew_std_prior.clone()
        self._rew_square_sum = torch.zeros(shape, dtype=torch.float64, device=self.device)
        self._rew_count = torch.full(shape, float(epsilon), dtype=torch.float64, device=self.device)
        self._value = torch.zeros(self.n_state, dtype=torch.float64, device=self.device)
        self._policy: np.ndarray | None = None
        self.gamma = gamma
        self.eps = epsilon
        self.max_iterations = int(max_iterations)
        self.updated = False
        self.last_sweeps = 0
        self._result = torch.empty(3, dtype=torch.float64, device=self.device)
        self._flag = torch.empty(1, dtype=torch.int32, device=self.device)
        self._workspace: torch.Tensor | None = None
        self._vi_scratch: torch.Tensor | None = None
        self._vi_out: torch.Tensor | None = None

    # ---------------------------------------------------------------------------------------------------- host views
    trans_count = property(lambda self: self._trans_count.cpu().numpy())
    rew_mean = property(lambda self: self._rew_mean.cpu().numpy())
    rew_std = property(lambda self: self._rew_std.cpu().numpy())
    rew_square_sum = property(lambda self: self._rew_square_sum.cpu().numpy())
    rew_count = property(lambda self: self._rew_count.cpu().numpy())
    value = property(lambda self: self._value.cpu().numpy())

    @property
    def policy(self) -> np.ndarray:
        if self._policy is None:
            raise AttributeError("PSRLModel.policy: no policy has been solved yet")
        return self._policy.copy()

    def _state(self) -> tuple[torch.Tensor, ...]:
        return self._trans_count, self._rew_mean, self._rew_std, self._rew_square_sum, self._rew_count

    # ---------------------------------------------------------------------------------------------------- posterior
    def observe(self, trans_count: Any, rew_sum: Any, rew_square_sum: Any, rew_count: Any) -> None:
        """Add a batch's dense counts and sums (psrl.py:65-98); the same per-element update as the row path."""
        shapes = ((self.n_state, self.n_action, self.n_state), *[(self.n_state, self.n_action)] * 3)
        arrays = (trans_count, rew_sum, rew_square_sum, rew_count)
        for name, a, shape in zip(("trans_count", "rew_sum", "rew_square_sum", "rew_count"), arrays, shapes, strict=True):
            if tuple(np.shape(a)) != shape:
                raise ValueError(f"PSRLModel.observe: {name} has shape {tuple(np.shape(a))}, expected {shape}")
        batch = tuple(to_device(np.asarray(a, dtype=np.float64) if not isinstance(a, torch.Tensor) else a, self.device,
                                dtype=torch.float64) for a in arrays)
        self.updated = False
        ops.psrl_observe(batch, self._state(), self._rew_std_prior, self._flag, self._result)

    def _observe_rows(self, rows: _Rows, perm: np.ndarray, add_done_loop: bool) -> tuple[float, float]:
        """The posterior update from the rows taken in ``perm``'s order; (mean(rew_mean), mean(rew_std))."""
        rows.check()
        n = len(rows)
        if len(perm) != n:
            raise ValueError(f"PSRL: a permutation of {len(perm)} rows for {n} rows")
        if n == 0:
            z = np.zeros((self.n_state, self.n_action))
            self.observe(np.zeros((self.n_state, self.n_action, self.n_state)), z, z, z)
        else:
            self._workspace = ops.psrl_update(rows.obs, rows.act, rows.obs_next, rows.rew, rows.done,
                                              to_device(np.asarray(perm, dtype=np.int64), self.device), sq_f32=rows.sq_f32,
                                              add_done_loop=add_done_loop, state=self._state(), rew_std_prior=self._rew_std_prior,
                                              workspace=self._workspace, result=self._result)
        res = self._result.cpu().numpy()
        if res[0] != 0:
            raise IndexError(f"PSRL: an obs / act / obs_next index lies outside [0, {self.n_state}) x [0, {self.n_action}); "
                             "the posterior is unchanged")
        self.updated = False
        return float(res[1]), float(res[2])

    # ---------------------------------------------------------------------------------------------------- draws
    def sample_trans_prob(self) -> torch.Tensor:
        return torch.distributions.Dirichlet(self._trans_count).sample()

    def sample_reward(self) -> torch.Tensor:
        return self._rew_mean + self._rew_std * torch.randn(self._rew_mean.shape, dtype=torch.float64, device=self.device)

    def _tie_noise(self, shape: tuple[int, ...]) -> torch.Tensor:
        return torch.randn(shape, dtype=torch.float64, device=self.device)

    # ---------------------------------------------------------------------------------------------------- solve
    def solve_policy(self) -> None:
        trans_prob = self.sample_trans_prob()
        rew = self.sample_reward()
        noise = self._tie_noise((self.n_state, self.n_action))
        self._vi_scratch, self._vi_out, policy, sweeps = _solve(trans_prob, rew, noise, self.gamma, self.eps, self.max_iterations,
                                                                self._value, self._vi_scratch, self._vi_out)
        self._policy, self.last_sweeps, self.updated = policy, sweeps, True

    @staticmethod
    def value_iteration(trans_prob: np.ndarray | torch.Tensor, rew: np.ndarray | torch.Tensor, gamma: float, eps: float,
                        value: np.ndarray | torch.Tensor, *, noise: np.ndarray | torch.Tensor | None = None,
                        max_iterations: int = DEFAULT_MAX_ITERATIONS,
                        device: torch.device | str | None = None) -> tuple[Any, Any]:
        """(policy, value) of value iteration on the device (psrl.py:116-150).  numpy inputs give numpy outputs, CUDA tensors give
        tensors.  Without ``noise`` the tie-break noise is ``np.random.randn`` for numpy inputs (numpy's global stream, as in the
        reference) and ``torch.randn`` on the device for tensors."""
        as_numpy = not isinstance(trans_prob, torch.Tensor)
        dev = ops._dev(device) if as_numpy else trans_prob.device
        if len(np.shape(rew)) != 2:
            raise ValueError(f"PSRLModel.value_iteration: rew must be [n_state, n_action], got shape {tuple(np.shape(rew))}")
        n_s, n_a = np.shape(rew)
        _check_states(n_s)
        P, R = (to_device(x, dev, dtype=torch.float64) for x in (trans_prob, rew))
        V = to_device(value, dev, dtype=torch.float64).clone()
        if noise is None:
            noise = np.random.randn(n_s, n_a) if as_numpy else torch.randn((n_s, n_a), dtype=torch.float64, device=dev)
        noise = to_device(noise, dev, dtype=torch.float64)
        _, _, policy, _ = _solve(P, R, noise, gamma, eps, max_iterations, V)
        if as_numpy:
            return policy, V.cpu().numpy()
        return torch.from_numpy(policy).to(dev), V

    def __call__(self, obs: np.ndarray, state: Any = None, info: Any = None) -> np.ndarray:
        if not self.updated:
            self.solve_policy()
        return self._policy[obs]


def _check_states(n_state: int) -> None:
    limit = ops.psrl_max_states()
    if n_state > limit:
        raise UnsupportedModelError(f"PSRL: {n_state} states do not fit value iteration's shared memory (at most {limit} on this "
                                    "device)")


def _solve(trans_prob: torch.Tensor, rew: torch.Tensor, noise: torch.Tensor, gamma: float, eps: float, max_iterations: int,
           value: torch.Tensor, scratch: torch.Tensor | None = None,
           out: torch.Tensor | None = None) -> tuple[torch.Tensor, torch.Tensor, np.ndarray, int]:
    """One ``ts_psrl_value_iteration`` and its one readback: (scratch, out, host policy, sweeps).  ``value`` becomes the solve's
    value; on non-convergence it is left unchanged and RuntimeError is raised."""
    if rew.dim() != 2:
        raise ValueError(f"PSRL value iteration: rew must be [n_state, n_action], got shape {tuple(rew.shape)}")
    n_s, n_a = rew.shape
    want = {"trans_prob": (trans_prob, (n_s, n_a, n_s)), "noise": (noise, (n_s, n_a)), "value": (value, (n_s,))}
    for name, (t, shape) in want.items():
        if tuple(t.shape) != shape:
            raise ValueError(f"PSRL value iteration: {name} has shape {tuple(t.shape)}, expected {shape} for rew {(n_s, n_a)}")
        if t.device != rew.device:
            raise ValueError(f"PSRL value iteration: {name} is on {t.device}, rew on {rew.device}")
    if value.dtype != torch.float64 or not value.is_contiguous():
        raise ValueError("PSRL value iteration: value must be a contiguous float64 tensor (it is updated in place)")
    args = [t.to(torch.float64).contiguous() for t in (trans_prob, rew, noise)]
    scratch, out = ops.psrl_value_iteration(*args, gamma, eps, max_iterations, value, scratch, out)
    host = out.cpu().numpy()
    sweeps = int(host[n_s])
    if not host[n_s + 1]:
        diff = float(host[n_s + 2:n_s + 3].view(np.float64)[0])
        raise RuntimeError(f"PSRL value iteration did not converge in {sweeps} sweeps (last max |V' - V| = {diff!r}); the previous "
                           "policy and value are kept")
    return scratch, out, host[:n_s].copy(), sweeps


class PSRLPolicy(Policy):
    """psrl.py:163-214, with the additive keywords ``max_iterations`` and ``device``."""

    def __init__(self, *, trans_count_prior: np.ndarray, rew_mean_prior: np.ndarray, rew_std_prior: np.ndarray, action_space: Any,
                 discount_factor: float = 0.99, epsilon: float = 0.01, observation_space: Any | None = None,
                 max_iterations: int = DEFAULT_MAX_ITERATIONS, device: torch.device | str | None = None) -> None:
        super().__init__(action_space=action_space, observation_space=observation_space, action_scaling=False,
                         action_bound_method=None)
        self.model = PSRLModel(trans_count_prior, rew_mean_prior, rew_std_prior, discount_factor, epsilon,
                               max_iterations=max_iterations, device=device)

    def forward(self, batch: Batch, state: Any = None, **kwargs: Any) -> Batch:
        assert isinstance(batch.obs, np.ndarray), "only support np.ndarray observation"
        act = self.model(batch.obs, state=state, info=getattr(batch, "info", None))
        return Batch(act=act)


class PSRL(OnPolicyAlgorithm):
    """Posterior sampling RL (psrl.py:217-276).  ``update()`` ignores ``batch_size`` and ``repeat``, as in the reference."""

    def __init__(self, *, policy: PSRLPolicy, add_done_loop: bool = False) -> None:
        super().__init__(policy=policy)
        self._add_done_loop = add_done_loop

    def _sample(self, buffer: ReplayBuffer, sample_size: int | None) -> tuple[Any, Any]:
        """All rows in ``buffer.sample(0)``'s order, from the device mirror when the buffer keeps one."""
        if sample_size in (0, None):
            indices = buffer.sample_indices(0)
            rows = _Rows.from_mirror(buffer, indices, self.policy.model.device)
            if rows is not None:
                return rows, indices
        return super()._sample(buffer, sample_size)

    def _update_with_batch(self, batch: Any, batch_size: int | None = None, repeat: int = 1) -> PSRLTrainingStats:
        model = self.policy.model
        rows = batch if isinstance(batch, _Rows) else _Rows.from_batch(batch, model.device)
        perm = np.random.permutation(len(rows))       # batch.split(size=1)'s order, on numpy's global stream
        mean, std = model._observe_rows(rows, perm, self._add_done_loop)
        return PSRLTrainingStats(psrl_rew_mean=mean, psrl_rew_std=std)
