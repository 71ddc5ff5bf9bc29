"""Flat f32 parameter / gradient / Adam-moment storage shared between torch modules and the CUDA kernels.

The kernels address an optimiser's parameters through ONE flat buffer: the fused actor-critic kernels (csrc/mlp.cu,
mlp_tc.cu) through the offsets of ``ts_actor_critic_desc``, the layer-wise networks (netgraph.py) through per-layer
offsets.  To keep ``state_dict()`` / ``load_state_dict()`` / the Collector's torch forward working unchanged (SURVEY 5:
checkpoint/resume), every ``nn.Parameter`` is re-pointed at a view of that buffer: kernels update the flat buffer in
place and the modules see the new weights without copies.
"""
from __future__ import annotations

import math
from typing import Any

import torch
from torch import nn
from torch.distributions import Categorical, Independent, Normal

from .._cabi import OPT_ADAM, OPT_RMSPROP, call, ptr, stream_ptr


class UnsupportedModelError(NotImplementedError):
    """Raised when actor / critic / dist_fn / optimizer are outside the fused kernel family.
    There is deliberately no eager-PyTorch fallback."""


def check_categorical_dist_fn(dist_fn: Any, act_dim: int, device: torch.device) -> None:
    """The categorical kernels hard-wire Categorical(probs = actor output) (test_ppo_discrete.py:108)."""
    probs = torch.full((2, act_dim), 1.0 / act_dim, device=device)
    probs[0, 0] += 0.25 / act_dim
    probs[0, -1] -= 0.25 / act_dim
    d = dist_fn(probs)
    if not isinstance(d, Categorical) or not torch.allclose(d.probs, probs, atol=1e-6):
        raise UnsupportedModelError(f"dist_fn must build Categorical(probs=actor output); got {d}")


def check_gaussian_dist_fn(dist_fn: Any, act_dim: int, device: torch.device) -> None:
    """The kernels hard-wire Independent(Normal(mu, sigma), 1) (mujoco_ppo.py:133-135)."""
    loc = torch.zeros(2, act_dim, device=device)
    d = dist_fn((loc, torch.ones_like(loc)))
    if not (isinstance(d, Independent) and isinstance(d.base_dist, Normal) and d.reinterpreted_batch_ndims == 1):
        raise UnsupportedModelError(f"dist_fn must build Independent(Normal(loc, scale), 1); got {d}")


def optimizer_hyperparams(optimizer: torch.optim.Optimizer, *, rmsprop: bool = True) -> dict[str, Any]:
    """The device step's hyper-parameters, keyed by ``ts_ppo_hparams`` field, for a torch Adam or (``rmsprop``) RMSprop;
    ``optimizer`` is ``OPT_ADAM`` or ``OPT_RMSPROP``.  RMSprop's ``alpha`` travels in ``beta2`` and its ``eps`` in
    ``adam_eps`` (include/ts_b200.h).  Every optimiser or option the kernels do not implement raises
    ``UnsupportedModelError``."""
    kind = type(optimizer)
    if kind is not torch.optim.Adam and not (rmsprop and kind is torch.optim.RMSprop):
        allowed = "torch.optim.Adam / torch.optim.RMSprop" if rmsprop else "torch.optim.Adam"
        raise UnsupportedModelError(f"fused update supports {allowed} only, got {kind.__name__}")
    if len(optimizer.param_groups) != 1:
        raise UnsupportedModelError("fused update supports a single param group")
    g = optimizer.param_groups[0]
    lr = g["lr"]
    lr = float(lr.item()) if isinstance(lr, torch.Tensor) else float(lr)
    if kind is torch.optim.RMSprop:
        # momentum and centered would each need a third state vector next to the parameters and square_avg; no reference
        # example uses them (examples/mujoco/mujoco_a2c.py:117-121 builds RMSprop(lr, eps, alpha))
        if g.get("momentum") or g.get("centered"):
            raise UnsupportedModelError("RMSprop momentum != 0 / centered=True unsupported: the device step keeps square_avg "
                                        "as its only state vector")
        if g.get("maximize"):
            raise UnsupportedModelError("RMSprop maximize=True unsupported")
        alpha = float(g["alpha"])
        if not all(math.isfinite(x) for x in (lr, alpha)):
            raise ValueError("non-finite RMSprop hyper-parameters")
        return dict(optimizer=OPT_RMSPROP, lr=lr, beta2=alpha, adam_eps=float(g["eps"]), weight_decay=float(g["weight_decay"]))
    if g.get("amsgrad") or g.get("maximize") or g.get("decoupled_weight_decay"):
        raise UnsupportedModelError("amsgrad / maximize / decoupled weight decay unsupported")
    b1, b2 = g["betas"]
    if not all(math.isfinite(x) for x in (lr, b1, b2)):
        raise ValueError("non-finite Adam hyper-parameters")
    return dict(optimizer=OPT_ADAM, lr=lr, beta1=float(b1), beta2=float(b2), adam_eps=float(g["eps"]),
                weight_decay=float(g["weight_decay"]))


def bind_optimizer(optim: Any, group: FlatGroup, *, rmsprop: bool = False, frozen: tuple[nn.Parameter, ...] = ()) -> None:
    """Let ``group`` hold the state of ``optim`` (an ``Algorithm.Optimizer``): the kernels step the flat buffers with the
    torch optimiser's hyper-parameters, and ``state_dict()`` / ``load_state_dict()`` go through ``group``.  ``rmsprop``:
    the caller steps through ``FlatGroup.optimizer_step`` or the actor-critic kernels, which also take torch RMSprop.
    ``frozen``: parameters with ``requires_grad=False`` that the optimiser lists but never steps (C51's ``support``); they
    keep their place in its param group, get no state and stay out of ``group``."""
    optimizer_hyperparams(optim._optim, rmsprop=rmsprop)
    if any(p.requires_grad for p in frozen):
        raise UnsupportedModelError("a parameter the optimiser may skip must have requires_grad=False")
    if set(map(id, optim._optim.param_groups[0]["params"])) != set(map(id, group.params)) | set(map(id, frozen)):
        raise UnsupportedModelError("optimizer parameters differ from the fused network's parameters")
    optim._flat = group


class FlatGroup:
    """Flat fp32 storage (parameters, gradient, Adam moments) of one optimiser's parameters.

    The Adam step count has one owner: a host int that ``adam_step`` advances, or -- once ``step_dev`` exists -- the
    int64[1] device counter that kernels advance without a host round trip.  ``device_step`` creates that counter up front
    (the fused actor-critic kernels); ``adam_step_device`` creates it on first use (CUDA-graph mode).  ``grad_extra``
    floats past the ``n`` parameters of ``grad`` are kernel scratch; ``partials`` and ``weight_image`` are scratch of the
    fused actor-critic kernels, set by the algorithm that runs them."""

    def __init__(self, params: list[nn.Parameter], device: torch.device, *, grad_extra: int = 0,
                 device_step: bool = False) -> None:
        self.params = list(params)
        self.device = device
        self.n = sum(p.numel() for p in self.params)
        self.flat = torch.empty(self.n, dtype=torch.float32, device=device)
        self.grad = torch.zeros(self.n + grad_extra, dtype=torch.float32, device=device)
        self.exp_avg = torch.zeros(self.n, dtype=torch.float32, device=device)
        self.exp_avg_sq = torch.zeros(self.n, dtype=torch.float32, device=device)
        self.norm_scratch = torch.zeros(256, dtype=torch.float64, device=device)
        self.partials: torch.Tensor | None = None
        self.weight_image: torch.Tensor | None = None
        self._step = 0
        self.step_dev = torch.zeros(1, dtype=torch.int64, device=device) if device_step else None
        self._offsets: dict[int, int] = {}
        off = 0
        for p in self.params:
            self._offsets[id(p)] = off
            off += p.numel()
        self._ptrs: list[int] = []
        self.adopt()

    @property
    def step(self) -> int | torch.Tensor:
        """The Adam step count where it lives: ``step_dev`` when it exists, else the host int."""
        return self.step_dev if self.step_dev is not None else self._step

    def offset(self, p: nn.Parameter) -> int:
        return self._offsets[id(p)]

    def view(self, buf: torch.Tensor, p: nn.Parameter) -> torch.Tensor:
        o = self._offsets[id(p)]
        return buf[o:o + p.numel()]

    def adopt(self) -> None:
        """Copy current parameter values into the flat buffer and re-point ``p.data`` at views."""
        with torch.no_grad():
            for p in self.params:
                v = self.view(self.flat, p).view(p.shape)
                if p.data.data_ptr() != v.data_ptr():
                    v.copy_(p.data.to(self.device, torch.float32))
                    p.data = v
        self._ptrs = [p.data.data_ptr() for p in self.params]

    def ensure_adopted(self) -> None:
        if [p.data.data_ptr() for p in self.params] != self._ptrs:
            self.adopt()

    def _advance_step(self) -> int:
        step = self.sync_step_from_device() + 1
        if self.step_dev is not None:
            self.step_dev.fill_(step)
        else:
            self._step = step
        return step

    def adam_step(self, optimizer: torch.optim.Optimizer, max_grad_norm: float | None) -> None:
        """``Algorithm.Optimizer.step`` after backward: clip_grad_norm_ (optional) + Adam (algorithm_base.py:496-500)."""
        hp = optimizer_hyperparams(optimizer, rmsprop=False)
        step = self._advance_step()
        call("ts_adam_step", ptr(self.flat), ptr(self.grad), ptr(self.exp_avg), ptr(self.exp_avg_sq), self.n, step,
             hp["lr"], hp["beta1"], hp["beta2"], hp["adam_eps"], hp["weight_decay"], float(max_grad_norm or 0.0),
             ptr(self.norm_scratch), stream_ptr(self.device))

    def optimizer_step(self, optimizer: torch.optim.Optimizer, max_grad_norm: float | None) -> None:
        """``adam_step``, or for a torch RMSprop clip_grad_norm_ (optional) + RMSprop (``ts_rmsprop_step``; square_avg in
        ``exp_avg_sq``)."""
        hp = optimizer_hyperparams(optimizer)
        if hp["optimizer"] == OPT_ADAM:
            self.adam_step(optimizer, max_grad_norm)
            return
        self._advance_step()
        call("ts_rmsprop_step", ptr(self.flat), ptr(self.grad), ptr(self.exp_avg_sq), self.n, hp["lr"], hp["beta2"],
             hp["adam_eps"], hp["weight_decay"], float(max_grad_norm or 0.0), ptr(self.norm_scratch), stream_ptr(self.device))

    def adam_step_device(self, optimizer: torch.optim.Optimizer, max_grad_norm: float | None) -> None:
        """Same step with the step number read from / advanced in DEVICE memory: nothing in the launch depends on host state,
        so it can live inside a captured CUDA graph."""
        hp = optimizer_hyperparams(optimizer, rmsprop=False)
        if self.step_dev is None:
            self.step_dev = torch.tensor([self._step], dtype=torch.int64, device=self.device)
        call("ts_adam_step_dev", ptr(self.flat), ptr(self.grad), ptr(self.exp_avg), ptr(self.exp_avg_sq), self.n, ptr(self.step_dev),
             hp["lr"], hp["beta1"], hp["beta2"], hp["adam_eps"], hp["weight_decay"], float(max_grad_norm or 0.0),
             ptr(self.norm_scratch), stream_ptr(self.device))

    def sync_step_from_device(self) -> int:
        """The step count as a host int: one read of ``step_dev`` when the device counter owns it."""
        return int(self.step_dev.item()) if self.step_dev is not None else self._step

    # -- torch.optim.Adam / RMSprop state interop --------------------------------------------
    def export_state(self, optimizer: torch.optim.Optimizer) -> None:
        """Expose the flat moments as the torch optimizer's per-parameter state (views): Adam's exp_avg / exp_avg_sq, or
        RMSprop's square_avg (``exp_avg_sq``)."""
        step = self.sync_step_from_device()
        if step == 0 and len(optimizer.state) == 0:
            return
        rmsprop = type(optimizer) is torch.optim.RMSprop
        for p in self.params:
            st = {"step": torch.tensor(float(step), dtype=torch.float32)}
            if rmsprop:
                st["square_avg"] = self.view(self.exp_avg_sq, p).view(p.shape)
            else:
                st["exp_avg"] = self.view(self.exp_avg, p).view(p.shape)
                st["exp_avg_sq"] = self.view(self.exp_avg_sq, p).view(p.shape)
            optimizer.state[p] = st

    def import_state(self, optimizer: torch.optim.Optimizer) -> None:
        """After ``optimizer.load_state_dict`` or an eager ``optimizer.step()``: pull its moments / step into the flat
        buffers, then expose them as the optimizer's state again."""
        steps = []
        rmsprop = type(optimizer) is torch.optim.RMSprop
        with torch.no_grad():
            for p in self.params:
                st = optimizer.state.get(p)
                m, v = self.view(self.exp_avg, p), self.view(self.exp_avg_sq, p)
                if not st:
                    m.zero_(); v.zero_()
                    continue
                if rmsprop:
                    v.copy_(st["square_avg"].to(self.device, torch.float32).reshape(-1))
                else:
                    m.copy_(st["exp_avg"].to(self.device, torch.float32).reshape(-1))
                    v.copy_(st["exp_avg_sq"].to(self.device, torch.float32).reshape(-1))
                steps.append(float(st["step"]))
        if steps and max(steps) != min(steps):
            raise UnsupportedModelError("per-parameter optimiser step counts differ; cannot fuse")
        step = int(round(steps[0])) if steps else 0
        if self.step_dev is not None:
            self.step_dev.fill_(step)
        else:
            self._step = step
        self.export_state(optimizer)


class DeviceScratch(dict):
    """An algorithm's named scratch: ``tensor`` returns the cached device tensor of that name while its shape and dtype still
    fit, so the update loop does no allocator traffic.  Other per-update state (pinned host buffers, the running-mean
    state of one update) may sit under names of its own."""

    def __init__(self, device: torch.device) -> None:
        super().__init__()
        self.device = device

    def tensor(self, name: str, shape: tuple[int, ...] | int, dtype: torch.dtype = torch.float32) -> torch.Tensor:
        shape = (shape,) if isinstance(shape, int) else tuple(shape)
        t = self.get(name)
        if t is None or t.shape != shape or t.dtype != dtype:
            t = self[name] = torch.empty(shape, dtype=dtype, device=self.device)
        return t
