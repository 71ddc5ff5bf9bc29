"""TEST INFRASTRUCTURE -- float64 restatement of imitation learning's update: the two losses with their gradients at the last
Linear's output written out by hand, and the update on a float64 copy of the actor stepped by torch's Adam.

Only ``tests/`` and ``tools/`` may import this module; ``tianshou_b200`` never does.  It restates
tianshou/algorithm/imitation/imitation_base.py:109-127 without the framework around it:

* regression (continuous): ``F.mse_loss(max_action * tanh(z), act)``, the mean over B * A elements, z the last Linear's output;
* classification (discrete): ``F.nll_loss(F.log_softmax(y), act)``, the mean over B, with y = z, or y = softmax(z) for a
  ``DiscreteActor(softmax_output=True)``: the reference then takes log_softmax of probabilities, and so does this restatement.

PINNING: tests/test_oracle_imitation.py replays tests/golden/il_ref_*.npz (outputs of the imported reference,
oracle/gen_golden_imitation.py) through ``imitation_update``.
"""
from __future__ import annotations

import numpy as np
import torch
from torch import nn


def _log_softmax(x: np.ndarray) -> np.ndarray:
    m = x.max(-1, keepdims=True)
    return x - m - np.log(np.exp(x - m).sum(-1, keepdims=True))


def mse_rows(z: np.ndarray, act: np.ndarray, max_action: float) -> tuple[float, np.ndarray]:
    """(loss, d loss / d z) of the regression loss."""
    z, act = np.asarray(z, np.float64), np.asarray(act, np.float64).reshape(np.shape(z))
    t = np.tanh(z)
    d = max_action * t - act
    return float((d * d).mean()), 2.0 * d / d.size * max_action * (1.0 - t * t)


def nll_rows(z: np.ndarray, act: np.ndarray, softmax_output: bool) -> tuple[float, np.ndarray, np.ndarray]:
    """(loss, d loss / d z, per-row losses) of the classification loss."""
    z = np.asarray(z, np.float64)
    B, A = z.shape
    rows = np.arange(B)
    hit = np.zeros((B, A))
    hit[rows, np.asarray(act).reshape(-1)] = 1.0
    y = np.exp(_log_softmax(z)) if softmax_output else z
    lp = _log_softmax(y)
    row = -lp[rows, np.asarray(act).reshape(-1)]
    g = (np.exp(lp) - hit) / B
    dz = y * (g - (y * g).sum(-1, keepdims=True)) if softmax_output else g
    return float(row.mean()), dz, row


def chain(mod: nn.Module) -> list[nn.Module]:
    """The actor's module chain: ``preprocess`` then ``last`` (ContinuousActorDeterministic, DiscreteActor), or the ``model`` /
    ``net`` Sequential of a Net / MLP / DQNet; ends in the last Linear."""
    if hasattr(mod, "preprocess") and hasattr(mod, "last"):
        return chain(mod.preprocess) + chain(mod.last)
    if isinstance(mod, nn.Sequential):
        return list(mod)
    for name in ("model", "net"):
        inner = getattr(mod, name, None)
        if isinstance(inner, nn.Module):
            return chain(inner)
    raise TypeError(f"no module chain in {type(mod).__name__}")


def last_output(actor: nn.Module, obs: torch.Tensor) -> torch.Tensor:
    """The last Linear's output z of the actor on ``obs`` (float64)."""
    x = obs
    for m in chain(actor):
        x = m(x)
    return x


def make_actor(cfg, mods):
    """The actor of a variant built from ``mods`` (the reference's modules, or tianshou_b200's at the same paths)."""
    Net_, CAD, DA, DQNet_ = mods
    torch.manual_seed(0)
    if cfg["kind"] == "cont":
        net = Net_(state_shape=(cfg["obs"],), action_shape=cfg["A"] if cfg["net_action"] else 0, hidden_sizes=cfg["hidden"])
        return CAD(preprocess_net=net, action_shape=cfg["A"], max_action=cfg["max_action"])
    if cfg["actor"] == "dqnet":
        return DQNet_(4, cfg["H"], cfg["W"], cfg["A"])
    if cfg["actor"] == "net":
        return Net_(state_shape=(cfg["obs"],), action_shape=cfg["A"], hidden_sizes=cfg["hidden"])
    return DA(preprocess_net=Net_(state_shape=(cfg["obs"],), hidden_sizes=cfg["hidden"]), action_shape=cfg["A"],
              softmax_output=cfg["softmax"])


class ImitationState:
    """A float64 copy of the actor and torch's Adam over its parameters, in ``parameters()`` order."""

    def __init__(self, actor: nn.Module, lr: float) -> None:
        self.actor = actor.double()
        self.params = list(actor.parameters())
        self.opt = torch.optim.Adam(self.params, lr=lr)


def imitation_update(s: ImitationState, obs: np.ndarray, act: np.ndarray, kind: str, max_action: float = 1.0,
                     softmax_output: bool = False) -> dict:
    """One update on the batch the reference's buffer delivered (``obs`` as stored: uint8 frames are read as their values, as
    ``DQNet`` reads them).  ``kind``: ``"cont"`` (regression) or anything else (classification).  Returns the loss, the
    gradient at z and the parameter gradients before the step."""
    x = torch.as_tensor(np.asarray(obs)).double()
    z = last_output(s.actor, x)
    zn = z.detach().numpy()
    if kind == "cont":
        loss, dz = mse_rows(zn, act, max_action)
        row = None
    else:
        loss, dz, row = nll_rows(zn, act, softmax_output)
    s.opt.zero_grad()
    z.backward(torch.as_tensor(dz))
    grads = [p.grad.detach().clone() for p in s.params]
    s.opt.step()
    return dict(loss=loss, dz=dz, rows=row, grads=grads)
