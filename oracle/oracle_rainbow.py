"""TEST INFRASTRUCTURE -- restatement of Rainbow DQN: C51 (oracle/oracle_c51.py) on noisy layers and dueling categorical heads,
with the noise draws, the lagged refresh and the train-mode target of the reference's update.

Only ``tests/`` and ``tools/`` may import this module; ``tianshou_b200`` never does.  It restates
tianshou/algorithm/modelfree/rainbow.py without the framework around it:

  noise   : rainbow.py ``_update_with_batch`` -- ``NoisyLinear.sample()`` (utils/net/discrete.py: ``randn(in)`` then ``randn(out)``,
            sign(x) sqrt|x|) for every noisy layer of the online network in ``modules()`` order, then of the lagged network
  lagged  : c51.py:143 -- the full copy when ``_iter % freq == 0`` (lagged_network.py:99-110 copies every parameter: on a tick
            the lagged network's fresh noise becomes the online network's), BEFORE the target is formed
  target  : c51.py:113-136 under ``torch_train_mode`` (algorithm_base.py:625): the online and the lagged network at s' both run
            with the train-mode weights mu + sigma * ger(eps_q, eps_p)
  network : common.py:355-364 / atari_network.py:196-206 -- logits = q - q.mean(dim=1, keepdim=True) + v, softmax over the atoms

``rainbow_update`` takes the noise as arguments (the goldens record the reference's draws) and runs the rows in float64 through
``oracle_c51.c51_rows``; ``keep_lagged_noise`` and ``target_eval`` are the two alternatives gen_golden_rainbow.py shows the
goldens tell apart.  ``rainbow_update_torch`` is the whole update in eager PyTorch with torch's own draws: the baseline of
tools/rainbow_timing.py and the RNG-parity reference of tests/test_rainbow_gpu.py.

PINNING: tests/test_oracle_rainbow.py replays tests/golden/rainbow_ref_*.npz (outputs of the imported reference,
oracle/gen_golden_rainbow.py) through ``rainbow_update`` and checks the dueling combine's gradient against autograd.
"""
from __future__ import annotations

from collections.abc import Callable

import numpy as np
import torch
import torch.nn.functional as F
from torch import nn

from oracle import oracle_c51 as oc
from oracle.oracle_discrete_bcq import obs_next_of
from oracle.oracle_offpolicy import nature_cnn


# ------------------------------------------------------------------------------------------------ layers and networks
class Noisy(nn.Module):
    """``NoisyLinear`` restated with its parameter order (mu_W, sigma_W, mu_bias, sigma_bias, eps_p, eps_q); the values come
    from ``seeded_params`` or a ``load_state_dict``."""

    def __init__(self, d_in: int, d_out: int):
        super().__init__()
        self.mu_W = nn.Parameter(torch.zeros(d_out, d_in))
        self.sigma_W = nn.Parameter(torch.zeros(d_out, d_in))
        self.mu_bias = nn.Parameter(torch.zeros(d_out))
        self.sigma_bias = nn.Parameter(torch.zeros(d_out))
        self.eps_p = nn.Parameter(torch.zeros(d_in), requires_grad=False)
        self.eps_q = nn.Parameter(torch.zeros(d_out), requires_grad=False)

    @staticmethod
    def f(x: torch.Tensor) -> torch.Tensor:
        x = torch.randn(x.size(0), device=x.device)
        return x.sign().mul_(x.abs().sqrt_())

    def sample(self) -> None:
        self.eps_p.copy_(self.f(self.eps_p))
        self.eps_q.copy_(self.f(self.eps_q))

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if self.training:
            return F.linear(x, self.mu_W + self.sigma_W * self.eps_q.ger(self.eps_p), self.mu_bias + self.sigma_bias * self.eps_q)
        return F.linear(x, self.mu_W, self.mu_bias)


def chain(sizes: list[int], noisy: bool, final_act: bool) -> nn.Sequential:
    """Linear (or noisy) layers over ``sizes`` with ReLU between them (and after the last with ``final_act``)."""
    mods: list[nn.Module] = []
    for i in range(len(sizes) - 1):
        mods.append(Noisy(sizes[i], sizes[i + 1]) if noisy else nn.Linear(sizes[i], sizes[i + 1]))
        if i < len(sizes) - 2 or final_act:
            mods.append(nn.ReLU())
    return nn.Sequential(*mods)


class RainbowView(nn.Module):
    """trunk -> Q head ``[B, A * N]`` (+ V head ``[B, N]``); registered in that order, the reference's.  ``logits`` is the
    dueling combine ``q - q.mean(1) + v`` (``q`` alone without a V head), ``forward`` its softmax over the atoms."""

    def __init__(self, trunk: nn.Module, Q: nn.Module, V: nn.Module | None, A: int, N: int):
        super().__init__()
        self.trunk, self.Q, self.V, self.A, self.N = trunk, Q, V, A, N

    def logits(self, x: torch.Tensor) -> torch.Tensor:
        h = self.trunk(x)
        q = self.Q(h).view(-1, self.A, self.N)
        if self.V is None:
            return q
        return q - q.mean(dim=1, keepdim=True) + self.V(h).view(-1, 1, self.N)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return self.logits(x).softmax(-1)


def rainbow_net(cfg: dict) -> RainbowView:
    """The oracle network of a golden's configuration (keys without the ``cfg_`` prefix):
    ``mlp``  -- ``Net(state_shape=obs, hidden_sizes=hidden, softmax=True, num_atoms=N, linear_layer=<noisy if trunk_noisy>,
               dueling_param=({hidden_sizes: q_hidden, linear_layer: noisy}, {hidden_sizes: v_hidden, linear_layer: <noisy if
               v_noisy>}))``;
    ``cnn``  -- ``RainbowNet(c=4, h=H, w=W, action_shape=A, num_atoms=N, is_dueling=dueling, is_noisy=noisy)``."""
    A, N = int(cfg["A"]), int(cfg["N"])
    if str(cfg["kind"]) == "cnn":
        conv = nature_cnn(4, int(cfg["H"]), int(cfg["W"]), 1)[0]
        with torch.no_grad():
            feat = int(conv(torch.zeros(1, 4, int(cfg["H"]), int(cfg["W"]))).shape[1])
        noisy, dueling = bool(cfg["noisy"]), bool(cfg["dueling"])
        Q = chain([feat, 512, A * N], noisy, False)
        V = chain([feat, 512, N], noisy, False) if dueling else None
        return RainbowView(conv, Q, V, A, N)
    hidden = [int(x) for x in cfg["hidden"]]
    trunk = chain([int(cfg["obs"]), *hidden], bool(cfg["trunk_noisy"]), True)
    Q = chain([hidden[-1], *[int(x) for x in cfg["q_hidden"]], A * N], True, False)
    V = chain([hidden[-1], *[int(x) for x in cfg["v_hidden"]], N], bool(cfg["v_noisy"]), False)
    return RainbowView(trunk, Q, V, A, N)


def net_from_golden(g) -> RainbowView:
    return rainbow_net({k[4:]: g[k] for k in g.files if k.startswith("cfg_")})


def noise_tensors(net: nn.Module) -> list[torch.Tensor]:
    """eps_p, eps_q of every noisy layer in ``modules()`` order: the order the draws happen in."""
    return [e for m in net.modules() if hasattr(m, "eps_p") for e in (m.eps_p, m.eps_q)]


def trainable(net: nn.Module) -> list[nn.Parameter]:
    return [p for p in net.parameters() if p.requires_grad]


def set_noise(net: nn.Module, flat: np.ndarray) -> None:
    """Write a concatenation of ``noise_tensors(net)`` into them."""
    off = 0
    with torch.no_grad():
        for e in noise_tensors(net):
            e.copy_(torch.as_tensor(flat[off:off + e.numel()], dtype=e.dtype))
            off += e.numel()
    assert off == len(flat), (off, len(flat))


def get_noise(net: nn.Module) -> np.ndarray:
    ts = noise_tensors(net)
    return np.concatenate([e.detach().cpu().numpy().reshape(-1) for e in ts]) if ts else np.zeros(0, np.float32)


def sample_noise(net: nn.Module) -> None:
    for m in net.modules():
        if hasattr(m, "sample"):
            m.sample()


# ------------------------------------------------------------------------------------------------ dueling combine, float64
def dueling(q: np.ndarray, v: np.ndarray) -> np.ndarray:
    """logits [B, A, N] = q - mean_a q + v from q [B, A, N] and v [B, N]."""
    q = np.asarray(q, np.float64)
    return q - q.mean(1, keepdims=True) + np.asarray(v, np.float64)[:, None, :]


def dueling_bwd(dl: np.ndarray) -> tuple[np.ndarray, np.ndarray]:
    """(dq [B, A, N], dv [B, N]) from d loss / d logits: dq = dl - mean_a dl, dv = sum_a dl."""
    dl = np.asarray(dl, np.float64)
    return dl - dl.mean(1, keepdims=True), dl.sum(1)


# ------------------------------------------------------------------------------------------------ update
class RainbowState(oc.C51State):
    """C51's state on a ``RainbowView``: the Adam optimiser lists the noise too, as the reference's does (it never gets state)."""

    def __init__(self, net: RainbowView, lr: float, freq: int, v_min: float, v_max: float):
        super().__init__(net, lr, freq, v_min, v_max)
        net.train()
        if self.old is not None:
            self.old.train()


def _tick(s: RainbowState, keep_lagged_noise: bool) -> None:
    if s.old is not None and s.iter % s.freq == 0:
        kept = get_noise(s.old)
        s.old.load_state_dict(s.net.state_dict())
        if keep_lagged_noise:
            set_noise(s.old, kept)
    s.iter += 1


def rainbow_update(s: RainbowState, obs_of: Callable[[np.ndarray], torch.Tensor], buf: dict, indices: np.ndarray,
                   is_weight: np.ndarray | None, gamma: float, n_step: int, noise_on: np.ndarray, noise_old: np.ndarray | None,
                   keep_lagged_noise: bool = False, target_eval: bool = False) -> dict:
    """One ``RainbowDQN.update`` on the sampled ``indices`` with the noise ``noise_on`` (online) and ``noise_old`` (lagged) as
    drawn: the forwards in torch fp32, the rows in float64 numpy, their gradient pushed back with autograd.
    ``keep_lagged_noise`` keeps the lagged network's own draw on a tick, ``target_eval`` forms the target with the mu weights
    (eval mode): neither is what the reference does."""
    dev = next(s.net.parameters()).device
    returns = oc._returns(s, buf, indices, gamma, n_step)
    set_noise(s.net, noise_on)
    if s.old is not None:
        set_noise(s.old, noise_old)
    _tick(s, keep_lagged_noise)
    nets = [s.net] + ([s.old] if s.old is not None else [])
    with torch.no_grad():
        for n in nets:
            n.train(not target_eval)
        x = obs_next_of(obs_of, buf, indices, dev)
        lo = s.net.logits(x)
        ln = s.old.logits(x) if s.old is not None else lo
        for n in nets:
            n.train()
    nd = oc.c51_target(lo.cpu().numpy(), ln.cpu().numpy(), s.z)
    logits = s.net.logits(obs_of(indices))
    act = np.asarray(buf["act"])[indices].astype(np.int64).reshape(-1)
    r = oc.c51_rows(logits.detach().cpu().numpy(), act, returns, s.z, s.v_min, s.v_max, s.delta_z, nd, is_weight)
    s.opt.zero_grad()
    logits.backward(torch.as_tensor(r["dlogits"], dtype=torch.float32, device=dev))
    s.opt.step()
    return dict(returns=returns, loss=r["loss"], prio=r["prio"])


def rainbow_update_torch(s: RainbowState, obs_of: Callable[[np.ndarray], torch.Tensor], buf: dict, indices: np.ndarray,
                         gamma: float, n_step: int) -> float:
    """The same update as the reference runs it in eager PyTorch: the n-step return on the host, the noise drawn with torch's
    ``randn`` (online, then lagged), the lagged refresh, the target and the loss in torch on the network's device, autograd,
    torch's Adam.  Returns the loss."""
    dev = next(s.net.parameters()).device
    z = torch.as_tensor(s.z, device=dev)
    returns = torch.as_tensor(oc._returns(s, buf, indices, gamma, n_step), device=dev)
    with torch.no_grad():
        sample_noise(s.net)
        if s.old is not None:
            sample_noise(s.old)
    _tick(s, False)
    with torch.no_grad():
        x = obs_next_of(obs_of, buf, indices, dev)
        dist = s.net(x)
        a = (dist * z).sum(2).argmax(1)
        nd = (s.old(x) if s.old is not None else dist)[torch.arange(len(indices), device=dev), a, :]
        target = oc.reference_target(nd, returns, z, s.v_min, s.v_max, s.delta_z)
    curr = s.net(obs_of(indices))
    act = torch.as_tensor(np.asarray(buf["act"])[indices].astype(np.int64), device=dev)
    loss = oc.reference_loss(curr, act, target, 1.0)[0]
    s.opt.zero_grad()
    loss.backward()
    s.opt.step()
    return loss.item()
