"""TD3+BC (arXiv:2106.06860): offline TD3 whose actor loss adds behaviour cloning, with the whole ``update()`` on the device.

Reference: tianshou/algorithm/imitation/td3_bc.py (TD3BC :14-127), algorithm_base.py:906-951 (OfflineAlgorithm).  Everything but
the actor loss is TD3's (modelfree/td3.py); ``ts_td3_actor_rows`` computes ``lmbda = alpha / mean|Q1(s, pi(s))|`` on the device,
so the update still reads its losses once, at its end.
"""
from __future__ import annotations

import torch
from torch import nn

from ...data import Batch
from ..base import OfflineAlgorithm
from ..modelfree.ddpg import ContinuousDeterministicPolicy
from ..modelfree.td3 import TD3, TD3TrainingStats
from ..optim import OptimizerFactory


class TD3BC(OfflineAlgorithm, TD3):
    """TD3+BC (td3_bc.py:14-127): TD3 on a fixed buffer whose actor loss is
    ``-lmbda * mean(Q1(s, pi(s))) + mean((pi(s) - batch.act)^2)`` with ``lmbda = alpha / mean|Q1(s, pi(s))|`` detached; the MSE
    averages over the B * A elements (``F.mse_loss``)."""

    def __init__(self, *, policy: ContinuousDeterministicPolicy, policy_optim: OptimizerFactory, critic: nn.Module,
                 critic_optim: OptimizerFactory, critic2: nn.Module | None = None, critic2_optim: OptimizerFactory | None = None,
                 tau: float = 0.005, gamma: float = 0.99, policy_noise: float = 0.2, update_actor_freq: int = 2,
                 noise_clip: float = 0.5, alpha: float = 2.5, n_step_return_horizon: int = 1) -> None:
        TD3.__init__(self, policy=policy, policy_optim=policy_optim, critic=critic, critic_optim=critic_optim, critic2=critic2,
                     critic2_optim=critic2_optim, tau=tau, gamma=gamma, policy_noise=policy_noise, noise_clip=noise_clip,
                     update_actor_freq=update_actor_freq, n_step_return_horizon=n_step_return_horizon)
        self.alpha = alpha

    def _bc_terms(self, batch: Batch) -> tuple[torch.Tensor | None, float]:
        return batch.act, float(self.alpha)

    def _update_with_batch(self, batch: Batch) -> TD3TrainingStats:
        return TD3._update_with_batch(self, batch)
