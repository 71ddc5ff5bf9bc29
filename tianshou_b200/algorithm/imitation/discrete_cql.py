"""Discrete conservative Q-learning (arXiv:2006.04779) on QR-DQN, with the whole ``update()`` on the device.

Reference: tianshou/algorithm/imitation/discrete_cql.py (DiscreteCQLTrainingStats :17-19, DiscreteCQL :23-113),
examples/offline/atari_cql.py and test/offline/test_discrete_cql.py (a ``QRDQNet`` / ``Net(num_atoms)`` quantile network).

The update is QR-DQN's (modelfree/qrdqn.py) with ``min_q_weight`` handed to ``ts_qrdqn_rows``, which adds the log-sum-exp
penalty over the quantile means and its gradient to every quantile of every action.
"""
from __future__ import annotations

from dataclasses import dataclass

from ...data import Batch
from ..base import OfflineAlgorithm
from ..modelfree.dqn import SimpleLossTrainingStats
from ..modelfree.qrdqn import QRDQN, QRDQNPolicy
from ..optim import OptimizerFactory


@dataclass(kw_only=True)
class DiscreteCQLTrainingStats(SimpleLossTrainingStats):
    cql_loss: float
    qr_loss: float


class DiscreteCQL(OfflineAlgorithm, QRDQN):
    """Discrete CQL, reference API and semantics (discrete_cql.py:23-113), with the reference's diamond: an offline algorithm
    that is also a ``QRDQN``.

    loss = qr_loss + min_q_weight * cql_loss, with qr_loss QR-DQN's importance-weighted quantile-Huber loss and cql_loss =
    mean_b(logsumexp_a m_a - m_act) over the quantile means m; the importance weight scales the quantile term only.  With
    ``min_q_weight == 0`` the penalty is neither computed nor reported (``cql_loss`` is 0); a negative weight is refused.
    """

    def __init__(self, *, policy: QRDQNPolicy, optim: OptimizerFactory, min_q_weight: float = 10.0, gamma: float = 0.99,
                 num_quantiles: int = 200, n_step_return_horizon: int = 1, target_update_freq: int = 0) -> None:
        QRDQN.__init__(self, policy=policy, optim=optim, gamma=gamma, num_quantiles=num_quantiles,
                       n_step_return_horizon=n_step_return_horizon, target_update_freq=target_update_freq)
        if min_q_weight < 0:
            raise ValueError(f"min_q_weight must be >= 0, got {min_q_weight}")
        self.min_q_weight = min_q_weight

    def _update_with_batch(self, batch: Batch) -> DiscreteCQLTrainingStats:
        l = self._quantile_step(batch, self.min_q_weight)
        return DiscreteCQLTrainingStats(loss=float(l[0]), qr_loss=float(l[1]), cql_loss=float(l[2]))
