from .base import Algorithm, OfflineAlgorithm, OffPolicyAlgorithm, OnPolicyAlgorithm, Policy, TrainingStats
from .flat_params import UnsupportedModelError
from .imitation import (BCQ, CQL, GAIL, TD3BC, BCQPolicy, BCQTrainingStats, CQLTrainingStats, DiscreteBCQ, DiscreteBCQPolicy,
                        DiscreteBCQTrainingStats, DiscreteCQL, DiscreteCQLTrainingStats, DiscreteCRR, DiscreteCRRTrainingStats,
                        GailTrainingStats)
from .modelfree.a2c import A2CTrainingStats, ActorCriticOnPolicyAlgorithm
from .modelfree.discrete_sac import DiscreteSAC
from .modelfree.fqf import FQF, FQFPolicy, FQFTrainingStats
from .modelfree.iqn import IQN, IQNPolicy
from .modelfree.npg import NPG, NPGTrainingStats
from .modelfree.ppo import A2C, PPO
from .modelfree.qrdqn import QRDQN, QRDQNPolicy
from .modelfree.redq import REDQ, REDQPolicy, REDQTrainingStats
from .modelfree.reinforce import DiscreteActorPolicy, ProbabilisticActorPolicy
from .modelfree.td3 import TD3, TD3TrainingStats
from .modelfree.trpo import TRPO, TRPOTrainingStats
from .optim import AdamOptimizerFactory, LRSchedulerFactoryLinear, OptimizerFactory, RMSpropOptimizerFactory

__all__ = [
    "Algorithm", "OfflineAlgorithm", "OffPolicyAlgorithm", "OnPolicyAlgorithm", "Policy", "TrainingStats",
    "UnsupportedModelError", "A2CTrainingStats", "ActorCriticOnPolicyAlgorithm", "PPO", "A2C", "NPG", "TRPO", "NPGTrainingStats", "TRPOTrainingStats",
    "GAIL", "GailTrainingStats", "DiscreteSAC", "BCQ", "BCQPolicy", "BCQTrainingStats", "CQL", "CQLTrainingStats", "TD3", "TD3TrainingStats", "TD3BC",
    "ProbabilisticActorPolicy", "DiscreteActorPolicy", "AdamOptimizerFactory", "LRSchedulerFactoryLinear", "OptimizerFactory",
    "RMSpropOptimizerFactory", "DiscreteBCQ", "DiscreteBCQPolicy", "DiscreteBCQTrainingStats", "DiscreteCRR",
    "DiscreteCRRTrainingStats", "QRDQN", "QRDQNPolicy", "DiscreteCQL", "DiscreteCQLTrainingStats", "IQN", "IQNPolicy",
    "FQF", "FQFPolicy", "FQFTrainingStats", "REDQ", "REDQPolicy", "REDQTrainingStats",
]
