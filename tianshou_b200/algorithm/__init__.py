from .base import Algorithm, OffPolicyAlgorithm, OnPolicyAlgorithm, Policy, TrainingStats
from .flat_params import UnsupportedModelError
from .imitation import GAIL, GailTrainingStats
from .modelfree.a2c import A2CTrainingStats, ActorCriticOnPolicyAlgorithm
from .modelfree.npg import NPG, NPGTrainingStats
from .modelfree.ppo import A2C, PPO
from .modelfree.reinforce import DiscreteActorPolicy, ProbabilisticActorPolicy
from .modelfree.trpo import TRPO, TRPOTrainingStats
from .optim import AdamOptimizerFactory, LRSchedulerFactoryLinear, OptimizerFactory, RMSpropOptimizerFactory

__all__ = [
    "Algorithm", "OffPolicyAlgorithm", "OnPolicyAlgorithm", "Policy", "TrainingStats",
    "UnsupportedModelError", "A2CTrainingStats", "ActorCriticOnPolicyAlgorithm", "PPO", "A2C", "NPG", "TRPO", "NPGTrainingStats", "TRPOTrainingStats",
    "GAIL", "GailTrainingStats",
    "ProbabilisticActorPolicy", "DiscreteActorPolicy", "AdamOptimizerFactory", "LRSchedulerFactoryLinear", "OptimizerFactory",
    "RMSpropOptimizerFactory",
]
