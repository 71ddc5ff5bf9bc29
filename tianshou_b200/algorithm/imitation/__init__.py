from .bcq import BCQ, BCQPolicy, BCQTrainingStats
from .cql import CQL, CQLTrainingStats
from .discrete_bcq import DiscreteBCQ, DiscreteBCQPolicy, DiscreteBCQTrainingStats
from .discrete_cql import DiscreteCQL, DiscreteCQLTrainingStats
from .discrete_crr import DiscreteCRR, DiscreteCRRTrainingStats
from .gail import GAIL, GailTrainingStats
from .imitation_base import ImitationPolicy, ImitationTrainingStats, OfflineImitationLearning, OffPolicyImitationLearning
from .td3_bc import TD3BC

__all__ = ["BCQ", "BCQPolicy", "BCQTrainingStats", "CQL", "CQLTrainingStats", "DiscreteBCQ", "DiscreteBCQPolicy",
           "DiscreteBCQTrainingStats", "DiscreteCQL", "DiscreteCQLTrainingStats", "DiscreteCRR", "DiscreteCRRTrainingStats", "GAIL", "GailTrainingStats", "ImitationPolicy",
           "ImitationTrainingStats", "OfflineImitationLearning", "OffPolicyImitationLearning", "TD3BC"]
