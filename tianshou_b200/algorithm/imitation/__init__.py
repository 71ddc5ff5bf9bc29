from .bcq import BCQ, BCQPolicy, BCQTrainingStats
from .cql import CQL, CQLTrainingStats
from .discrete_bcq import DiscreteBCQ, DiscreteBCQPolicy, DiscreteBCQTrainingStats
from .discrete_crr import DiscreteCRR, DiscreteCRRTrainingStats
from .gail import GAIL, GailTrainingStats
from .td3_bc import TD3BC

__all__ = ["BCQ", "BCQPolicy", "BCQTrainingStats", "CQL", "CQLTrainingStats", "DiscreteBCQ", "DiscreteBCQPolicy",
           "DiscreteBCQTrainingStats", "DiscreteCRR", "DiscreteCRRTrainingStats", "GAIL", "GailTrainingStats", "TD3BC"]
