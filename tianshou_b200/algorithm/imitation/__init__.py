from .bcq import BCQ, BCQPolicy, BCQTrainingStats
from .cql import CQL, CQLTrainingStats
from .gail import GAIL, GailTrainingStats
from .td3_bc import TD3BC

__all__ = ["BCQ", "BCQPolicy", "BCQTrainingStats", "CQL", "CQLTrainingStats", "GAIL", "GailTrainingStats", "TD3BC"]
