from .cql import CQL, CQLTrainingStats
from .gail import GAIL, GailTrainingStats

__all__ = ["CQL", "CQLTrainingStats", "GAIL", "GailTrainingStats"]
