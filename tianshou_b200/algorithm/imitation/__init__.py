from .gail import GAIL, GailTrainingStats

__all__ = ["GAIL", "GailTrainingStats"]
