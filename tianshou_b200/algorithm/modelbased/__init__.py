from .icm import ICMOffPolicyWrapper, ICMOnPolicyWrapper, ICMTrainingStats
from .psrl import PSRL, PSRLModel, PSRLPolicy, PSRLTrainingStats

__all__ = ["ICMOffPolicyWrapper", "ICMOnPolicyWrapper", "ICMTrainingStats", "PSRL", "PSRLModel", "PSRLPolicy", "PSRLTrainingStats"]
