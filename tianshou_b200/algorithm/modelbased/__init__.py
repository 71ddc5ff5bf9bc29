from .icm import ICMOffPolicyWrapper, ICMOnPolicyWrapper, ICMTrainingStats

__all__ = ["ICMOffPolicyWrapper", "ICMOnPolicyWrapper", "ICMTrainingStats"]
