"""tianshou_b200 -- H100-native policy-update hot path behind Tianshou's Batch / ReplayBuffer /
Algorithm / Policy API (reference: thu-ml/tianshou 2.0.1).  See DESIGN.md."""
__version__ = "0.1.0"

from . import data  # noqa: F401
