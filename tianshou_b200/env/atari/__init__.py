from .atari_network import DQNet, QRDQNet, ScaledObsInputActionReprNet, scale_obs

__all__ = ["DQNet", "QRDQNet", "ScaledObsInputActionReprNet", "scale_obs"]
