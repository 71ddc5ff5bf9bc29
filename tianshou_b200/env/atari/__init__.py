from .atari_network import C51Net, DQNet, QRDQNet, RainbowNet, ScaledObsInputActionReprNet, scale_obs

__all__ = ["C51Net", "DQNet", "QRDQNet", "RainbowNet", "ScaledObsInputActionReprNet", "scale_obs"]
