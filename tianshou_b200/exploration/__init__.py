from .random import BaseNoise, GaussianNoise, OUNoise

__all__ = ["BaseNoise", "GaussianNoise", "OUNoise"]
