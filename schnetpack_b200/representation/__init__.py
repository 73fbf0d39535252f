from .painn import PaiNN, PaiNNInteraction, PaiNNMixing
from .schnet import SchNet, SchNetInteraction
from .so3net import SO3net

__all__ = ["PaiNN", "PaiNNInteraction", "PaiNNMixing", "SchNet", "SchNetInteraction", "SO3net"]
