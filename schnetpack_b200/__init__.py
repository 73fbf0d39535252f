"""schnetpack_b200 -- H100-native (sm_90a) implementation of SchNetPack's message-passing hot path.

Drop-in module mirrors (same constructor signatures, tensor-dict protocol and ``state_dict`` keys as the reference):
``representation.{PaiNN,SchNet}``, ``nn.{GaussianRBF,BesselRBF,CosineCutoff,Dense,shifted_softplus,scatter_add,...}``,
``atomistic.{PairwiseDistances,Atomwise,Forces}``, ``model.{NeuralNetworkPotential,convert_model,GraphedPotential}``;
callers either side of the path: ``neighbors.CellListNeighborList`` (device-resident neighbour list), ``md.DeviceMD``
(CUDA-graph velocity-Verlet step), ``relax.DeviceLBFGS`` (batchwise L-BFGS relaxation in a CUDA graph), ``neb.DeviceNEB``
(climbing-image nudged elastic band, every image of every band in one captured step), ``parallel``
(batch sharding, graph partition + halo exchange), ``structure`` (radial distribution functions and mean-squared
displacements accumulated inside the captured MD step), ``exchange`` (temperature replica exchange in the captured MD
step).
All arithmetic runs in the hand-written CUDA library ``csrc/libspk_b200.so`` (C ABI: ``include/spk_b200.h``).
"""
from . import properties  # noqa: F401
from . import nn  # noqa: F401
from . import representation  # noqa: F401
from . import atomistic  # noqa: F401
from . import model  # noqa: F401
from . import neighbors  # noqa: F401
from . import md  # noqa: F401
from . import structure  # noqa: F401
from . import exchange  # noqa: F401
from . import relax  # noqa: F401
from . import neb  # noqa: F401
from . import parallel  # noqa: F401
from .model import GraphedPotential, NeuralNetworkPotential, convert_model  # noqa: F401

__version__ = "0.1.0"
