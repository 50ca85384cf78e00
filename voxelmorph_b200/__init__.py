"""voxelmorph_b200 — H100-native (sm_90a) VxmDense registration path.

Mirrors the torch backend of voxelmorph (`voxelmorph.torch.{layers,networks,losses,modelio}`)
class for class; every operator runs in a hand-written CUDA kernel reached through the
C ABI declared in include/vxm_b200.h (libvxm_b200.so).  No CPU or torch-operator fallback.
"""
__version__ = '0.1'

from . import _lib
from . import layers
from . import networks
from . import losses
from . import modelio
from . import optim
from . import dist
from . import generators
from . import utils
from .networks import default_unet_features

__all__ = ["layers", "networks", "losses", "modelio", "optim", "dist", "generators", "utils", "default_unet_features"]
