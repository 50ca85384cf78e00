"""`import voxelmorph as vxm` for the unmodified reference scripts (scripts/torch/train.py, register.py):
the import surface of the reference package (voxelmorph/__init__.py:20-44) re-exported from `voxelmorph_b200`,
whose operators are hand-written sm_90a kernels behind the C ABI of include/vxm_b200.h.

    os.environ['VXM_BACKEND'] = 'pytorch'; import voxelmorph as vxm
    vxm.networks.VxmDense, vxm.layers.{SpatialTransformer,VecInt,ResizeTransform}, vxm.losses.{NCC,MSE,Dice,Grad},
    vxm.generators.{volgen,scan_to_scan,scan_to_atlas,semisupervised}, vxm.py.utils.*, vxm.torch.*, vxm.default_unet_features

Only the pytorch backend exists here (the reference's default, tensorflow, is a different framework and out of
scope): importing without VXM_BACKEND=pytorch fails loudly instead of silently picking another implementation.
Through this package the U-Net runs on the tensor-core engine by default (VXM_B200_CONV_ENGINE overrides), and
under torchrun (RANK / WORLD_SIZE in the environment) a VxmDense becomes data parallel transparently
(voxelmorph_b200/dist.py: parameter broadcast, one gradient allreduce per backward, rank-0-only save).
"""
import os

__version__ = '0.2'

from . import py                         # noqa: E402
from .py.utils import default_unet_features   # noqa: E402,F401

backend = py.utils.get_backend()
if backend != 'pytorch':
    raise ImportError("this voxelmorph build (voxelmorph_b200, H100 / sm_90a) provides the pytorch backend only: "
                      "set the VXM_BACKEND environment variable to 'pytorch' before importing voxelmorph")
os.environ['NEURITE_BACKEND'] = 'pytorch'

import voxelmorph_b200 as _impl          # noqa: E402

_impl.ops.set_default_engine('tc')       # tensor cores unless VXM_B200_CONV_ENGINE says otherwise

from . import generators                 # noqa: E402,F401
from . import torch                      # noqa: E402,F401
from .torch import layers                # noqa: E402,F401
from .torch import networks              # noqa: E402,F401
from .torch import losses                # noqa: E402,F401
