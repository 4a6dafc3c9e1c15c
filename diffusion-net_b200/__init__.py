"""H100-native (sm_90a) DiffusionNetBlock hot path behind the reference module API.

Public surface mirrors ``diffusion_net`` (reference ``src/diffusion_net/__init__.py:1-3``):
``layers`` (DiffusionNet, DiffusionNetBlock, LearnedTimeDiffusion, SpatialGradientFeatures,
MiniMLP) and ``geometry`` (to_basis / from_basis).  ``ops.set_engine`` picks the arithmetic of
the dense contractions; ``_lib.build`` compiles the in-tree C-ABI library.
"""
__version__ = "0.1.0"

from . import _lib, ops, geometry, layers, synthetic, streaming, dist, graphs, batch, fmaps  # noqa: F401,E402
from .layers import (DiffusionNet, DiffusionNetBlock, LearnedTimeDiffusion,  # noqa: F401,E402
                     SpatialGradientFeatures, MiniMLP)
from .fmaps import (FunctionalMapCorrespondenceWithDiffusionNetFeatures, compute_correspondence,  # noqa: F401,E402
                    pointwise_map, PairBatch, PairDataset, pointwise_map_batch)
from .geometry import to_basis, from_basis  # noqa: F401,E402
from .ops import set_engine, get_engine, prepare_operators  # noqa: F401,E402
from .batch import BatchSlot, MeshBatch, MeshDataset  # noqa: F401,E402
