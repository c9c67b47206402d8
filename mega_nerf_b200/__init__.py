"""H100-native drop-in for the Mega-NeRF rendering hot path.

Mirrors the reference's Python call surface (mega_nerf/rendering.py, ray_utils.py, models/*.py) on top
of libmn_b200.so (hand-written sm_90a CUDA behind the C ABI in include/mn_b200.h).
"""
from .modules import (Embedding, ShiftedSoftplus, NeRF, MegaNeRF, Cascade, get_nerf, get_bg_nerf,  # noqa: F401
                      set_precision, get_precision, set_train_precision, get_train_precision)
from .render import render_rays, render_rays_fused, render_rays_train  # noqa: F401
from .graph import GraphedRenderRays, GraphedTrainStep  # noqa: F401
from .raygen import get_ray_directions, get_rays, get_rays_batch  # noqa: F401
from .sh import eval_sh  # noqa: F401
from .install import install  # noqa: F401
from . import cluster_masks  # noqa: F401
from . import octree  # noqa: F401
from . import expert_parallel  # noqa: F401
