"""stardist_b200 -- H100-native (sm_90a) implementation of StarDist's prediction hot path.

Public surface mirrors the reference package (`stardist`): StarDist2D / Config2D,
non_maximum_suppression*, polygons_to_label, dist_to_coord, ... .  All compute runs in
hand-written CUDA kernels behind the C ABI of include/stardist_b200.h; there is no CPU fallback.
"""
__version__ = "0.1.0"

from .nms import (non_maximum_suppression, non_maximum_suppression_sparse, non_maximum_suppression_inds,
                  non_maximum_suppression_3d, non_maximum_suppression_3d_sparse, non_maximum_suppression_3d_inds)
from .geometry import (ray_angles, dist_to_coord, polygons_to_label, polygons_to_label_coord,
                       polyhedron_to_label, dist_to_coord3D, star_dist, star_dist3D, relabel_image_stardist,
                       relabel_image_stardist3D)
from .rays3d import Rays_GoldenSpiral, Rays_Explicit, Rays_Cartesian, Rays_SubDivide, Rays_Tetra, Rays_Octo, rays_from_json
from .matching import relabel_sequential
from .models import Config2D, StarDist2D, Config3D, StarDist3D
from .utils import normalize, calculate_extents, edt_prob, fill_label_holes, sample_points
from .sample_patches import sample_patches
from .io.rois import export_imagej_rois
