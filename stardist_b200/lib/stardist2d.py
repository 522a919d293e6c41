"""Drop-in for `stardist.lib.stardist2d` (reference: stardist/lib/stardist2d.cpp:621-632).

c_non_max_suppression_inds(dist f32[n,R] C-contig, points f32[n,2], use_kdtree:int, use_bbox:int,
                           verbose:int, thresh:f32) -> bool[n]         ("O!O!iiif", stardist2d.cpp:396)
Inputs must be sorted by descending score (as stardist/nms.py:186-227 guarantees).
c_star_dist(src uint16[H,W], n_rays:int, grid_y:int, grid_x:int) -> float32[(H-1)//grid_y+1, (W-1)//grid_x+1, n_rays]
                                                                     ("O!iii", stardist2d.cpp:55-125)
"""
import numpy as np
from .. import _lib as L


def c_non_max_suppression_inds(dist, points, use_kdtree, use_bbox, verbose, thresh):
    if not (isinstance(dist, np.ndarray) and isinstance(points, np.ndarray)):
        raise TypeError("dist and points must be numpy arrays")
    if dist.dtype != np.float32 or points.dtype != np.float32:
        raise TypeError("dist and points must be float32")
    if dist.ndim != 2 or points.ndim != 2 or points.shape[1] != 2 or points.shape[0] != dist.shape[0]:
        raise ValueError("expected dist (n,R) and points (n,2)")
    lib = L.require_cuda()
    dist = np.ascontiguousarray(dist); points = np.ascontiguousarray(points)
    n, R = dist.shape
    result = np.zeros(n, dtype=np.bool_)
    if n > 0:
        L.check(lib._LIB_non_maximum_suppression_2d(L.ptr(dist), L.ptr(points), n, R, float(thresh),
                                                   int(use_bbox), int(use_kdtree), int(verbose), L.ptr(result)))
    return result


def c_star_dist(src, n_rays, grid_y, grid_x):
    from ..geometry.distances import direction_table_2d, walk_bound, output_shape
    if not isinstance(src, np.ndarray):
        raise TypeError("src must be a numpy array")
    if src.dtype != np.uint16 or src.ndim != 2:
        raise TypeError("src must be a 2-dimensional uint16 array")
    n_rays, gy, gx = int(n_rays), int(grid_y), int(grid_x)
    if n_rays < 1 or gy < 1 or gx < 1:
        raise ValueError("n_rays, grid_y and grid_x must be >= 1")
    lib = L.require_cuda()
    dirs = np.ascontiguousarray(direction_table_2d(n_rays))
    walk_bound(dirs, src.shape)
    src = np.ascontiguousarray(src)
    dst = np.empty(output_shape(src.shape, (gy, gx)) + (n_rays,), np.float32)
    lib._LIB_star_dist_2d(L.ptr(src), src.shape[0], src.shape[1], n_rays, gy, gx, L.ptr(dirs), L.ptr(dst))
    msg = lib.sdb_last_error()
    if msg:
        raise L.StarDistB200Error(msg.decode("utf-8", "replace"))
    return dst
