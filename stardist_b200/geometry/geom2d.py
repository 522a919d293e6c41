"""2D geometry of the prediction path, device backed.

Mirrors stardist/geometry/geom2d.py: ray_angles (:214), dist_to_coord (:130-146),
polygons_to_label_coord (:149-166), polygons_to_label (:169-197).  numpy in, numpy out; the
work runs in the CUDA kernels of csrc/label2d.cu.
"""
import numpy as np
import torch
from .. import _lib as L
from ..utils import _raise
from .distances import star_dist_device, label_map_to_device, centroids_device, check_points_in, output_shape, _check_grid


def ray_angles(n_rays=32):
    return np.linspace(0, 2 * np.pi, n_rays, endpoint=False)


def _sincos_table(n_rays, device):
    phis = ray_angles(n_rays)
    tab = np.concatenate([np.sin(phis), np.cos(phis)]).astype(np.float64)
    return torch.from_numpy(tab).to(device)


def dist_to_coord_device(dist_d, points_f64_d, scale_dist=(1, 1)):
    """dist_d float32[n,R], points_f64_d float64[n,2] on the device -> coord float32[n,2,R] (device)"""
    lib = L.require_cuda()
    n, R = dist_d.shape
    coord = torch.empty((n, 2, R), dtype=torch.float32, device=dist_d.device)
    if n > 0:
        tab = _sincos_table(R, dist_d.device)
        L.check(lib.sdb_dist_to_coord_2d(L.ptr(dist_d), L.ptr(points_f64_d), n, R, L.ptr(tab),
                                        float(scale_dist[0]), float(scale_dist[1]),
                                        L.ptr(coord), L.stream_ptr()))
    return coord


def dist_to_coord(dist, points, scale_dist=(1, 1)):
    """convert from polar to cartesian coordinates for a list of distances and center points
    dist.shape   = (n_polys, n_rays)
    points.shape = (n_polys, 2)
    len(scale_dist) = 2
    return coord.shape = (n_polys,2,n_rays)
    """
    dist = np.asarray(dist)
    points = np.asarray(points)
    assert dist.ndim == 2 and points.ndim == 2 and len(dist) == len(points) \
        and points.shape[1] == 2 and len(scale_dist) == 2
    L.require_cuda()
    dev = torch.device("cuda")
    d = torch.from_numpy(np.ascontiguousarray(dist, dtype=np.float32)).to(dev)
    p = torch.from_numpy(np.ascontiguousarray(points, dtype=np.float64)).to(dev)
    return dist_to_coord_device(d, p, scale_dist).cpu().numpy()


def polygons_to_label_coord(coord, shape, labels=None):
    """renders polygons to image of given shape

    coord.shape   = (n_polys, 2, n_rays)
    """
    coord = np.asarray(coord)
    if labels is None:
        labels = np.arange(len(coord))
    labels = np.asarray(labels)
    if not (labels.ndim == 1 and np.issubdtype(labels.dtype, np.integer)):
        raise ValueError("labels must be an array of integers")
    assert coord.ndim == 3 and coord.shape[1] == 2 and len(coord) == len(labels)
    lib = L.require_cuda()
    n, _, R = coord.shape
    out = np.zeros(tuple(int(s) for s in shape), np.int32)
    c = np.ascontiguousarray(coord, dtype=np.float32)
    lab = np.ascontiguousarray(labels, dtype=np.int32)
    L.check(lib._LIB_polygons_to_label_2d(L.ptr(c), L.ptr(lab), n, R, out.shape[0], out.shape[1], L.ptr(out)))
    return out


def paint_order(prob):
    """np.argsort(prob, kind='stable') (geom2d.py:191) -> (ind, rank)"""
    ind = np.argsort(prob, kind='stable')
    rank = np.empty_like(ind)
    rank[ind] = np.arange(len(ind))
    return ind, rank


def polygons_to_label(dist, points, shape, prob=None, thr=-np.inf, scale_dist=(1, 1)):
    """converts distances and center points to label image

    dist.shape   = (n_polys, n_rays)
    points.shape = (n_polys, 2)

    label ids will be consecutive and adhere to the order given
    """
    dist = np.asarray(dist)
    points = np.asarray(points)
    prob = np.inf * np.ones(len(points)) if prob is None else np.asarray(prob)
    assert dist.ndim == 2 and points.ndim == 2 and len(dist) == len(points)
    assert len(points) == len(prob) and points.shape[1] == 2 and prob.ndim == 1
    ind = prob > thr
    points = points[ind]
    dist = dist[ind]
    prob = prob[ind]
    ind = np.argsort(prob, kind='stable')
    points = points[ind]
    dist = dist[ind]
    coord = dist_to_coord(dist, points, scale_dist=scale_dist)
    return polygons_to_label_coord(coord, shape=shape, labels=ind)


def star_dist(a, n_rays=32, grid=(1, 1), mode='cpp'):
    """'a' assumbed to be a label image with integer values that encode object ids. id 0 denotes background.

    Star distances float32 [(H-1)//grid[0]+1, (W-1)//grid[1]+1, n_rays] (stardist/geometry/geom2d.py:80-92), bit-identical
    to the reference's C++.  Modes 'cpp' and 'opencl' both run the CUDA kernel with the C++ semantics; there is no 'python'
    mode (no CPU fallback)."""
    n_rays >= 3 or _raise(ValueError("need 'n_rays' >= 3"))
    if mode == 'python':
        raise NotImplementedError("star_dist: mode 'python' has no CPU implementation here; use 'cpp'")
    if mode not in ('cpp', 'opencl'):
        raise ValueError("Unknown mode %s" % mode)
    (np.isscalar(n_rays) and 0 < int(n_rays)) or _raise(ValueError())
    L.require_cuda()
    a = np.asarray(a).astype(np.uint16, copy=False)
    if a.ndim != 2:
        raise ValueError("star_dist: label image must be 2-dimensional")
    d = torch.from_numpy(np.ascontiguousarray(a)).to("cuda")
    return star_dist_device(d, int(n_rays), grid).cpu().numpy()


def relabel_image_stardist(lbl, n_rays, **kwargs):
    """relabel each label region in `lbl` with its star representation (stardist/geometry/geom2d.py:200-211): the polygon of
    n_rays star distances at each region's centroid, painted with polygons_to_label.  Centroids, the distances at the
    centroids and the painting stay on the device; `kwargs` (grid) as in star_dist, including the reference's indexing of
    the subsampled map with full-resolution centroids (IndexError where numpy raises)."""
    from ..matching import _check_label_array
    _check_label_array(lbl, "lbl")
    if not lbl.ndim == 2:
        raise ValueError("lbl image should be 2 dimensional")
    n_rays >= 3 or _raise(ValueError("need 'n_rays' >= 3"))
    mode = kwargs.pop('mode', 'cpp')
    grid = tuple(kwargs.pop('grid', (1, 1)))
    if kwargs:
        raise TypeError("unexpected keyword arguments %s" % sorted(kwargs))
    if mode == 'python':
        raise NotImplementedError("star_dist: mode 'python' has no CPU implementation here; use 'cpp'")
    lib = L.require_cuda()
    seq, n, labels = label_map_to_device(lbl)
    d_lbl = torch.from_numpy(np.ascontiguousarray(lbl.astype(np.uint16, copy=False))).to("cuda")
    points = centroids_device(seq, n) if n > 0 else torch.zeros((0, 2), dtype=torch.int32, device="cuda")
    check_points_in(points, output_shape(lbl.shape, _check_grid(grid, 2)))
    dist = star_dist_device(d_lbl, int(n_rays), grid, points=points)
    ny, nx = lbl.shape
    out = torch.empty((ny, nx), dtype=torch.int32, device="cuda")
    # polygons_to_label(dist, points, shape): all scores infinite, so the stable order is the region order and ids are 1..n
    coord = dist_to_coord_device(dist, points.to(torch.float64)) if n > 0 else torch.zeros((0, 2, int(n_rays)), device="cuda")
    order = torch.arange(n, dtype=torch.int32, device="cuda")
    ids = order + 1
    L.check(lib.sdb_polygons_to_label_2d(L.ptr(coord), L.ptr(order), L.ptr(ids), n, int(n_rays), ny, nx, L.ptr(out), L.stream_ptr()))
    return out.cpu().numpy()

