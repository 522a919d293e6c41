"""Drop-in for `stardist.lib.stardist3d` (reference: stardist/lib/stardist3d.cpp:351-378).

c_non_max_suppression_inds(dist f32[n,R], points f32[n,3], verts f32[R,3], faces i32[F,3], scores f32[n],
                           use_bbox:int, use_kdtree:int, verbose:int, thresh:f32) -> bool[n]
                                                        ("O!O!O!O!O!iiif", stardist3d.cpp:23)
   NOTE: bbox/kdtree order is swapped relative to the 2D entry point, as in the reference.
c_polyhedron_to_label(dist, points, verts, faces, labels i32[n], render_mode:int, verbose:int,
                      use_overlap_label:int, overlap_label:int, (nz,ny,nx)) -> int32[nz,ny,nx]
                                                        ("O!O!O!O!O!iiii(iii)", stardist3d.cpp:93)
c_star_dist3d(src uint16[D,H,W], dz, dy, dx float32[n_rays], n_rays:int, grid_z:int, grid_y:int, grid_x:int)
                      -> float32[(D-1)//grid_z+1, (H-1)//grid_y+1, (W-1)//grid_x+1, n_rays]
                                                        ("O!O!O!O!iiii", stardist3d.cpp:245-345)
Inputs must be sorted by descending score.  Backed by the reference-signature C ABI
_LIB_non_maximum_suppression_sparse / _LIB_polyhedron_to_label of libstardist_b200.so.
"""
import ctypes
import numpy as np
from .. import _lib as L

_P = ctypes.c_void_p


def _chk(a, dtype, ndim, name):
    if not isinstance(a, np.ndarray): raise TypeError("%s must be a numpy array" % name)
    if a.dtype != dtype: raise TypeError("%s must be %s" % (name, np.dtype(dtype).name))
    if a.ndim != ndim: raise ValueError("%s must be %d-dimensional" % (name, ndim))
    return np.ascontiguousarray(a)


def _raise_on_error(lib):
    """the reference-signature entry points return void: a failure zeroes the result and leaves its message behind"""
    msg = lib.sdb_last_error()
    if msg:
        raise L.StarDistB200Error(msg.decode("utf-8", "replace"))


def c_non_max_suppression_inds(dist, points, verts, faces, scores, use_bbox, use_kdtree, verbose, thresh):
    dist = _chk(dist, np.float32, 2, "dist"); points = _chk(points, np.float32, 2, "points")
    verts = _chk(verts, np.float32, 2, "verts"); faces = _chk(faces, np.int32, 2, "faces")
    scores = _chk(scores, np.float32, 1, "scores")
    n, R = dist.shape
    if points.shape != (n, 3) or verts.shape != (R, 3) or faces.shape[1] != 3 or len(scores) != n:
        raise ValueError("inconsistent shapes")
    if R > 256 or len(faces) > 512 or R < 4:
        raise ValueError("stardist_b200: between 4 and 256 rays and at most 512 faces are supported (got %d / %d)" % (R, len(faces)))
    lib = L.require_cuda()
    result = np.zeros(n, np.bool_)
    f = lib._LIB_non_maximum_suppression_sparse
    f.restype = None
    f.argtypes = [_P, _P, _P, ctypes.c_int, ctypes.c_int, ctypes.c_int, _P, _P, ctypes.c_float, ctypes.c_int, ctypes.c_int, ctypes.c_int, _P]
    if n > 0:
        f(L.ptr(scores), L.ptr(dist), L.ptr(points), n, R, len(faces), L.ptr(verts), L.ptr(faces), float(thresh),
          int(use_bbox), int(use_kdtree), int(verbose), L.ptr(result))
        _raise_on_error(lib)
    return result


def c_polyhedron_to_label(dist, points, verts, faces, labels, render_mode, verbose, use_overlap_label, overlap_label, shape):
    dist = _chk(dist, np.float32, 2, "dist"); points = _chk(points, np.float32, 2, "points")
    verts = _chk(verts, np.float32, 2, "verts"); faces = _chk(faces, np.int32, 2, "faces")
    labels = _chk(labels, np.int32, 1, "labels")
    n, R = dist.shape
    nz, ny, nx = (int(s) for s in shape)
    if R > 256 or len(faces) > 512:      # static shared-memory limits of the kernels (the reference has none)
        raise ValueError("stardist_b200: at most 256 rays / 512 faces are supported (got %d / %d)" % (R, len(faces)))
    lib = L.require_cuda()
    result = np.zeros((nz, ny, nx), np.int32)
    f = lib._LIB_polyhedron_to_label
    f.restype = None
    f.argtypes = [_P, _P, _P, _P] + [ctypes.c_int] * 3 + [_P] + [ctypes.c_int] * 7 + [_P]
    f(L.ptr(dist), L.ptr(points), L.ptr(verts), L.ptr(faces), n, R, len(faces), L.ptr(labels), nz, ny, nx,
      int(render_mode), int(verbose), int(use_overlap_label), int(overlap_label), L.ptr(result))
    _raise_on_error(lib)
    return result


def c_star_dist3d(src, dz, dy, dx, n_rays, grid_z, grid_y, grid_x):
    from ..geometry.distances import walk_bound, output_shape
    src = _chk(src, np.uint16, 3, "src")
    n_rays = int(n_rays)
    comps = [_chk(a, np.float32, 1, name) for a, name in ((dz, "dz"), (dy, "dy"), (dx, "dx"))]
    if n_rays < 1 or any(len(a) < n_rays for a in comps):
        raise ValueError("n_rays must be >= 1 and dz, dy, dx must hold n_rays values each")
    grid = tuple(int(g) for g in (grid_z, grid_y, grid_x))
    if min(grid) < 1:
        raise ValueError("grid values must be >= 1")
    lib = L.require_cuda()
    rays = np.ascontiguousarray(np.stack([a[:n_rays] for a in comps]))
    walk_bound(rays, src.shape)
    dst = np.empty(output_shape(src.shape, grid) + (n_rays,), np.float32)
    lib._LIB_star_dist_3d(L.ptr(src), *src.shape, n_rays, *grid, L.ptr(rays), L.ptr(dst))
    _raise_on_error(lib)
    return dst
