"""Star distances and region statistics on the device (csrc/stardist.cu).

The reference computes the 2-D ray directions in its C++ as `const float dy = cos(phi)` with a float `phi`, which
resolves to libm's single-precision cosf / sinf.  Those are not correctly rounded, and no other routine (numpy, CUDA's
cosf, a float64 cos rounded to float32) agrees with them on every entry.  So the table is built here at run time with the
process's own libm, the library the reference extension links too.
"""
import ctypes, ctypes.util, functools
import numpy as np
from .. import _lib as L


@functools.lru_cache(maxsize=None)
def _libm():
    m = ctypes.CDLL(ctypes.util.find_library("m") or "libm.so.6")
    for f in (m.cosf, m.sinf):
        f.argtypes = [ctypes.c_float]
        f.restype = ctypes.c_float
    return m


@functools.lru_cache(maxsize=64)
def _direction_table_2d(n_rays):
    m = _libm()
    st = np.float32((2 * np.pi) / n_rays)                      # const float st_rays = (2*M_PI) / n_rays
    phi = np.arange(n_rays, dtype=np.float32) * st             # const float phi = k*st_rays
    tab = np.empty((2, n_rays), np.float32)
    tab[0] = [m.cosf(float(p)) for p in phi]                   # dy
    tab[1] = [m.sinf(float(p)) for p in phi]                   # dx
    tab.setflags(write=False)
    return tab


def direction_table_2d(n_rays):
    """float32 [2, n_rays]: row 0 dy = cosf(phi_k), row 1 dx = sinf(phi_k), phi_k = float32(k) * float32(2 pi / n_rays)
    (stardist2d.cpp:92-97), with libm's single-precision functions"""
    return _direction_table_2d(int(n_rays))


def rays_table_3d(rays):
    """float32 [3, n_rays] = (dz, dy, dx) of rays.vertices (geom3d.py:17-24)"""
    return np.ascontiguousarray(np.asarray(rays.vertices).T, dtype=np.float32)


def walk_bound(table, shape):
    """step cap of every walk of the direction table over an image of `shape`; ValueError when a ray could stall"""
    table = np.ascontiguousarray(table, np.float32)
    shape = [int(s) for s in shape]
    cap = ctypes.c_longlong(0)
    if L.load().sdb_star_dist_walk_bound(L.ptr(table), len(shape), table.shape[1], L.iarr(shape), ctypes.byref(cap)) != 0:
        raise ValueError(L.load().sdb_last_error().decode("utf-8", "replace"))
    return cap.value


def output_shape(shape, grid):
    return tuple((int(s) - 1) // int(g) + 1 for s, g in zip(shape, grid))


def _check_grid(grid, ndim):
    grid = tuple(grid)
    if len(grid) != ndim or not all(int(g) == g and int(g) >= 1 for g in grid):
        raise ValueError("grid must be %d positive integers (got %s)" % (ndim, grid))
    return tuple(int(g) for g in grid)


def _star_dist_device(lbl, table, grid, points):
    import torch
    lib = L.require_cuda()
    ndim = lbl.dim()
    if not (isinstance(lbl, torch.Tensor) and lbl.is_cuda and lbl.dtype in (torch.int32, torch.uint16) and ndim in (2, 3)):
        raise ValueError("star_dist: expected a CUDA int32 or uint16 label tensor of %s dimensions" % ("2" if ndim == 2 else "3"))
    lbl = lbl.contiguous()
    grid = _check_grid(grid, ndim)
    walk_bound(table, lbl.shape)
    R = table.shape[1]
    if points is None:
        out = torch.empty(output_shape(lbl.shape, grid) + (R,), dtype=torch.float32, device=lbl.device)
        n = 0
    else:
        if not (isinstance(points, torch.Tensor) and points.is_cuda and points.dim() == 2 and points.shape[1] == ndim):
            raise ValueError("points must be a CUDA tensor of shape (n, %d)" % ndim)
        points = points.to(torch.int32).contiguous()
        n = points.shape[0]
        out = torch.empty((n, R), dtype=torch.float32, device=lbl.device)
    if out.numel() == 0:
        return out
    tab = np.ascontiguousarray(table, np.float32)
    nb = 2 if lbl.dtype == torch.uint16 else 4
    if ndim == 2:
        L.check(lib.sdb_star_dist_2d(L.ptr(lbl), nb, lbl.shape[0], lbl.shape[1], grid[0], grid[1], R, L.ptr(tab), L.ptr(points), n,
                                     L.ptr(out), L.stream_ptr()))
    else:
        L.check(lib.sdb_star_dist_3d(L.ptr(lbl), nb, lbl.shape[0], lbl.shape[1], lbl.shape[2], grid[0], grid[1], grid[2], R, L.ptr(tab),
                                     L.ptr(points), n, L.ptr(out), L.stream_ptr()))
    return out


def star_dist_device(lbl, n_rays=32, grid=(1, 1), points=None):
    """star_dist of a CUDA int32 / uint16 label map [H, W] (labels compared by their low 16 bits, as the reference's uint16
    cast does) -> CUDA float32 [(H-1)//gy+1, (W-1)//gx+1, n_rays]; with `points` (CUDA int [n, 2], indices into that
    subsampled grid) only those pixels -> [n, n_rays].  The result is left on the tensor's stream, nothing is synchronised."""
    n_rays = int(n_rays)
    if n_rays < 1:
        raise ValueError("need 'n_rays' >= 1")
    return _star_dist_device(lbl, direction_table_2d(n_rays), grid, points)


def star_dist3D_device(lbl, rays, grid=(1, 1, 1), points=None):
    """star_dist3D of a CUDA int32 / uint16 label volume [D, H, W] along rays.vertices -> CUDA float32
    [(D-1)//gz+1, (H-1)//gy+1, (W-1)//gx+1, len(rays)]; with `points` (CUDA int [n, 3]) only those voxels -> [n, len(rays)]"""
    return _star_dist_device(lbl, rays_table_3d(rays), grid, points)


def region_stats_device(lbl, n_labels):
    """per-label statistics of a sequential CUDA int32 label map (values 0..n_labels): (count int64 [n], coordinate sums
    int64 [n, ndim], bbox min / max int32 [n, ndim], inclusive), index l - 1 for label l (sdb_region_stats)"""
    import torch
    lib = L.require_cuda()
    if not (isinstance(lbl, torch.Tensor) and lbl.is_cuda and lbl.dtype == torch.int32 and lbl.dim() in (2, 3)):
        raise ValueError("region_stats_device expects a CUDA int32 label map of 2 or 3 dimensions")
    lbl = lbl.contiguous()
    nd, n, dev = lbl.dim(), int(n_labels), lbl.device
    count = torch.empty(n, dtype=torch.int64, device=dev)
    sums = torch.empty((n, nd), dtype=torch.int64, device=dev)
    bmin = torch.empty((n, nd), dtype=torch.int32, device=dev)
    bmax = torch.empty((n, nd), dtype=torch.int32, device=dev)
    L.check(lib.sdb_region_stats(L.ptr(lbl), nd, L.iarr(lbl.shape), n, L.ptr(count), L.ptr(sums), L.ptr(bmin), L.ptr(bmax),
                                 L.stream_ptr()))
    return count, sums, bmin, bmax


def label_map_to_device(lbl):
    """host label array -> (CUDA int32 map relabelled sequentially, number of labels, CUDA int32 original labels in ascending
    order).  Negative or non-integer labels raise
    ValueError like _check_label_array, and so do labels that do not fit int32."""
    import torch
    from ..matching import _check_label_array, relabel_sequential_device
    _check_label_array(lbl, "lbl")
    L.require_cuda()
    if lbl.size and int(lbl.max()) > np.iinfo(np.int32).max:
        raise ValueError("lbl: labels above 2^31 - 1 are not supported")
    d = torch.from_numpy(np.ascontiguousarray(lbl, dtype=np.int32)).to("cuda")
    if d.numel() == 0:
        return d, 0, torch.zeros(0, dtype=torch.int32, device=d.device)
    d, fwd, n = relabel_sequential_device(d)
    return d, n, torch.nonzero(fwd > 0).flatten().to(torch.int32)


def centroids_device(lbl_seq, n_labels):
    """regionprops(...).centroid cast to int, in ascending label order: int64 sum / count in float64, truncated (CUDA int32 [n, ndim])"""
    import torch
    count, sums, _, _ = region_stats_device(lbl_seq, n_labels)
    return (sums.to(torch.float64) / count.to(torch.float64)[:, None]).to(torch.int32)


def check_points_in(points, out_shape):
    """numpy's IndexError for points outside the subsampled map (the reference indexes it with full-resolution centroids)"""
    import torch
    if points.shape[0] == 0:
        return
    hi = points.amax(dim=0).cpu().tolist()
    for a, (h, s) in enumerate(zip(hi, out_shape)):
        if h >= s:
            raise IndexError("index %d is out of bounds for axis %d with size %d" % (h, a, s))
