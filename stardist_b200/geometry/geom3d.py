"""3D geometry of the prediction path, device backed.

Mirrors stardist/geometry/geom3d.py: polyhedron_to_label (:100-198), dist_to_volume / dist_to_centroid (:220-258),
dist_to_coord3D (:261-275).
"""
import numpy as np
from ..utils import _normalize_grid, _raise
from .distances import star_dist3D_device, label_map_to_device, centroids_device, check_points_in, output_shape


RENDER_MODES = ("full", "kernel", "hull", "bbox", "debug")      # index = render_mode of the C entry point
SD3_MAX_RAYS, SD3_MAX_FACES = 256, 512                           # the 3-D kernels' limits (csrc/nms3d_pair.cuh)


def _as_rows(a, what):
    """one polyhedron may be given as a flat vector"""
    a = np.asanyarray(a)
    return a.reshape(1, -1) if a.ndim == 1 else a


def polyhedron_to_label(dist, points, rays, shape, prob=None, thr=-np.inf, labels=None, mode="full", verbose=True, overlap_label=None):
    """Label image of shape `shape` from star-convex polyhedra (API of stardist/geometry/geom3d.py:100-198).

    dist (n, n_rays) ray lengths, points (n, 3) centres, rays a Rays object; prob (n,) scores (default all one) select the
    polyhedra with prob >= thr and fix the painting order -- descending score, the first polyhedron covering a voxel wins;
    labels (n,) ids to write (default 1..n); mode one of RENDER_MODES; overlap_label: value for voxels covered more than once.
    Rendering: csrc/label3d.cu through the reference-signature entry point."""
    from ..lib.stardist3d import c_polyhedron_to_label
    n = len(points)
    if n == 0:
        verbose and print("warning: empty list of points (returning background-only image)")
        return np.zeros(shape, np.uint16)
    dist, points = _as_rows(dist, "dist"), _as_rows(points, "points")
    labels = np.arange(1, n + 1) if labels is None else np.asanyarray(labels)
    prob = np.ones(n) if prob is None else np.asanyarray(prob)
    # argument checks, with the reference's messages
    problems = (
        (np.amin(dist) <= 0, ValueError("distance array should be positive!")),
        (dist.ndim != 2, ValueError("dist should be 2 dimensional but has shape %s" % str(dist.shape))),
        (dist.ndim == 2 and dist.shape[1] != len(rays), ValueError("inconsistent number of rays!")),
        (len(prob) != n, ValueError("len(prob) != len(points)")),
        (len(labels) != n, ValueError("len(labels) != len(points)")),
        (mode not in RENDER_MODES, KeyError("Unknown render mode '%s' , allowed:  %s" % (mode, RENDER_MODES))),
    )
    for failed, err in problems:
        if failed:
            raise err
    # selection and painting order in one index vector: the survivors of the threshold, best score first
    # (the reference's argsort()[::-1] is unstable on ties; defined here as the stable sort, see DESIGN.md)
    chosen = np.flatnonzero(prob >= thr)
    if chosen.size == 0:
        verbose and print("warning: no points found with probability>= {thr:.4f} (returning background-only image)".format(thr=thr))
        return np.zeros(shape, np.uint16)
    chosen = chosen[np.argsort(prob[chosen], kind='stable')[::-1]]
    return c_polyhedron_to_label(np.ascontiguousarray(dist[chosen], np.float32), np.ascontiguousarray(points[chosen], np.float32),
                                 np.ascontiguousarray(rays.vertices, np.float32), np.ascontiguousarray(rays.faces, np.int32),
                                 np.ascontiguousarray(labels[chosen], np.int32), np.int32(RENDER_MODES.index(mode)), np.int32(verbose),
                                 np.int32(overlap_label is not None), np.int32(0 if overlap_label is None else overlap_label), shape)


def dist_to_coord3D(dist, points, rays_vertices):
    """ converts dist/points/rays_vertices to list of coords """
    dist = np.asarray(dist)
    points = np.asarray(points)
    rays_vertices = np.asarray(rays_vertices)
    if not all((len(dist) == len(points), dist.ndim == 2, points.ndim == 2,
                points.shape[-1] == 3, rays_vertices.shape[-1] == 3, dist.shape[-1] == len(rays_vertices))):
        raise ValueError(f"Wrong shapes! dist -> (m,n) points -> (m,3) rays_vertices -> (m,)")
    return points[:, np.newaxis] + dist[..., np.newaxis] * rays_vertices


def star_dist3D(lbl, rays, grid=(1, 1, 1), mode='cpp'):
    """lbl assumbed to be a label image with integer values that encode object ids. id 0 denotes background.

    Star distances float32 [(D-1)//gz+1, (H-1)//gy+1, (W-1)//gx+1, len(rays)] along rays.vertices
    (stardist/geometry/geom3d.py:17-24, 87-97), bit-identical to the reference's C++.  Modes 'cpp' and 'opencl' both run
    the CUDA kernel with the C++ semantics; there is no 'python' mode (no CPU fallback)."""
    import torch
    from .. import _lib as L
    grid = _normalize_grid(grid, 3)
    if mode == 'python':
        raise NotImplementedError("star_dist3D: mode 'python' has no CPU implementation here; use 'cpp'")
    if mode not in ('cpp', 'opencl'):
        raise ValueError("Unknown mode %s" % mode)
    L.require_cuda()
    lbl = np.asarray(lbl).astype(np.uint16, copy=False)
    if lbl.ndim != 3:
        raise ValueError("star_dist3D: label image must be 3-dimensional")
    d = torch.from_numpy(np.ascontiguousarray(lbl)).to("cuda")
    return star_dist3D_device(d, rays, grid).cpu().numpy()


def relabel_image_stardist3D(lbl, rays, verbose=False, **kwargs):
    """relabel each label region in `lbl` with its star representation (stardist/geometry/geom3d.py:201-217): the
    polyhedron of the star distances (at least 1e-3) at each region's centroid, painted by polyhedron_to_label with the
    region labels.  Centroids, distances and painting stay on the device; `kwargs` (grid) as in star_dist3D, including the
    reference's indexing of the subsampled map with full-resolution centroids (IndexError where numpy raises)."""
    import torch
    from .. import _lib as L
    from ..matching import _check_label_array
    _check_label_array(lbl, "lbl")
    if not lbl.ndim == 3:
        raise ValueError("lbl image should be 3 dimensional")
    mode = kwargs.pop('mode', 'cpp')
    grid = _normalize_grid(kwargs.pop('grid', (1, 1, 1)), 3)
    if kwargs:
        raise TypeError("unexpected keyword arguments %s" % sorted(kwargs))
    if mode == 'python':
        raise NotImplementedError("star_dist3D: mode 'python' has no CPU implementation here; use 'cpp'")
    lib = L.require_cuda()
    seq, n, labels = label_map_to_device(lbl)
    d_lbl = torch.from_numpy(np.ascontiguousarray(lbl.astype(np.uint16, copy=False))).to("cuda")
    points = centroids_device(seq, n) if n > 0 else torch.zeros((0, 3), dtype=torch.int32, device="cuda")
    check_points_in(points, output_shape(lbl.shape, grid))
    dist = star_dist3D_device(d_lbl, rays, grid, points=points)
    if n == 0:
        verbose and print("warning: empty list of points (returning background-only image)")
        return np.zeros(lbl.shape, np.uint16)
    dist = torch.clamp_min(dist, 1e-3)
    # the region labels in ascending order (regionprops), painted as polyhedron_to_label paints equal scores: last first
    flip = torch.arange(n - 1, -1, -1, device="cuda")
    dist, pts, labels = dist[flip].contiguous(), points[flip].to(torch.float32).contiguous(), labels[flip].contiguous()
    verts = torch.from_numpy(np.ascontiguousarray(rays.vertices, np.float32)).to("cuda")
    faces = torch.from_numpy(np.ascontiguousarray(rays.faces, np.int32)).to("cuda")
    nz, ny, nx = lbl.shape
    out = torch.empty((nz, ny, nx), dtype=torch.int32, device="cuda")
    if verbose:
        print("+++++++++++++++ polyhedra to label (GPU) +++++++++++++++ \nn_polys = %d n_rays = %d n_faces = %d nz,ny,nx = %d %d %d"
              % (n, len(rays), len(rays.faces), nz, ny, nx))
    L.check(lib.sdb_polyhedron_to_label(L.ptr(dist), L.ptr(pts), L.ptr(verts), L.ptr(faces), n, len(rays), len(rays.faces),
                                        L.ptr(labels), nz, ny, nx, RENDER_MODES.index("full"), 0, 0, L.ptr(out), L.stream_ptr()))
    return out.cpu().numpy()


def _dist_to_poly(dist, rays, absolute=None):
    """sdb_dist_to_volume (absolute None) / sdb_dist_to_centroid on a float32 map [nz, ny, nx, n_rays] (numpy or CUDA)"""
    import torch
    from .. import _lib as L
    verts = np.ascontiguousarray(rays.vertices, np.float32)
    faces = np.ascontiguousarray(rays.faces, np.int32)
    if len(verts) > SD3_MAX_RAYS or len(faces) > SD3_MAX_FACES:
        raise ValueError("rays with %d vertices and %d faces: at most %d rays and %d faces are supported"
                         % (len(verts), len(faces), SD3_MAX_RAYS, SD3_MAX_FACES))
    if faces.size and (faces.min() < 0 or faces.max() >= len(verts)):
        raise ValueError("rays.faces must index rays.vertices")
    if isinstance(dist, torch.Tensor):
        if not (dist.is_cuda and dist.dtype == torch.float32):
            raise ValueError("a tensor dist must be a CUDA float32 tensor")
        d_dist = dist.contiguous()
    lib = L.require_cuda()
    if not isinstance(dist, torch.Tensor):
        d_dist = torch.from_numpy(dist).cuda()
    nz, ny, nx, n_rays = (int(s) for s in d_dist.shape)
    d_verts, d_faces = torch.from_numpy(verts).cuda(), torch.from_numpy(faces).cuda()
    out = torch.empty((nz, ny, nx) + (() if absolute is None else (3,)), dtype=torch.float32, device=d_dist.device)
    if absolute is None:
        L.check(lib.sdb_dist_to_volume(L.ptr(d_dist), nz, ny, nx, n_rays, L.ptr(d_verts), L.ptr(d_faces), len(faces), L.ptr(out),
                                       L.stream_ptr()))
    else:
        L.check(lib.sdb_dist_to_centroid(L.ptr(d_dist), nz, ny, nx, n_rays, L.ptr(d_verts), L.ptr(d_faces), len(faces),
                                         int(absolute), L.ptr(out), L.stream_ptr()))
    return out if isinstance(dist, torch.Tensor) else out.cpu().numpy()


def dist_to_volume(dist, rays):
    """ returns areas of polyhedra
        dist.shape = (nz,ny,nx,nrays)

    The volume of the star-convex polyhedron of every voxel (stardist/geometry/geom3d.py:220-236 over c_dist_to_volume),
    float32 (nz, ny, nx), bit-identical to the reference; one device thread per voxel (helpers.cu).  dist may be a CUDA
    float32 tensor, which gives a CUDA tensor.  At most 256 rays / 512 faces (ValueError)."""
    import torch
    if not isinstance(dist, torch.Tensor):
        dist = np.asanyarray(dist)
    dist.ndim == 4 or _raise(ValueError("dist.ndim = {dist.ndim} but should be 4".format(dist = dist)))
    dist.shape[-1]== len(rays) or _raise(ValueError("dist.shape[-1] = {d} but should be {l}".format(d = dist.shape[-1], l = len(rays))))
    if not isinstance(dist, torch.Tensor):
        dist = np.ascontiguousarray(dist.astype(np.float32, copy=False))
    return _dist_to_poly(dist, rays)


def dist_to_centroid(dist, rays, mode='absolute'):
    """ returns centroids of polyhedra

        dist.shape = (nz,ny,nx,nrays)
        mode = 'absolute' or 'relative'

    float32 (nz, ny, nx, 3) (stardist/geometry/geom3d.py:239-258 over c_dist_to_centroid), bit-identical to the reference;
    with mode 'absolute' the voxel's (z, y, x) is added.  dist may be a CUDA float32 tensor, which gives a CUDA tensor."""
    import torch
    dist.ndim == 4 or _raise(ValueError("dist.ndim = {dist.ndim} but should be 4".format(dist = dist)))
    dist.shape[-1]== len(rays) or _raise(ValueError("dist.shape[-1] = {d} but should be {l}".format(d = dist.shape[-1], l = len(rays))))
    if not isinstance(dist, torch.Tensor):
        dist = np.ascontiguousarray(dist.astype(np.float32, copy=False))

    mode in ('absolute', 'relative') or _raise(ValueError("mode should be either 'absolute' or 'relative'"))
    return _dist_to_poly(dist, rays, absolute=(mode == 'absolute'))
