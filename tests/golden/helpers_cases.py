"""Inputs of the helpers fixture (make_helpers.py -> helpers.npz): mask_to_categorical, sample_points, sample_patches /
get_valid_inds and dist_to_volume / dist_to_centroid on small seeded inputs.

* mask_to_categorical: 2-D and 3-D label maps in uint16 / int32 / int64 with non-sequential ids up to 2^31 - 1, dict classes
  (with class 0, None objects and keys that do not occur), integer and None classes, n_classes 1 and 5.
* sample_points: bool and integer masks (values 0..3, so `& 1` matters), b in {None, 0, 2, 7}, with and without prob.
* sample_patches / get_valid_inds: even and odd patch sizes (a clipped crop, and crops of different shapes that np.stack
  refuses), with and without valid_inds and a filter, several dtypes (one of 3-byte elements), n_valid < n_samples.
* dist_to_volume / dist_to_centroid: random positive maps for Rays_GoldenSpiral(96), Rays_Octo and Rays_Cartesian (whose
  pole faces are degenerate), with some zero rays."""
import numpy as np

INT32_MAX = 2 ** 31 - 1


def _blobs(rng, shape, n):
    """label image with n random ellipsoids painted in order, ids 1..n"""
    y = np.zeros(shape, np.int32)
    grids = np.meshgrid(*[np.arange(s) for s in shape], indexing='ij')
    for k in range(1, n + 1):
        c = [rng.uniform(0, s) for s in shape]
        r = [rng.uniform(1.5, max(2.0, s / 5)) for s in shape]
        y[sum(((g - ci) / ri) ** 2 for g, ci, ri in zip(grids, c, r)) <= 1] = k
    return y


def _renumber(y, ids):
    lut = np.zeros(int(y.max()) + 1, np.int64)
    lut[1:] = ids[:int(y.max())]
    return lut[y]


def categorical_cases():
    """name -> (y, n_classes, classes)"""
    rng = np.random.default_rng(11)
    out = {}
    y = _blobs(rng, (48, 56), 14)
    ids = rng.choice(np.arange(1, 60000), 14, replace=False)
    y16 = _renumber(y, ids).astype(np.uint16)
    labels = sorted(set(np.unique(y16[y16 > 0]).tolist()))
    cls = {l: [None, 0, 1, 2, 3, 4, 5][i % 7] for i, l in enumerate(labels)}
    cls.update({60001: 3, 60002: None, 60003: 0})                     # keys that do not occur
    out['2d_u16_dict_n5'] = (y16, 5, cls)
    y3 = _blobs(rng, (10, 20, 24), 9)
    out['3d_i32_int_n3'] = (y3.astype(np.int32), 3, 2)
    out['3d_i32_none_n3'] = (y3.astype(np.int32), 3, None)
    big = np.array([1, 7, 2 ** 20, 2 ** 30 + 5, INT32_MAX - 1, INT32_MAX, 99, 12345, 4, 2 ** 31 - 100], np.int64)
    y64 = _renumber(_blobs(rng, (40, 40), 10), big)
    out['2d_i64_big_dict_n1'] = (y64, 1, {int(l): [1, None, 0][i % 3] for i, l in enumerate(big)})
    out['2d_i64_big_int_n1'] = (y64, 1, 1)
    out['2d_i32_int0_n5'] = (y.astype(np.int32), 5, 0)
    out['2d_empty_n5'] = (np.zeros((7, 9), np.int32), 5, 1)
    return out


def sample_points_cases():
    """name -> (n_samples, mask, prob, b, seed)"""
    rng = np.random.default_rng(12)
    prob = rng.uniform(0, 1, (60, 72)).astype(np.float32)
    m_int = rng.integers(0, 4, (60, 72)).astype(np.uint8)
    return {
        'bool_b2_prob': (200, prob > 0.4, prob, 2, 1),
        'bool_b7_noprob': (50, prob > 0.7, None, 7, 2),
        'uint8_bnone_prob': (120, m_int, prob, None, 3),
        'int32_b0_noprob': (80, m_int.astype(np.int32), None, 0, 4),
        'int64_b2_prob': (33, (m_int.astype(np.int64) - 1) * 3, prob, 2, 5),
    }


def fg_filter(img, patch_size):
    """a patch filter: the voxels above the 0.8 quantile"""
    return img > np.quantile(img, 0.8)


def sparse_filter(img, patch_size):
    """a patch filter that keeps three positions (n_valid < n_samples)"""
    m = np.zeros(img.shape, bool)
    m[tuple(np.array(img.shape) // 2)] = True
    m[tuple(np.array(img.shape) // 2 - 1)] = True
    m[tuple(np.array(img.shape) // 2 + 1)] = True
    return m


FILTERS = dict(fg=fg_filter, sparse=sparse_filter)


def sample_patches_cases():
    """name -> (datas, patch_size, n_samples, valid_inds: None, 'plain' or a FILTERS key, seed)"""
    rng = np.random.default_rng(13)
    x2 = rng.uniform(0, 1, (40, 50)).astype(np.float32)
    y2 = rng.integers(0, 60000, (40, 50)).astype(np.uint16)
    s3 = np.array([b'%03d' % (i % 1000) for i in range(40 * 50)], 'S3').reshape(40, 50)
    x3 = rng.uniform(0, 1, (12, 20, 24)).astype(np.float64)
    y3 = rng.integers(-5, 2 ** 40, (12, 20, 24)).astype(np.int64)
    c3 = (x3 + 1j * x3[::-1]).astype(np.complex128)
    b3 = x3 > 0.5
    small = rng.uniform(0, 1, (5, 7)).astype(np.float32)
    odd = rng.uniform(0, 1, (9, 11)).astype(np.float32)
    return {
        '2d_even_plain_meshgrid': ([x2, y2, s3], (8, 10), 6, None, 1),
        '2d_even_valid_plain': ([x2, y2], (8, 10), 5, 'plain', 2),
        '2d_odd_valid_fg': ([x2, y2, s3], (7, 9), 7, 'fg', 3),
        '2d_odd_clipped_one': ([small], (5, 5), 1, None, 4),
        '2d_odd_clipped_mismatch': ([odd], (5, 7), 20, None, 5),
        '3d_even_meshgrid': ([x3, y3, c3, b3], (4, 8, 6), 4, None, 6),
        '3d_odd_valid_fg': ([x3, y3, b3], (3, 5, 7), 9, 'fg', 7),
        '3d_sparse_replace': ([x3, y3], (4, 6, 6), 8, 'sparse', 8),
    }


def dist_cases():
    """name -> (dist float32 [nz, ny, nx, n_rays], rays)"""
    import os, sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
    from stardist_b200.rays3d import Rays_GoldenSpiral, Rays_Octo, Rays_Cartesian
    rng = np.random.default_rng(14)
    out = {}
    for name, rays, shape in (('golden96', Rays_GoldenSpiral(96), (6, 7, 8)), ('octo', Rays_Octo(n_level=3), (5, 6, 7)),
                              ('cartesian', Rays_Cartesian(n_rays_x=10, n_rays_z=6), (4, 5, 6)), ('golden96_aniso', Rays_GoldenSpiral(96, anisotropy=(2, 1, 1)), (3, 4, 5))):
        d = rng.uniform(0.5, 30, shape + (len(rays),)).astype(np.float32)
        d[rng.uniform(size=d.shape) < 0.05] = 0
        d[0, 0, 0] = 0                                                         # a voxel with every ray zero
        out[name] = (d, rays)
    return out
