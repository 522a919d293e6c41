"""Star distances, region statistics, relabel_image_stardist(3D) and calculate_extents on the device, against the reference's
C++ at run time (oracle/_ref) and the golden fixture (tests/golden/star_dist.npz, make_star_dist.py)."""
import os, sys, json
import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
import star_dist_cases as C
from oracle import ref_ext

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sd():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import stardist_b200
    return stardist_b200


@pytest.fixture(scope="module")
def golden():
    g = np.load(os.path.join(HERE, "golden", "star_dist.npz"))
    return g, json.loads(g["hashes"].tobytes().decode())


def _ref2(m, R, grid=(1, 1)):
    return ref_ext.stardist2d().c_star_dist(np.asarray(m).astype(np.uint16), np.int32(R), np.int32(grid[0]), np.int32(grid[1]))


def _ref3(m, rays, grid=(1, 1, 1)):
    tab = np.asarray(rays.vertices).T.astype(np.float32)
    return ref_ext.stardist3d().c_star_dist3d(np.asarray(m).astype(np.uint16), *[np.ascontiguousarray(t) for t in tab], len(rays), *grid)


def _same(got, want):
    assert got.dtype == np.float32 and got.shape == want.shape, (got.dtype, got.shape, want.shape)
    assert np.array_equal(got, want), int((got != want).sum())


def test_golden_dense_cases(sd, golden):
    from stardist_b200.lib.stardist2d import c_star_dist
    from stardist_b200.lib.stardist3d import c_star_dist3d
    _, hashes = golden
    rays = C.ray_sets()
    m2, m3 = C.maps_2d(), C.maps_3d()
    for key, (h, shape) in hashes.items():
        parts = key.split("/")
        grid = tuple(int(g) for g in parts[-1].split(","))
        if parts[0] == "s2":
            m, R = m2[parts[1]], int(parts[2])
            for mode in ("cpp", "opencl"):
                got = sd.star_dist(m, R, grid=grid, mode=mode)
                assert got.dtype == np.float32 and list(got.shape) == shape and C.sha(got) == h, (key, mode)
            got = c_star_dist(m.astype(np.uint16), R, *grid)
        else:
            m, r = m3[parts[1]], rays[parts[2]]
            for mode in ("cpp", "opencl"):
                got = sd.star_dist3D(m, r, grid=grid, mode=mode)
                assert got.dtype == np.float32 and list(got.shape) == shape and C.sha(got) == h, (key, mode)
            tab = np.asarray(r.vertices).T.astype(np.float32)
            got = c_star_dist3d(m.astype(np.uint16), *[np.ascontiguousarray(t) for t in tab], len(r), *grid)
        assert list(got.shape) == shape and C.sha(got) == h, key
        if ref_ext.available():
            want = _ref2(m, R, grid) if parts[0] == "s2" else _ref3(m, r, grid)
            _same(got, want)


@pytest.mark.skipif(not ref_ext.available(), reason="oracle/_ref not built")
def test_demo_mask_every_n_rays(sd):
    m = C.demo_mask()[:256, :256]
    for R in range(3, 257):
        _same(sd.star_dist(m, R), _ref2(m, R))


@pytest.mark.skipif(not ref_ext.available(), reason="oracle/_ref not built")
@pytest.mark.parametrize("dtype", [np.int8, np.int16, np.int32, np.int64, np.uint8, np.uint16, np.uint32])
def test_input_dtypes(sd, dtype):
    """the reference's test_types"""
    m = C.ellipses_2d((48, 52), 6, seed=5) % 120
    m3 = C.ellipsoids_3d((12, 20, 22), 4, seed=5) % 120
    rays = C.ray_sets()["gs32"]
    _same(sd.star_dist(m.astype(dtype), 32), _ref2(m.astype(dtype), 32))
    _same(sd.star_dist3D(m3.astype(dtype), rays), _ref3(m3.astype(dtype), rays))


@pytest.mark.skipif(not ref_ext.available(), reason="oracle/_ref not built")
def test_at_size(sd):
    import bench_data
    lbl = bench_data.ellipse_labels((1024, 1024), seed=0)          # the benchmark's 2-D ground truth
    _same(sd.star_dist(lbl, 32), _ref2(lbl, 32))
    vol = bench_data.ellipsoid_labels((64, 256, 256), seed=0)
    rays = C.ray_sets()["gs96"]
    _same(sd.star_dist3D(vol, rays), _ref3(vol, rays))


def test_device_and_point_paths(sd):
    import torch
    from stardist_b200.geometry.distances import star_dist_device, star_dist3D_device
    m = C.ellipses_2d((50, 61), 7, seed=4)
    for grid in C.GRIDS_2D:
        host = sd.star_dist(m, 32, grid=grid)
        for dt in (torch.int32, torch.uint16):
            d = torch.from_numpy(m.astype(np.int32 if dt == torch.int32 else np.uint16)).cuda()
            dev = star_dist_device(d, 32, grid)
            assert dev.is_cuda and dev.dtype == torch.float32
            _same(dev.cpu().numpy(), host)
            pts = np.stack(np.nonzero(np.ones(host.shape[:2], bool)), 1)[::3]
            got = star_dist_device(d, 32, grid, points=torch.from_numpy(pts).cuda()).cpu().numpy()
            _same(got, host[tuple(pts.T)])
    m3 = C.ellipsoids_3d((12, 18, 20), 4, seed=6)
    rays = C.ray_sets()["gs96"]
    for grid in C.GRIDS_3D:
        host = sd.star_dist3D(m3, rays, grid=grid)
        d = torch.from_numpy(m3).cuda()
        _same(star_dist3D_device(d, rays, grid).cpu().numpy(), host)
        pts = np.stack(np.nonzero(np.ones(host.shape[:3], bool)), 1)[::5]
        _same(star_dist3D_device(d, rays, grid, points=torch.from_numpy(pts).cuda()).cpu().numpy(), host[tuple(pts.T)])


def _stats_np(m):
    m = np.asarray(m)
    n = int(m.max()) if m.size else 0
    idx = np.argwhere(m > 0)
    lab = m[m > 0] - 1
    count = np.bincount(lab, minlength=n)
    sums = np.stack([np.bincount(lab, idx[:, a], minlength=n) for a in range(m.ndim)], 1).astype(np.int64)
    bmin = np.stack([np.array([idx[lab == l, a].min() for l in range(n)]) for a in range(m.ndim)], 1) if n else np.zeros((0, m.ndim))
    bmax = np.stack([np.array([idx[lab == l, a].max() for l in range(n)]) for a in range(m.ndim)], 1) if n else np.zeros((0, m.ndim))
    return count, sums, bmin, bmax


def test_region_stats(sd):
    import torch
    from stardist_b200.geometry.distances import region_stats_device
    from stardist_b200.matching import relabel_sequential
    rng = np.random.default_rng(0)
    maps = [rng.integers(0, 30, (37, 45)), C.ellipses_2d(), C.ellipsoids_3d(), C.big_labels(C.ellipsoids_3d()),
            rng.integers(0, 7, (9, 70, 33)), np.zeros((5, 6), np.int64), C.singles_3d()]
    sparse = np.zeros((300, 301), np.int64)
    sparse[rng.integers(0, 300, 50), rng.integers(0, 301, 50)] = rng.integers(1, 1 << 30, 50)
    maps.append(sparse)
    for m in maps:
        seq = relabel_sequential(np.asarray(m))[0].astype(np.int32)
        n = int(seq.max())
        got = region_stats_device(torch.from_numpy(seq).cuda(), n)
        for g, w in zip(got, _stats_np(seq)):
            assert np.array_equal(g.cpu().numpy(), w)
    with pytest.raises(sd._lib.StarDistB200Error):
        region_stats_device(torch.full((4, 4), 3, dtype=torch.int32, device="cuda"), 2)


def test_relabel_2d_equals_polygons_to_label_on_frozen_input(sd, golden):
    from make_star_dist import RELABEL_2D
    g, _ = golden
    m2 = C.maps_2d()
    for i, (name, R, grid) in enumerate(RELABEL_2D):
        if "relabel2d/%d/raises" % i in g.files:
            with pytest.raises(IndexError):
                sd.relabel_image_stardist(m2[name], R, grid=grid)
            continue
        dist, points = g["relabel2d/%d/dist" % i], g["relabel2d/%d/points" % i]
        got = sd.relabel_image_stardist(m2[name], R, grid=grid)
        want = sd.polygons_to_label(dist, points, shape=m2[name].shape)
        assert got.dtype == want.dtype and np.array_equal(got, want), (name, R)


def test_relabel_3d_golden(sd, golden):
    import hullcheck
    from make_star_dist import RELABEL_3D
    g, _ = golden
    rays_all, m3 = C.ray_sets(), C.maps_3d()
    for i, (name, rname) in enumerate(RELABEL_3D):
        lbl, rays = m3[name], rays_all[rname]
        got = sd.relabel_image_stardist3D(lbl, rays)
        want = g["relabel3d/%d" % i]
        assert got.shape == want.shape
        diff = np.argwhere(got != want)
        if len(diff) == 0:
            continue
        # the polyhedra as the reference builds them, to classify the differing voxels
        labs = np.unique(lbl[lbl > 0])
        pts = np.array([np.argwhere(lbl == l).mean(0).astype(int) for l in labs])
        dist = np.maximum(sd.star_dist3D(lbl, rays)[tuple(pts.T)], 1e-3)
        cover = np.zeros(lbl.shape, np.int32)
        for k in range(len(labs)):
            cover += sd.polyhedron_to_label(dist[k:k + 1], pts[k:k + 1], rays, lbl.shape, verbose=False) > 0
        overlap = cover[tuple(diff.T)] >= 2
        rest = diff[~overlap]
        # reference order among equal scores is unspecified: only voxels covered twice or more may take another label;
        # the others must lie exactly on a hull facet (tests/hullcheck.py)
        if len(rest):
            mask = np.zeros(lbl.shape, bool); mask[tuple(rest.T)] = True
            hullcheck.assert_only_exact_hull_boundary_voxels_differ(np.where(mask, got, want), want, dist, pts.astype(np.float32), rays.vertices)


def _circle_image(shape, radius, eps):
    """the reference's tests/utils.py circle_image, centred"""
    xs = tuple(np.arange(s) - s // 2 for s in shape)
    Xs = np.meshgrid(*xs, indexing="ij")
    R = np.sqrt(np.sum([X ** 2 / e ** 2 for X, e in zip(Xs, eps)], axis=0))
    return (R < radius).astype(np.uint16)


def _rel_error(lbl1, lbl2):
    return 1 - np.count_nonzero(np.bitwise_and(lbl1 > 0, lbl2 > 0)) / np.count_nonzero(lbl1 > 0)


@pytest.mark.parametrize("n_rays", [32, 64])
@pytest.mark.parametrize("eps", [(1, 1), (.4, 1.3)])
def test_relabel_consistency_2d(sd, n_rays, eps):
    """the reference's tests/test_stardist2D.py test_relabel_consistency: an already star-convex image relabels to itself"""
    lbl1 = _circle_image((32, 32), 8, eps)
    lbl2 = sd.relabel_image_stardist(lbl1, n_rays)
    assert _rel_error(lbl1, lbl2) < 1e-1


@pytest.mark.parametrize("n_rays", [64, 128])
@pytest.mark.parametrize("eps", [(1, 1, 1), (.4, 1.3, .7)])
def test_relabel_consistency_3d(sd, n_rays, eps):
    """the reference's tests/test_stardist3D.py test_relabel_consistency"""
    rays = sd.Rays_GoldenSpiral(n_rays, anisotropy=1. / np.array(eps))
    lbl1 = sd.relabel_image_stardist3D(_circle_image((32, 32, 32), 8, eps), rays)
    lbl2 = sd.relabel_image_stardist3D(lbl1, rays)
    assert _rel_error(lbl1, lbl2) < 1e-1


def test_calculate_extents_golden(sd, golden):
    g, _ = golden
    e2, e3 = C.maps_2d(), C.maps_3d()
    ext = {"ellipses": e2["ellipses"], "demo": e2["demo"], "border": e2["border"], "empty": e2["empty"],
           "ellipsoids": e3["ellipsoids"], "border3d": e3["border"], "big_labels3d": e3["big_labels"]}
    for k, m in ext.items():
        for fname, f in (("median", np.median), ("max", np.max)):
            got, want = np.asarray(sd.calculate_extents(m, f)), g["extents/%s/%s" % (k, fname)]
            assert got.dtype == want.dtype and np.array_equal(got, want), (k, fname, got, want)
    got = sd.calculate_extents([e2["ellipses"], e2["border"], e2["singles"]])
    assert np.array_equal(got, g["extents/list/median"])
    got = sd.calculate_extents(np.stack([e3["ellipsoids"], e3["big_labels"]]))
    assert np.array_equal(got, g["extents/stack/median"])


def test_argument_errors_launch_nothing(sd):
    import torch
    from stardist_b200 import _lib as L
    from stardist_b200.lib.stardist3d import c_star_dist3d
    from stardist_b200.geometry.distances import star_dist3D_device
    m = C.ellipses_2d((20, 20), 3)
    L.launch_count(reset=True)
    with pytest.raises(ValueError):
        sd.star_dist(m, 2)
    with pytest.raises(ValueError):
        sd.relabel_image_stardist(m, 2)

    class Bad:
        vertices = np.array([[1, 0, 0], [0, 0, 0], [0, 1, 0], [0, 0, 1]], np.float64)
        faces = np.array([[0, 2, 3]])
        def __len__(self): return 4
    with pytest.raises(ValueError):
        sd.star_dist3D(m[None], Bad())
    Bad.vertices = Bad.vertices + np.array([0, 0, 1e-3])
    with pytest.raises(ValueError):
        star_dist3D_device(torch.from_numpy(m[None]).cuda(), Bad())
    tab = np.zeros((3, 4), np.float32)
    with pytest.raises(ValueError):
        c_star_dist3d(m[None].astype(np.uint16), *tab, 4, 1, 1, 1)
    with pytest.raises(ValueError):
        sd.relabel_image_stardist(-m, 32)
    with pytest.raises(ValueError):
        sd.relabel_image_stardist3D(-m[None], sd.Rays_GoldenSpiral(32))
    with pytest.raises(ValueError):
        sd.relabel_image_stardist(m.astype(np.int64) + (1 << 31), 32)
    with pytest.raises(ValueError):
        sd.calculate_extents(m.astype(np.int64) + (1 << 31))
    assert L.launch_count() == 0
