"""Star distances without a GPU: the float32 restatement of the kernels' per-ray arithmetic (tests/star_dist_emu.py), driven
by the product's host direction table, equals the reference's C++ (oracle/_ref) bit for bit; the golden fixture is
reproducible; the product refuses to run without CUDA."""
import os, sys, json
import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
import star_dist_emu as E
import star_dist_cases as C
from oracle import ref_ext
from stardist_b200.geometry.distances import direction_table_2d, rays_table_3d, walk_bound

needs_ref = pytest.mark.skipif(not ref_ext.available(), reason="oracle/_ref not built")


def _ref2(m, R, grid=(1, 1)):
    return ref_ext.stardist2d().c_star_dist(np.asarray(m).astype(np.uint16), np.int32(R), np.int32(grid[0]), np.int32(grid[1]))


def _ref3(m, rays_tab, grid=(1, 1, 1)):
    return ref_ext.stardist3d().c_star_dist3d(np.asarray(m).astype(np.uint16), *[np.ascontiguousarray(t) for t in rays_tab],
                                               rays_tab.shape[1], *grid)


@needs_ref
@pytest.mark.parametrize("n_rays", list(range(3, 65)) + [96, 128, 255, 256])
def test_emulated_2d_equals_reference(n_rays):
    m = C.ellipses_2d((24, 26), 4, seed=2)
    tab = direction_table_2d(n_rays)
    for grid in ((1, 1), (2, 3)):
        want = _ref2(m, n_rays, grid)
        got = E.star_dist_2d(m, tab, grid)
        assert got.dtype == want.dtype and got.shape == want.shape
        assert np.array_equal(got, want), (grid, int((got != want).sum()))


@needs_ref
@pytest.mark.parametrize("rname", list(C.ray_sets()))
def test_emulated_3d_equals_reference(rname):
    m = C.ellipsoids_3d((10, 14, 16), 4, seed=1)
    tab = rays_table_3d(C.ray_sets()[rname])
    for grid in C.GRIDS_3D:
        want = _ref3(m, tab, grid)
        got = E.star_dist_3d(m, tab, grid)
        assert got.shape == want.shape and np.array_equal(got, want), (grid, int((got != want).sum()))


@needs_ref
@pytest.mark.parametrize("name", ["border", "singles", "constant", "big_labels", "int8_negative"])
def test_emulated_edge_maps_equal_reference(name):
    m = C.maps_2d()[name]
    assert np.array_equal(E.star_dist_2d(m, direction_table_2d(32)), _ref2(m, 32))
    m3 = C.maps_3d()[name]
    tab = rays_table_3d(C.ray_sets()["gs32"])
    assert np.array_equal(E.star_dist_3d(m3, tab), _ref3(m3, tab))


def test_direction_table_is_float32_libm():
    tab = direction_table_2d(32)
    assert tab.dtype == np.float32 and tab.shape == (2, 32)
    assert tab[0, 0] == 1 and tab[1, 0] == 0
    # close to the float64 angles, but built from libm's single-precision functions
    phi = np.arange(32, dtype=np.float32) * np.float32(2 * np.pi / 32)
    assert np.allclose(tab[0], np.cos(phi.astype(np.float64)), atol=1e-6)
    assert np.allclose(tab[1], np.sin(phi.astype(np.float64)), atol=1e-6)


def test_walk_bound_rejects_stalling_rays():
    with pytest.raises(ValueError):
        walk_bound(np.zeros((3, 4), np.float32), (5, 6, 7))                       # zero ray
    short = np.array([[1e-3], [0], [0]], np.float32)
    with pytest.raises(ValueError):
        walk_bound(short, (5, 6, 7))                                                 # below 2^-8
    tiny = np.array([[2 ** -7], [0], [0]], np.float32)
    assert walk_bound(tiny, (5, 6, 7)) > 0
    with pytest.raises(ValueError):
        walk_bound(tiny, (5, 6, 1 << 20))                                            # x + d == x before the walk leaves
    cap = walk_bound(direction_table_2d(32), (24, 24))
    assert 25 <= cap < 100


def test_centroid_stand_in_equals_definition():
    import make_star_dist as M
    for m in (C.ellipses_2d(), C.border_3d(), C.singles_2d()):
        regs = M.regionprops(m)
        labels = np.unique(m[m > 0])
        assert [r.label for r in regs] == list(labels)
        for r in regs:
            want = np.argwhere(m == r.label).mean(axis=0)
            assert np.array_equal(np.array(r.centroid), want)
            assert r.bbox == tuple(np.argwhere(m == r.label).min(0)) + tuple(np.argwhere(m == r.label).max(0) + 1)


@needs_ref
def test_golden_generator_is_deterministic():
    """the case maps are reproducible and a re-run of the reference on a few of them gives the stored hashes"""
    import make_star_dist as M
    for a, b in zip(C.maps_2d().values(), C.maps_2d().values()):
        assert np.array_equal(a, b)
    g = np.load(os.path.join(HERE, "golden", "star_dist.npz"))
    hashes = json.loads(g["hashes"].tobytes().decode())
    g2, g3, _ = M.reference_modules()
    entries = M.dense_entries(g2, g3)
    assert set(entries) == set(hashes)
    for key in ("s2/ellipses/7/2,4", "s2/border/32/3,1", "s3/ellipsoids/gs32/1,2,4", "s3/big_labels/cartesian/1,1,1"):
        d = entries[key]()
        assert [C.sha(d), list(d.shape)] == hashes[key], key


def test_product_raises_without_cuda():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is visible")
    import stardist_b200 as sd
    from stardist_b200.lib.stardist2d import c_star_dist
    from stardist_b200.lib.stardist3d import c_star_dist3d
    m = C.ellipses_2d((16, 16), 2)
    rays = C.ray_sets()["gs32"]
    tab = rays_table_3d(rays)
    for call in (lambda: sd.star_dist(m, 32), lambda: sd.star_dist3D(m[None], rays), lambda: sd.relabel_image_stardist(m, 32),
                 lambda: sd.relabel_image_stardist3D(m[None], rays), lambda: sd.calculate_extents(m),
                 lambda: c_star_dist(m.astype(np.uint16), 32, 1, 1), lambda: c_star_dist3d(m[None].astype(np.uint16), *tab, 32, 1, 1, 1)):
        with pytest.raises(sd._lib.StarDistB200Error):
            call()


def test_argument_errors_without_gpu():
    import stardist_b200 as sd
    m = C.ellipses_2d((16, 16), 2)
    with pytest.raises(ValueError):
        sd.star_dist(m, 2)
    with pytest.raises(NotImplementedError):
        sd.star_dist(m, 32, mode='python')
    with pytest.raises(ValueError):
        sd.star_dist(m, 32, mode='nope')
    with pytest.raises(ValueError):
        sd.relabel_image_stardist(-m, 32)
    with pytest.raises(ValueError):
        sd.star_dist3D(m[None], C.ray_sets()["gs32"], grid=(3, 1, 1))
