"""mask_to_categorical, sample_points, sample_patches / get_valid_inds and dist_to_volume / dist_to_centroid without a device:
every argument error is raised with the reference's type and message before the device is touched; the host halves of
sample_points and sample_patches (the draw, the crop starts and shapes) give the reference's results and np.random state
(tests/golden/helpers.npz) with the device step replaced by numpy; a float32 / float64 numpy restatement of the polyhedron
volume and centroid equals the reference extension on the fixture; and the new entry points are declared in the header and
the ctypes table."""
import json, os, re, sys
import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
sys.path.insert(0, ROOT)
import helpers_cases as C

ENTRY_POINTS = ("sdb_label_class_map", "sdb_mask_compact_count", "sdb_mask_compact_write", "sdb_gather_patches",
                "sdb_dist_to_volume", "sdb_dist_to_centroid")


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(HERE, "golden", "helpers.npz"))


@pytest.fixture
def no_device(monkeypatch):
    from stardist_b200 import _lib
    monkeypatch.setattr(_lib, 'require_cuda', lambda: pytest.fail("device touched"))


def _state_equals(golden, key):
    _, k, pos, has_gauss, cached = np.random.get_state()
    return (np.array_equal(k, golden[key + "/key"]) and pos == golden[key + "/pos"]
            and np.array_equal([has_gauss, cached], golden[key + "/gauss"]))


def test_entry_points_declared():
    header = open(os.path.join(ROOT, "include", "stardist_b200.h")).read()
    table = open(os.path.join(ROOT, "stardist_b200", "_lib.py")).read()
    for name in ENTRY_POINTS:
        assert re.search(r"\bint %s\(" % name, header), name
        assert "lib.%s.argtypes" % name in table, name


def test_top_level_exports():
    import stardist_b200 as S
    from stardist_b200.io.rois import export_imagej_rois
    from stardist_b200.sample_patches import get_valid_inds, sample_patches
    assert S.sample_patches is sample_patches and S.export_imagej_rois is export_imagej_rois
    assert S.sample_points.__module__ == "stardist_b200.utils" and callable(get_valid_inds)


# ------------------------------------------------------------------------------------------------ argument errors
def test_mask_to_categorical_errors(no_device):
    from stardist_b200.utils import mask_to_categorical as m2c
    y = np.array([[0, 1], [2, 2]], np.int32)
    cases = [
        (lambda: m2c(y.astype(np.float32), 2, 1), "y must be an array of non-negative integers."),
        (lambda: m2c(-y, 2, 1), "y must be an array of non-negative integers."),
        (lambda: m2c(list(y), 2, 1), "y must be an array of non-negative integers."),
        (lambda: m2c(y, True, 1), "n_classes is 'True' but should be a positive integer"),
        (lambda: m2c(y, 0, 1), "n_classes is '0' but should be a positive integer"),
        (lambda: m2c(y, 2.0, 1), "n_classes is '2.0' but should be a positive integer"),
        (lambda: m2c(y, 2, 'a'), "classes should be dict, single scalar, or None!"),
        (lambda: m2c(y, 2, True), "classes should be dict, single scalar, or None!"),
        (lambda: m2c(y, 2, 1.0), "classes should be dict, single scalar, or None!"),
        (lambda: m2c(y, 2, {1: 1, 2: 3}), "Wrong class id '3' (for n_classes=2)"),
        (lambda: m2c(y, 2, {1: 1, 2: 2, 9: -1}), "Wrong class id '-1' (for n_classes=2)"),       # a key that does not occur
        (lambda: m2c(y, 2, {1: True, 2: 2}), "Wrong class id 'True' (for n_classes=2)"),
        (lambda: m2c(y, 2, {1: 1.0, 2: 2}), "Wrong class id '1.0' (for n_classes=2)"),
        (lambda: m2c(y.astype(np.int64) * 2 ** 31, 2, 1), "mask_to_categorical: labels must be below 2^31"),
    ]
    for call, msg in cases:
        with pytest.raises(ValueError) as e:
            call()
        assert str(e.value) == msg


def test_sample_points_errors(no_device):
    from stardist_b200.utils import sample_points
    m = np.ones((8, 9), np.float32)
    for b in (None, 0, 2):
        with pytest.raises(TypeError) as e:
            sample_points(5, m, b=b)
        want = None
        try:
            m & (np.zeros_like(m) if (b is not None and b > 0) else True)
        except TypeError as err:
            want = str(err)
        assert str(e.value) == want
    with pytest.raises(ValueError, match="2-dimensional"):
        sample_points(5, np.ones((3, 8, 9), bool))
    import torch
    with pytest.raises(TypeError):
        sample_points(5, torch.ones((8, 9), dtype=torch.bool))                   # not on the device


def test_sample_patches_errors(no_device):
    from stardist_b200.sample_patches import sample_patches, get_valid_inds
    a = np.zeros((10, 12), np.float32)
    with pytest.raises(ValueError) as e:
        sample_patches([a], (4,), 2)
    assert str(e.value) == ""
    with pytest.raises(ValueError) as e:
        sample_patches([a, np.zeros((10, 11))], (4, 4), 2)
    assert str(e.value) == "all input shapes must be the same: (10, 12) / (10, 11)"
    with pytest.raises(ValueError) as e:
        sample_patches([a], (4, 13), 2)
    assert str(e.value) == "patch_size (4, 13) negative or larger than data shape (10, 12) along some dimensions"
    with pytest.raises(ValueError) as e:
        sample_patches([a], (4, 4), 2, valid_inds=(np.zeros(0, np.uint32), np.zeros(0, np.uint32)))
    assert str(e.value) == "no regions to sample from!"
    with pytest.raises(ValueError) as e:
        sample_patches([a], (4, 4), 0)
    assert str(e.value) == "need at least one array to stack"
    with pytest.raises(ValueError) as e:
        get_valid_inds(a, (4, 4, 1))
    assert str(e.value) == ""
    with pytest.raises(ValueError) as e:
        get_valid_inds(a, (0, 4))
    assert str(e.value) == "patch_size (0, 4) negative or larger than image shape (10, 12) along some dimensions"


def test_dist_to_poly_errors(no_device):
    from stardist_b200.geometry.geom3d import dist_to_volume, dist_to_centroid
    from stardist_b200.rays3d import Rays_GoldenSpiral
    rays = Rays_GoldenSpiral(16)
    d = np.ones((2, 3, 4, 16), np.float32)
    for f in (dist_to_volume, dist_to_centroid):
        with pytest.raises(ValueError) as e:
            f(d[0], rays)
        assert str(e.value) == "dist.ndim = 3 but should be 4"
        with pytest.raises(ValueError) as e:
            f(d[..., :15], rays)
        assert str(e.value) == "dist.shape[-1] = 15 but should be 16"
    with pytest.raises(ValueError) as e:
        dist_to_centroid(d, rays, mode='abs')
    assert str(e.value) == "mode should be either 'absolute' or 'relative'"
    with pytest.raises(AttributeError):
        dist_to_centroid(d.tolist(), rays)                                       # the reference reads dist.ndim first
    big = Rays_GoldenSpiral(300)
    with pytest.raises(ValueError, match="at most 256 rays and 512 faces"):
        dist_to_volume(np.ones((1, 1, 1, 300), np.float32), big)


# ------------------------------------------------------------------------------------------------ host halves
def _compact_numpy(mask, nonzero, lo, hi, prob=None):
    m = np.asarray(mask)
    m = (m != 0) if nonzero else (m & 1).astype(bool)
    box = tuple(slice(a, b) for a, b in zip(lo, hi))
    idx = np.nonzero(m[box])
    return tuple((i + a).astype(np.int32) for i, a in zip(idx, lo)), None


@pytest.mark.parametrize("name", sorted(C.sample_points_cases()))
def test_sample_points_host_half(name, golden, no_device, monkeypatch):
    from stardist_b200 import utils as U
    monkeypatch.setattr(U, '_mask_compact_device', _compact_numpy)
    n, mask, prob, b, seed = C.sample_points_cases()[name]
    np.random.seed(seed)
    got = U.sample_points(n, mask, prob=prob, b=b)
    want = golden["sp/%s/out" % name]
    assert got.dtype == want.dtype and np.array_equal(got, want)
    assert _state_equals(golden, "sp/%s/state" % name)


def _gather_numpy(data, starts, extent):
    return np.stack([data[tuple(slice(s, s + e) for s, e in zip(st, extent))] for st in starts])


@pytest.mark.parametrize("name", sorted(C.sample_patches_cases()))
def test_sample_patches_host_half(name, golden, no_device, monkeypatch):
    import importlib
    SP = importlib.import_module("stardist_b200.sample_patches")           # the module; the package attribute is the function
    monkeypatch.setattr(SP, '_gather', _gather_numpy)
    datas, ps, n, vi, seed = C.sample_patches_cases()[name]
    if vi is not None:
        vi = tuple(golden["vi/%s/%d" % (name, a)] for a in range(len(ps)))
    np.random.seed(seed)
    if "spa/%s/error" % name in golden.files:
        with pytest.raises(ValueError) as e:
            SP.sample_patches(datas, ps, n, valid_inds=vi)
        assert str(e.value) == str(golden["spa/%s/error" % name])
    else:
        got = SP.sample_patches(datas, ps, n, valid_inds=vi)
        assert len(got) == len(datas)
        for k, g in enumerate(got):
            want = golden["spa/%s/out/%d" % (name, k)]
            assert g.dtype == want.dtype and np.array_equal(g, want)
    assert _state_equals(golden, "spa/%s/state" % name)


def test_get_valid_inds_without_filter(golden, no_device):
    from stardist_b200.sample_patches import get_valid_inds
    datas, ps, _, vi, _ = C.sample_patches_cases()['2d_even_valid_plain']
    got = get_valid_inds(datas[0], ps)
    for a, g in enumerate(got):
        want = golden["vi/2d_even_valid_plain/%d" % a]
        assert g.dtype == want.dtype == np.uint32 and np.array_equal(g, want)


# ------------------------------------------------------------------------------------------------ polyhedra restated
def poly_numpy(dist, verts, faces, absolute=None):
    """stardist3d_impl.cpp polyhedron_volume / polyhedron_centroid over all voxels at once: float32 products and sums, and
    the centroid's `R += .25 * (A + B + C) * vol` as a double product and double add rounded to float"""
    f32, f64 = np.float32, np.float64
    d = dist.astype(f32)
    vol = np.zeros(d.shape[:-1], f32)
    R = np.zeros(d.shape[:-1] + (3,), f32)
    for iA, iB, iC in faces:
        A, B, Cc = (d[..., i, None] * verts[i] for i in (iA, iB, iC))             # float32 [..., 3] (z, y, x)
        M0, M1, M2 = B - A, Cc - A, f32(0) - A
        det = (M0[..., 0] * (M1[..., 1] * M2[..., 2] - M2[..., 1] * M1[..., 2])
               - M0[..., 1] * (M1[..., 0] * M2[..., 2] - M1[..., 2] * M2[..., 0])
               + M0[..., 2] * (M1[..., 0] * M2[..., 1] - M1[..., 1] * M2[..., 0]))
        cv = det / f32(6)
        if absolute is not None:
            R = (R.astype(f64) + (0.25 * (A + B + Cc).astype(f64)) * cv.astype(f64)[..., None]).astype(f32)
        vol = vol + cv
    if absolute is None:
        return vol
    ok = vol.astype(f64) > 1e-10
    c = np.where(ok[..., None], R / np.where(ok, vol, f32(1))[..., None], f32(0)).astype(f32)
    if absolute:
        idx = np.stack(np.meshgrid(*[np.arange(s) for s in vol.shape], indexing='ij'), axis=-1).astype(f32)
        c = c + idx
    return c


@pytest.mark.parametrize("name", sorted(C.dist_cases()))
def test_polyhedra_restatement_equals_reference(name, golden):
    d, rays = C.dist_cases()[name]
    v, f = golden["dist/%s/verts" % name], golden["dist/%s/faces" % name]
    assert np.array_equal(v, np.float32(rays.vertices)) and np.array_equal(f, rays.faces)
    assert np.array_equal(poly_numpy(d, v, f), golden["dist/%s/volume" % name])
    assert np.array_equal(poly_numpy(d, v, f, True), golden["dist/%s/centroid_abs" % name])
    assert np.array_equal(poly_numpy(d, v, f, False), golden["dist/%s/centroid_rel" % name])


def test_fixture_cls_dicts_are_reference_order(golden):
    """the inverted dicts of the fixture list classes in first-occurrence order of the dict and labels in dict order"""
    from stardist_b200.utils import _invert_dict
    y, n, cls = C.categorical_cases()['2d_u16_dict_n5']
    want = json.loads(str(golden["m2c/2d_u16_dict_n5/cls_dict"]))
    assert [[k, v] for k, v in _invert_dict(cls).items()] == want
