"""mask_to_categorical, sample_points, sample_patches / get_valid_inds and dist_to_volume / dist_to_centroid on the device:
every case of tests/golden/helpers.npz (the reference's own functions and extension) bit for bit, with numpy and with
CUDA-tensor input, with the reference's np.random state after each draw; the polyhedra of a 64x256x256x96 random map and of a
3-D model's device predict equal the reference extension (oracle/_ref); and the class map of the 1024^2 benchmark ground
truth equals the reference's rule written out in numpy."""
import importlib, json, os, sys
import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
sys.path.insert(0, ROOT)
import helpers_cases as C

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def golden():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return np.load(os.path.join(HERE, "golden", "helpers.npz"))


def _sp():
    return importlib.import_module("stardist_b200.sample_patches")


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _state_equals(golden, key):
    _, k, pos, has_gauss, cached = np.random.get_state()
    return (np.array_equal(k, golden[key + "/key"]) and pos == golden[key + "/pos"]
            and np.array_equal([has_gauss, cached], golden[key + "/gauss"]))


@pytest.mark.parametrize("name", sorted(C.categorical_cases()))
def test_mask_to_categorical_equals_reference(name, golden):
    from stardist_b200.utils import mask_to_categorical
    y, n, cls = C.categorical_cases()[name]
    want = golden["m2c/%s/out" % name]
    want_dict = json.loads(str(golden["m2c/%s/cls_dict" % name]))
    for arg in (y, _cuda(y.astype(np.int32))):
        got, d = mask_to_categorical(arg, n, cls, return_cls_dict=True)
        got = got if isinstance(got, np.ndarray) else got.cpu().numpy()
        assert got.dtype == np.float32 and np.array_equal(got, want), name
        assert [[k, [int(l) for l in v]] for k, v in d.items()] == want_dict
        assert np.array_equal(mask_to_categorical(arg, n, cls) if isinstance(arg, np.ndarray) else
                              mask_to_categorical(arg, n, cls).cpu().numpy(), want)


def test_mask_to_categorical_device_errors(golden):
    import torch
    from stardist_b200.utils import mask_to_categorical
    y = np.array([[0, 1], [2, 5]], np.int32)
    with pytest.raises(ValueError) as e:
        mask_to_categorical(y, 2, {1: 1, 2: 2})
    assert str(e.value) == ("all gt labels should be present in class dict provided \ngt_labels found\n{1, 2, 5}\n"
                            "class dict labels provided\n{1, 2}")
    with pytest.raises(ValueError) as e:
        mask_to_categorical(y, 2, 3)                                           # the broadcast class is checked per label
    assert str(e.value) == "Wrong class id '3' (for n_classes=2)"
    assert np.array_equal(mask_to_categorical(np.zeros((2, 2), np.int32), 2, 3)[..., 0], np.ones((2, 2)))
    with pytest.raises(ValueError) as e:
        mask_to_categorical(_cuda(-y), 2, 1)
    assert str(e.value) == "y must be an array of non-negative integers."
    with pytest.raises(ValueError):
        mask_to_categorical(_cuda(y).to(torch.int64), 2, 1)


def test_mask_to_categorical_benchmark_ground_truth(golden):
    """1024^2 ground truth of the benchmark (about 1000 objects), random dict classes including None, against the reference's
    rule in numpy"""
    import bench_data
    from stardist_b200 import _lib
    from stardist_b200.utils import mask_to_categorical
    _, y = bench_data.synthetic_image((1024, 1024), seed=0)
    labels = np.unique(y[y > 0])
    assert len(labels) > 500
    rng = np.random.default_rng(0)
    cls = {int(l): [None, 0, 1, 2, 3][int(c)] for l, c in zip(labels, rng.integers(0, 5, len(labels)))}
    want = np.zeros(y.shape + (4,), np.float32)
    for l, c in cls.items():
        if c is None:
            want[y == l, :] = -1
        else:
            want[y == l, c] = 1
    want[..., 0] = (y == 0)
    _lib.launch_count(reset=True)
    got = mask_to_categorical(y, 3, cls)
    assert np.array_equal(got, want)
    assert _lib.launch_count() <= 8
    assert np.array_equal(mask_to_categorical(_cuda(y.astype(np.int32)), 3, cls).cpu().numpy(), want)


@pytest.mark.parametrize("name", sorted(C.sample_points_cases()))
def test_sample_points_equals_reference(name, golden):
    import torch
    from stardist_b200.utils import sample_points
    n, mask, prob, b, seed = C.sample_points_cases()[name]
    want = golden["sp/%s/out" % name]
    variants = [(mask, prob), (_cuda(mask), prob)]
    if prob is not None:
        variants.append((_cuda(mask), _cuda(prob)))
    for m, p in variants:
        np.random.seed(seed)
        got = sample_points(n, m, prob=p, b=b)
        assert got.dtype == want.dtype and np.array_equal(got, want), name
        assert _state_equals(golden, "sp/%s/state" % name)


def test_sample_points_empty_and_errors(golden):
    from stardist_b200 import _lib
    from stardist_b200.utils import sample_points
    m = np.zeros((20, 20), bool)
    m[0, :] = True                                                             # only on the border
    with pytest.raises(ValueError, match="a must be greater than 0"):
        sample_points(3, m, b=2)
    _lib.launch_count(reset=True)
    with pytest.raises(ValueError):
        sample_points(3, _cuda(m), prob=_cuda(np.ones((20, 21), np.float32)))
    assert _lib.launch_count() == 0


def test_sample_points_device_predict(golden):
    """sample_points(200, prob > 0.2) on a device-resident 2-D predict equals the same call on the numpy maps"""
    from stardist_b200 import Config2D, StarDist2D
    from stardist_b200.utils import sample_points
    model = StarDist2D(Config2D(n_rays=32), name=None, basedir=None)
    img = np.random.default_rng(5).uniform(0, 1, (256, 320)).astype(np.float32)
    prob_d = model._predict_device(img)[0]
    prob = prob_d.cpu().numpy()
    thr = float(np.quantile(prob, 0.5))
    np.random.seed(9)
    want = sample_points(200, prob > thr, prob=prob)
    state = np.random.get_state()
    np.random.seed(9)
    got = sample_points(200, prob_d > thr, prob=prob_d)
    assert np.array_equal(got, want)
    assert all(np.array_equal(a, b) for a, b in zip(np.random.get_state(), state))


def _datas_as_tensors(datas):
    return [_cuda(a) for a in datas if a.dtype.kind != 'S']


@pytest.mark.parametrize("name", sorted(C.sample_patches_cases()))
def test_sample_patches_equals_reference(name, golden):
    SP = _sp()
    datas, ps, n, vi, seed = C.sample_patches_cases()[name]
    if vi is not None:
        filt = None if vi == 'plain' else C.FILTERS[vi]
        got_vi = SP.get_valid_inds(datas[0], ps, filt)
        vi = tuple(golden["vi/%s/%d" % (name, a)] for a in range(len(ps)))
        assert len(got_vi) == len(vi) and all(g.dtype == np.uint32 and np.array_equal(g, w) for g, w in zip(got_vi, vi))
        if filt is not None:                                                   # a filter that returns a CUDA mask
            got_t = SP.get_valid_inds(datas[0], ps, lambda img, p: _cuda(filt(img, p)))
            assert all(np.array_equal(g, w) for g, w in zip(got_t, vi))
    err = golden.get("spa/%s/error" % name)
    for ds in (datas, _datas_as_tensors(datas)):
        np.random.seed(seed)
        if err is not None:
            with pytest.raises(ValueError) as e:
                SP.sample_patches(ds, ps, n, valid_inds=vi)
            assert str(e.value) == str(err)
        else:
            got = SP.sample_patches(ds, ps, n, valid_inds=vi)
            want = [golden["spa/%s/out/%d" % (name, k)] for k, a in enumerate(datas) if ds is datas or a.dtype.kind != 'S']
            assert len(got) == len(want)
            for g, w in zip(got, want):
                g = g if isinstance(g, np.ndarray) else g.cpu().numpy()
                assert g.dtype == w.dtype and np.array_equal(g, w), name
        assert _state_equals(golden, "spa/%s/state" % name)


@pytest.mark.parametrize("name", sorted(C.dist_cases()))
def test_dist_to_polyhedra_equal_reference(name, golden):
    from stardist_b200.geometry.geom3d import dist_to_volume, dist_to_centroid
    d, rays = C.dist_cases()[name]
    for arg in (d, _cuda(d)):
        for got, key in ((dist_to_volume(arg, rays), "volume"), (dist_to_centroid(arg, rays), "centroid_abs"),
                         (dist_to_centroid(arg, rays, mode='relative'), "centroid_rel")):
            got = got if isinstance(got, np.ndarray) else got.cpu().numpy()
            want = golden["dist/%s/%s" % (name, key)]
            assert got.dtype == np.float32 and got.shape == want.shape and np.array_equal(got, want), (name, key)


def _ref_poly(d, rays):
    from oracle import ref_ext
    if not ref_ext.available():
        pytest.skip("oracle/_ref not present")
    ext = ref_ext.stardist3d()
    v = np.ascontiguousarray(rays.vertices, np.float32); f = np.ascontiguousarray(rays.faces, np.int32)
    return ext.c_dist_to_volume(d, v, f), ext.c_dist_to_centroid(d, v, f, np.int32(1))


def test_dist_to_polyhedra_large_map(golden):
    from stardist_b200.geometry.geom3d import dist_to_volume, dist_to_centroid
    from stardist_b200.rays3d import Rays_GoldenSpiral
    rays = Rays_GoldenSpiral(96)
    d = np.random.default_rng(21).uniform(0.5, 12, (64, 256, 256, 96)).astype(np.float32)
    vol_ref, cen_ref = _ref_poly(d, rays)
    d_t = _cuda(d)
    assert np.array_equal(dist_to_volume(d_t, rays).cpu().numpy(), vol_ref)
    assert np.array_equal(dist_to_centroid(d_t, rays).cpu().numpy(), cen_ref)


def test_dist_to_volume_of_a_device_predict(golden):
    from stardist_b200 import Config3D, StarDist3D, Rays_GoldenSpiral
    from stardist_b200.geometry.geom3d import dist_to_volume, dist_to_centroid
    rays = Rays_GoldenSpiral(96)
    model = StarDist3D(Config3D(rays=rays), name=None, basedir=None)
    k, b = model.weights['dist']; model.weights['dist'] = (k, b + np.float32(4.0)); model._net = None
    vol = np.random.default_rng(22).uniform(0, 1, (24, 48, 40)).astype(np.float32)
    dist_d = model._predict_device(vol)[1]
    dist = dist_d.cpu().numpy()
    vol_ref, cen_ref = _ref_poly(dist, rays)
    assert np.array_equal(dist_to_volume(dist_d, rays).cpu().numpy(), vol_ref)
    assert np.array_equal(dist_to_centroid(dist_d, rays).cpu().numpy(), cen_ref)
