"""Training batches on the device (stardist_b200.models.StarDistData2D / StarDistData3D) against the reference's own
generators (tests/golden/train_batch.npz), the reference test's assertions, the per-patch composition of the pinned
star_dist_device / edt_prob_device, batch-item independence, and argument errors."""
import json, os, sys, warnings
import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
sys.path.insert(0, os.path.dirname(HERE))
import train_batch_cases as C

pytestmark = pytest.mark.gpu


def _meta():
    z = np.load(os.path.join(HERE, "golden", "train_batch.npz"))
    return json.loads(bytes(z["meta"]).decode()), z


def _make(name):
    from stardist_b200.models import StarDistData2D, StarDistData3D
    from stardist_b200.rays3d import Rays_GoldenSpiral
    dim, X, Y, kw, seed, batches = C.cases()[name]
    np.random.seed(seed)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        gen = (StarDistData2D if dim == 2 else StarDistData3D)(X, Y, **C.make_kwargs(kw, Rays_GoldenSpiral))
    return gen, batches


def _ulp(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64))


@pytest.mark.parametrize("name", sorted(C.cases()))
def test_fixture_batches(name):
    meta, z = _meta()
    rec = meta[name]
    gen, batches = _make(name)
    ulp_case = name in C.ulp_cases()
    host = []
    for i, b in zip(batches, rec["batches"]):
        assert [int(v) for v in gen.batch(i)] == b["index"]
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            (x,), outs = gen[i]
        assert sum("constant label image" in str(m.message) for m in w) == b["n_constant"]
        assert gen.last_positions.cpu().numpy().tolist() == b["positions"]
        arrs = (x,) + tuple(outs)
        assert len(arrs) == len(b["outputs"])
        for k, (a, (shape, dtype, h)) in enumerate(zip(arrs, b["outputs"])):
            assert list(a.shape) == shape and str(a.dtype) == dtype, (k, a.shape, a.dtype, shape, dtype)
            if ulp_case and k in (1, 2):
                continue
            assert C.sha(a) == h, "output %d of batch %d differs" % (k, i)
        if ulp_case:
            R = outs[1].shape[-1] - 1
            pw, dw = z["%s/%d/prob" % (name, i)], z["%s/%d/dist_mask" % (name, i)]
            d1, d2 = _ulp(outs[0], pw), _ulp(outs[1][..., R], dw)
            assert d1.max() <= 1 and d2.max() <= 1
            print("%s batch %d: %d prob / %d dist_mask values 1 ulp off" % (name, i, int((d1 > 0).sum()), int((d2 > 0).sum())))
        host.append(arrs)
    # batch_device gives the same, element for element, from the same stream
    gen, batches = _make(name)
    for i, arrs in zip(batches, host):
        gen.batch(i)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            (x,), outs = gen.batch_device(i)
        for a, d in zip(arrs, (x,) + tuple(outs)):
            assert d.is_cuda and np.array_equal(d.cpu().numpy(), a)


@pytest.mark.parametrize("name", [n for n in sorted(C.cases()) if n.endswith("_neg")])
def test_reference_negative_label_assertions(name):
    """test_model2D.py::test_stardistdata: prob == -1, dist_mask == 0, dist == 0 (and prob_class == -1) on the negative mask"""
    gen, _ = _make(name)
    Y = C.cases()[name][2][0]
    mask_neg = (Y < 0)[gen.ss_grid[1:3]]
    (x,), b = gen[0]
    prob, dist, dist_mask = b[0][0, ..., 0], b[1][0, ..., :-1], b[1][0, ..., -1]
    assert mask_neg.any()
    assert np.all(prob[mask_neg] == -1) and np.all(dist_mask[mask_neg] == 0) and np.all(dist[mask_neg] == 0)
    if len(b) == 3:
        assert np.all(b[2][0][mask_neg] == -1)


def _compose(gen, outs, Y, dim):
    """the per-patch composition of star_dist_device / star_dist3D_device and edt_prob_device on the same crops"""
    import torch
    from stardist_b200.geometry.distances import star_dist_device, star_dist3D_device
    from stardist_b200.labelprep import edt_prob_device
    pos = gen.last_positions.cpu().numpy()
    prob, dam = outs[0].cpu().numpy(), outs[1].cpu().numpy()
    for b, k in enumerate(gen.last_index):
        sl = tuple(slice(r - p // 2, r - p // 2 + p) for r, p in zip(pos[b], gen.patch_size))
        crop = torch.from_numpy(np.ascontiguousarray(np.maximum(Y[k][sl], 0), dtype=np.int32)).cuda()
        if dim == 2:
            d = star_dist_device(crop, gen.n_rays, gen.grid)
            e = edt_prob_device(crop[gen.ss_grid[1:]].contiguous())
        else:
            d = star_dist3D_device(crop, gen.rays, gen.grid)
            e = edt_prob_device(crop, gen.anisotropy)[gen.ss_grid[1:]]
        assert np.array_equal(dam[b, ..., :-1], d.cpu().numpy())
        assert np.array_equal(prob[b, ..., 0], e.cpu().numpy()) and np.array_equal(dam[b, ..., -1], e.cpu().numpy())


def test_composition_at_size_2d():
    import bench_data
    from stardist_b200.models import StarDistData2D
    Y = [bench_data.ellipse_labels((1024, 1024), seed=s) for s in range(2)]
    X = [y.astype(np.float32) for y in Y]
    np.random.seed(0)
    gen = StarDistData2D(X, Y, batch_size=8, n_rays=32, length=4, patch_size=(256, 256), grid=(2, 2), foreground_prob=0.9)
    for i in range(2):
        (x,), outs = gen.batch_device(i)
        _compose(gen, outs, Y, 2)


def test_composition_at_size_3d():
    import bench_data
    from stardist_b200.models import StarDistData3D
    from stardist_b200.rays3d import Rays_GoldenSpiral
    Y = [bench_data.ellipsoid_labels((128, 256, 256), seed=0)]
    X = [y.astype(np.float32) for y in Y]
    np.random.seed(0)
    gen = StarDistData3D(X, Y, batch_size=2, rays=Rays_GoldenSpiral(96), length=2, patch_size=(64, 128, 128), grid=(1, 2, 2),
                         anisotropy=(2, 1, 1))
    (x,), outs = gen.batch_device(0)
    _compose(gen, outs, Y, 3)


def test_batch_boundary():
    """an object that touches the edge shared by consecutive items in memory gets the targets of its patch alone"""
    from stardist_b200.models import StarDistData2D
    y0 = np.zeros((16, 16), np.int32); y0[10:16, 3:12] = 1              # touches the bottom edge of item 0
    y1 = np.zeros((16, 16), np.int32); y1[0:5, 4:10] = 2                # touches the top edge of item 1
    X = [np.zeros((16, 16), np.float32)] * 2
    together = StarDistData2D(X, [y0, y1], batch_size=2, n_rays=8, length=1, patch_size=(16, 16))
    np.random.seed(1)
    _, outs = together[0]
    order = [int(v) for v in together.last_index]
    for b, k in enumerate(order):
        alone = StarDistData2D([X[k]], [[y0, y1][k]], batch_size=1, n_rays=8, length=1, patch_size=(16, 16))
        _, o = alone[0]
        assert np.array_equal(outs[0][b], o[0][0]) and np.array_equal(outs[1][b], o[1][0])


def test_argument_errors_launch_nothing():
    from stardist_b200 import _lib
    from stardist_b200.models import StarDistData2D
    y = np.zeros((32, 32), np.int32); y[4:9, 4:9] = 1
    x = np.zeros((32, 32), np.float32)
    kw = dict(batch_size=1, n_rays=8, length=1, patch_size=(16, 16))
    _lib.launch_count(reset=True)
    with pytest.raises(NotImplementedError):
        StarDistData2D([x], [y], shape_completion=True, **kw)
    with pytest.raises(ValueError):
        StarDistData2D((v for v in [x]), [y], **kw)
    with pytest.raises(ValueError):
        StarDistData2D([x], [y], **dict(kw, patch_size=(64, 16)))
    with pytest.raises(ValueError):
        StarDistData2D([x, x], [y], **kw)
    with pytest.raises(AssertionError):
        StarDistData2D([x], [y], foreground_prob=1.5, **kw)
    with pytest.raises(ValueError):
        StarDistData2D([x], [y], n_classes=2, classes=[{1: 3}], **kw)
    with pytest.raises(ValueError):
        StarDistData2D([x], [y.astype(np.int64) + 2 ** 31], **kw)
    assert _lib.launch_count() == 0
