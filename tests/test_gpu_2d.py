"""GPU parity tests of the 2D path (run on the H100 box: pytest -m gpu).  Everything goes through
the C ABI of libstardist_b200.so; the checker is the oracle (reference C++ in oracle/_ref, numpy
restatements) and the committed golden vectors.  Integer/index results must be bit-exact."""
import os, sys
import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import cases
from oracle import ref_ext, geom2d_np, nms_np, unet_torch, pipeline2d

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sd():
    import stardist_b200
    from stardist_b200 import _lib
    _lib.require_cuda()
    return stardist_b200


@pytest.mark.parametrize("name", list(cases.NMS2D_CASES))
@pytest.mark.parametrize("use_kdtree", [1, 0])
def test_nms2d_golden(sd, name, use_kdtree, golden_dir):
    from stardist_b200.lib.stardist2d import c_non_max_suppression_inds
    g = np.load(os.path.join(golden_dir, "nms2d.npz"))
    d, p, s, thr = cases.nms2d_inputs(name)
    keep = c_non_max_suppression_inds(d, p, use_kdtree, 1, 0, thr)
    want = np.unpackbits(g["%s/keep_kd%d" % (name, use_kdtree)])[:len(d)].astype(bool)
    assert keep.dtype == np.bool_ and np.array_equal(keep, want)


@pytest.mark.parametrize("n,R,radius,noise,thr,seed", [(20000, 32, 8, .2, .4, 0), (5000, 96, 12, .3, .5, 1),
                                                       (3000, 32, 1.5, .9, .3, 2), (1, 32, 5, 0, .4, 3), (2, 7, 5, .1, .4, 4)])
def test_nms2d_vs_reference_ext(sd, n, R, radius, noise, thr, seed):
    """random candidate clouds (incl. degenerate tiny polygons): product == reference C++"""
    from stardist_b200.lib.stardist2d import c_non_max_suppression_inds
    rng = np.random.default_rng(seed)
    pts = rng.integers(0, 300, (n, 2)).astype(np.float32)
    dist = (radius * (1 + noise * rng.uniform(-1, 1, (n, R)))).astype(np.float32)
    dist = np.maximum(np.float32(1e-3), dist)
    for use_bbox in (1, 0):
        want = ref_ext.stardist2d().c_non_max_suppression_inds(dist, pts, 1, use_bbox, 0, np.float32(thr))
        got = c_non_max_suppression_inds(dist, pts, 1, use_bbox, 0, np.float32(thr))
        assert np.array_equal(got, want)


def test_nms2d_empty_and_errors(sd):
    from stardist_b200.lib.stardist2d import c_non_max_suppression_inds
    out = c_non_max_suppression_inds(np.zeros((0, 32), np.float32), np.zeros((0, 2), np.float32), 1, 1, 0, np.float32(.4))
    assert out.shape == (0,)
    with pytest.raises(TypeError):
        c_non_max_suppression_inds(np.zeros((2, 32)), np.zeros((2, 2), np.float32), 1, 1, 0, np.float32(.4))


def test_dist_to_coord_bit_exact(sd):
    rng = np.random.default_rng(0)
    for R in (32, 11, 96):
        dist = rng.uniform(0.001, 50, (500, R)).astype(np.float32)
        pts = rng.integers(0, 4000, (500, 2))
        got = sd.dist_to_coord(dist, pts)
        want = geom2d_np.dist_to_coord(dist, pts)
        assert got.dtype == np.float32 and np.array_equal(got.view(np.int32), want.view(np.int32))
        got = sd.dist_to_coord(dist, pts * np.array([2.0, 0.5]), scale_dist=(2.0, 0.5))
        want = geom2d_np.dist_to_coord(dist, pts * np.array([2.0, 0.5]), scale_dist=(2.0, 0.5))
        assert np.array_equal(got.view(np.int32), want.view(np.int32))


def test_polygons_to_label_bit_exact(sd):
    rng = np.random.default_rng(1)
    shape = (257, 301)
    for R, n in ((32, 300), (8, 50), (64, 100)):
        pts = rng.integers(-5, 310, (n, 2))
        dist = (rng.uniform(2, 18, (n, 1)) * (1 + .3 * rng.uniform(-1, 1, (n, R)))).astype(np.float32)
        prob = rng.uniform(0, 1, n).astype(np.float32)
        prob[::7] = prob[3]           # ties
        got = sd.polygons_to_label(dist, pts, shape, prob=prob)
        want = geom2d_np.polygons_to_label(dist, pts, shape, prob=prob)
        assert got.dtype == np.int32 and np.array_equal(got, want)
    assert np.array_equal(sd.polygons_to_label(np.zeros((0, 32), np.float32), np.zeros((0, 2), int), shape),
                          np.zeros(shape, np.int32))


def test_threshold_sort_gather(sd):
    import torch, ctypes
    from stardist_b200 import _lib as L
    lib = L.require_cuda()
    rng = np.random.default_rng(2)
    for shape, grid, b in (((130, 77), (1, 1), 2), ((64, 64), (2, 2), 2), ((9, 40, 33), (1, 2, 2), 2), ((50, 60), (1, 1), 0)):
        nd = len(shape)
        prob = rng.uniform(0, 1, shape).astype(np.float32)
        prob.flat[::13] = prob.flat[5]       # ties
        R = 5
        dist = rng.uniform(-1, 10, shape + (R,)).astype(np.float32)
        valid = tuple(s - 3 for s in shape)
        pd = torch.from_numpy(prob).cuda(); dd = torch.from_numpy(dist).cuda()
        npix = prob.size
        sidx = torch.empty(npix, dtype=torch.int32, device='cuda'); sprob = torch.empty(npix, dtype=torch.float32, device='cuda')
        cnt = ctypes.c_int(0)
        L.check(lib.sdb_threshold_sort(L.ptr(pd), nd, L.iarr(shape), L.iarr(valid), L.iarr([b] * nd), L.iarr([b] * nd),
                                      0.6, L.ptr(sidx), L.ptr(sprob), npix, ctypes.byref(cnt), L.stream_ptr()))
        n = cnt.value
        mask = nms_np._ind_prob_thresh(prob, np.float32(0.6), b=(b if b > 0 else None))
        idx = np.stack(np.where(mask), 1)
        ok = np.all(idx < np.array(valid), 1)
        flat = np.ravel_multi_index(idx[ok].T, shape)
        order = np.argsort(prob.ravel()[flat], kind='stable')[::-1]
        want_idx = flat[order]
        assert n == len(want_idx)
        assert np.array_equal(sidx[:n].cpu().numpy(), want_idx)
        assert np.array_equal(sprob[:n].cpu().numpy(), prob.ravel()[want_idx])
        od = torch.empty((n, R), dtype=torch.float32, device='cuda'); op = torch.empty((n, nd), dtype=torch.float32, device='cuda')
        L.check(lib.sdb_gather_candidates(L.ptr(dd), L.ptr(sidx), n, R, nd, L.iarr(shape), L.iarr(grid), L.ptr(od), L.ptr(op), L.stream_ptr()))
        assert np.array_equal(od.cpu().numpy(), np.maximum(np.float32(1e-3), dist.reshape(-1, R)[want_idx]))
        assert np.array_equal(op.cpu().numpy(), (np.stack(np.unravel_index(want_idx, shape), 1) * np.array(grid)).astype(np.float32))


@pytest.mark.parametrize("shape,grid", [((64, 96), (1, 1)), ((48, 80), (2, 2))])
def test_unet_forward_vs_torch_fp32(sd, shape, grid):
    """float outputs: tolerance 1e-5 relative to the map's scale (north_star), vs torch-CPU fp32"""
    import torch
    cfg = sd.Config2D(n_rays=32, grid=grid)
    model = sd.StarDist2D(cfg, name=None, basedir=None)
    rng = np.random.default_rng(3)
    img = rng.uniform(0, 1, shape).astype(np.float32)
    x = torch.from_numpy(img[None, ..., None]).cuda()
    prob, dist = model.net.forward(x)
    rp, rd = unet_torch.forward(cfg, model.weights, img[None, ..., None])
    p, d = prob.cpu().numpy(), dist.cpu().numpy()
    assert p.shape == rp.shape and d.shape == rd.shape
    assert np.max(np.abs(p - rp)) <= 1e-5 * max(1.0, np.max(np.abs(rp)))
    assert np.max(np.abs(d - rd)) <= 1e-5 * max(1e-3, np.max(np.abs(rd))) + 1e-7


@pytest.mark.parametrize("shape", [(96, 128), (101, 75)])
def test_predict_instances_vs_oracle(sd, shape):
    """whole pipeline: integer outputs bit-exact given the same network maps; also the reference
    invariants dense == sparse (tests/test_model2D.py:442-449)"""
    cfg = sd.Config2D(n_rays=32)
    model = sd.StarDist2D(cfg, name=None, basedir=None)
    rng = np.random.default_rng(4)
    img = rng.uniform(0, 1, shape).astype(np.float32)
    pthr = pipeline2d.quantile_prob_thresh(model, img, 0.95)
    labels, res = model.predict_instances(img, prob_thresh=pthr, nms_thresh=0.3)
    ref_labels, ref = pipeline2d.predict_instances(cfg, model.weights, img, pthr, 0.3, cand_from=model)
    assert labels.shape == shape and len(res['prob']) > 3
    assert np.array_equal(res['points'], ref['points'])
    assert np.array_equal(res['prob'], ref['prob'])
    assert np.array_equal(res['coord'].view(np.int32), ref['coord'].view(np.int32))
    assert np.array_equal(labels, ref_labels)
    if shape[0] % 8 == 0 and shape[1] % 8 == 0:
        l2, r2 = model.predict_instances(img, prob_thresh=pthr, nms_thresh=0.3, sparse=False)
        assert np.array_equal(labels, l2) and np.array_equal(res['points'], r2['points'])


def test_nms2d_survivors_and_paint_order(sd):
    """device-side survivor list + paint order (incl. tied scores) == numpy on the keep mask"""
    import torch, ctypes
    from stardist_b200 import _lib as L
    from stardist_b200.geometry.geom2d import paint_order
    lib = L.require_cuda()
    rng = np.random.default_rng(5)
    n, R = 6000, 32
    pts = rng.integers(0, 200, (n, 2)).astype(np.float32)
    dist = (9 * (1 + 0.2 * rng.uniform(-1, 1, (n, R)))).astype(np.float32)
    prob = np.round(rng.uniform(0.5, 1, n), 2).astype(np.float32)          # many ties
    o = np.argsort(prob, kind='stable')[::-1]
    dist, pts, prob = np.ascontiguousarray(dist[o]), np.ascontiguousarray(pts[o]), np.ascontiguousarray(prob[o])
    d_d, p_d = torch.from_numpy(dist).cuda(), torch.from_numpy(pts).cuda()
    keep = torch.zeros(n, dtype=torch.uint8, device='cuda'); sel = torch.empty(n, dtype=torch.int32, device='cuda')
    nk = ctypes.c_int(0)
    L.check(lib.sdb_nms2d_survivors(L.ptr(d_d), L.ptr(p_d), n, R, 0.4, 1, 1, 0, L.ptr(keep), L.ptr(sel), ctypes.byref(nk), L.stream_ptr()))
    keep_h = keep.cpu().numpy().astype(bool)
    want = ref_ext.stardist2d().c_non_max_suppression_inds(dist, pts, 1, 1, 0, np.float32(0.4))
    assert np.array_equal(keep_h, want)
    assert nk.value == int(want.sum()) and np.array_equal(sel[:nk.value].cpu().numpy(), np.nonzero(want)[0])
    pk = torch.from_numpy(prob[want]).cuda()
    rank = torch.empty(nk.value, dtype=torch.int32, device='cuda'); ids = torch.empty(nk.value, dtype=torch.int32, device='cuda')
    L.check(lib.sdb_paint_order_2d(L.ptr(pk), nk.value, L.ptr(rank), L.ptr(ids), L.stream_ptr()))
    ind, rk = paint_order(prob[want])
    assert np.array_equal(rank.cpu().numpy(), rk) and np.array_equal(ids.cpu().numpy(), ind + 1)


@pytest.mark.parametrize("shape,n_tiles", [((200, 312), (2, 3)), ((136, 120), (1, 2)), ((264, 264), (4, 4))])
def test_predict_n_tiles_equals_untiled(sd, shape, n_tiles):
    """n_tiles (base.py:446-529): tile-by-tile network passes with receptive-field overlap give the same maps and
    the same instances as the single pass"""
    rng = np.random.default_rng(shape[0])
    img = rng.uniform(0, 1, shape).astype(np.float32)
    model = sd.StarDist2D(sd.Config2D(n_rays=32), name=None, basedir=None)
    p1, d1 = model.predict(img)
    p2, d2 = model.predict(img, n_tiles=n_tiles)
    assert p1.shape == p2.shape == shape and d1.shape == d2.shape
    # same per-pixel arithmetic, but small tiles may pick a different tensor-core kernel variant (summation order):
    # equal to the float tolerance of the maps, not bitwise
    assert np.max(np.abs(p1 - p2)) <= 1e-5 * max(1.0, np.max(np.abs(p1)))
    assert np.max(np.abs(d1 - d2)) <= 1e-5 * max(1e-3, np.max(np.abs(d1))) + 1e-7
    thr = float(np.quantile(p1, 0.97))
    l1, r1 = model.predict_instances(img, prob_thresh=thr, nms_thresh=0.4)
    l2, r2 = model.predict_instances(img, prob_thresh=thr, nms_thresh=0.4, n_tiles=n_tiles)
    assert abs(len(r1['prob']) - len(r2['prob'])) <= max(2, len(r1['prob']) // 100)
    assert np.mean(l1 != l2) < 5e-3
    with pytest.raises(ValueError):
        model.predict(img[..., None], axes='YXC', n_tiles=(1, 1, 2))


def test_reference_2d_demo_model_reproduces_reference_test(sd):
    """The reference's shipped `2D_demo` weights (tests/golden/demo2d.npz) on its test image through the product path:
    matching(mask, labels, 0.5) must give the numbers the reference's own test pins, (fp, tp, fn) == (5, 114, 11)
    (stardist tests/test_model2D.py:92-106), and the instances must equal the CPU oracle's."""
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    import demo2d
    from stardist_b200.utils import normalize
    from stardist_b200.matching import matching
    kwargs, weights, thr, img, mask = demo2d.load()
    cfg = sd.Config2D(**kwargs)
    model = sd.StarDist2D(cfg, name=None, basedir=None, weights=weights)
    model.thresholds = dict(prob=thr['prob'], nms=thr['nms'])
    x = normalize(img, 1, 99.8)
    prob, dist = model.predict(x, n_tiles=(2, 3))
    assert prob.shape == dist.shape[:2] and dist.shape[-1] == cfg.n_rays
    labels, polygons = model.predict_instances(x)
    assert labels.shape == img.shape[:2]
    assert labels.max() == len(polygons['coord']) == len(polygons['points']) == len(polygons['prob'])
    st = matching(mask, labels, thresh=0.5)
    assert (st.fp, st.tp, st.fn) == demo2d.REFERENCE_TEST_STATS
    ref_labels, ref = pipeline2d.predict_instances(cfg, weights, x, thr['prob'], thr['nms'])
    assert np.array_equal(polygons['points'], ref['points'])
    assert np.mean(labels != ref_labels) < 1e-3          # the oracle ran its own (torch-CPU) network: float-induced tolerance
    # the integer path on the trained model's real maps: same floats in (cand_from=model), bit-equal results out
    labels2, polygons2 = model.predict_instances(x)
    ex_labels, ex = pipeline2d.predict_instances(cfg, weights, x, thr['prob'], thr['nms'], cand_from=model)
    assert np.array_equal(polygons2['points'], ex['points']) and np.array_equal(polygons2['prob'], ex['prob'])
    assert np.array_equal(polygons2['coord'].view(np.int32), ex['coord'].view(np.int32)) and np.array_equal(labels2, ex_labels)
    # float maps of the TRAINED network (tensor-core path) against a float64 evaluation: the 1e-5 relative bar
    import torch
    prob1, dist1 = model.predict(x)
    rp64, rd64 = unet_torch.forward(cfg, weights, x[None, ..., None].astype(np.float32), dtype=torch.float64)
    rd64 = np.maximum(1e-3, rd64[0])
    assert np.max(np.abs(prob1 - rp64[0])) <= 1e-5 * max(1.0, np.max(np.abs(rp64)))
    assert np.max(np.abs(dist1 - rd64)) <= 1e-5 * np.max(np.abs(rd64))



@pytest.mark.parametrize("grid", [(1, 1), (2, 2)])
def test_multiclass_head(sd, grid):
    """n_classes: extra features_class conv + softmax head (model2d.py:339-347); predict returns (prob, dist, prob_class),
    predict_instances adds class_prob / class_id of the survivors (model2d.py:556-560), sparse == dense path"""
    rng = np.random.default_rng(11)
    img = rng.uniform(0, 1, (80, 144)).astype(np.float32)      # divisible by 8 * grid: the oracle gets the unpadded image
    cfg = sd.Config2D(n_rays=32, grid=grid, n_classes=3)
    model = sd.StarDist2D(cfg, name=None, basedir=None)
    assert 'features_class' in model.weights and model.weights['prob_class'][0].shape[-1] == 4
    prob, dist, pc = model.predict(img)
    rp, rd, rpc = unet_torch.forward(cfg, model.weights, img[None, ..., None])
    assert pc.shape == prob.shape + (4,)
    assert np.max(np.abs(prob - rp[0])) <= 1e-5 and np.max(np.abs(pc - rpc[0])) <= 1e-5
    assert np.allclose(pc.sum(-1), 1, atol=1e-5)
    thr = float(np.quantile(prob, 0.95))
    labels, res = model.predict_instances(img, prob_thresh=thr, nms_thresh=0.4)
    assert res['class_prob'].shape == (len(res['prob']), 4)
    pts = res['points'] // np.array(grid)
    assert np.array_equal(res['class_prob'], pc[pts[:, 0], pts[:, 1]])
    assert np.array_equal(res['class_id'], np.argmax(res['class_prob'], -1))
    labels2, res2 = model.predict_instances(img, prob_thresh=thr, nms_thresh=0.4, sparse=False)
    assert np.array_equal(labels, labels2) and np.array_equal(res['class_id'], res2['class_id'])


def test_cli_predict_on_model_folder(sd, tmp_path):
    """python -m stardist_b200.scripts.predict on a model folder (config.json + thresholds.json + weights.npz) and a TIFF:
    the written label image equals predict_instances on the same normalised input; ROI set has one entry per instance"""
    import json, zipfile
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    import demo2d
    from stardist_b200.io import tiff
    from stardist_b200.utils import normalize
    from stardist_b200.scripts import predict as cli
    kwargs, weights, thr, img, mask = demo2d.load()
    folder = tmp_path / "demo_model"; folder.mkdir()
    cfg = sd.Config2D(**kwargs)
    json.dump({k: v for k, v in vars(cfg).items() if isinstance(v, (int, float, str, bool, list, tuple, type(None), dict))}, open(folder / "config.json", "w"))
    json.dump(thr, open(folder / "thresholds.json", "w"))
    np.savez(folder / "weights.npz", **{n + "/kernel": k for n, (k, b) in weights.items()}, **{n + "/bias": b for n, (k, b) in weights.items()})
    tiff.imwrite(tmp_path / "nuclei.tif", img)
    written = cli.main(["-i", str(tmp_path / "nuclei.tif"), "-m", str(folder), "-o", str(tmp_path / "out"), "--n_tiles", "2", "2", "--rois"])
    labels = tiff.imread(written[0])
    model = sd.StarDist2D(None, name="demo_model", basedir=str(tmp_path))
    ref_labels, res = model.predict_instances(normalize(img, 1, 99.8), n_tiles=(2, 2))
    assert np.array_equal(labels, ref_labels) and labels.max() == len(res['prob'])
    with zipfile.ZipFile(str(tmp_path / "out" / "nuclei.stardist.rois.zip")) as z:
        assert len(z.namelist()) == len(res['prob'])


@pytest.mark.parametrize("grid", [(2, 1), (1, 2), (4, 2)])
def test_anisotropic_grid_vs_oracle(sd, grid):
    """grids with different factors per axis (valid in the reference: the grid stem pools (2,1) / (1,2), model2d.py:316-325)
    must not run on the 2x2-only tensor-core executor: maps equal the torch restatement, instances equal the oracle's"""
    import torch
    from stardist_b200.models.unet_device import UNetDevice2DTC
    cfg = sd.Config2D(n_rays=32, grid=grid)
    assert not UNetDevice2DTC.supported(cfg)
    model = sd.StarDist2D(cfg, name=None, basedir=None)
    rng = np.random.default_rng(5)
    img = rng.uniform(0, 1, (96, 128)).astype(np.float32)
    prob, dist = model.net.forward(torch.from_numpy(img[None, ..., None]).cuda())
    rp, rd = unet_torch.forward(cfg, model.weights, img[None, ..., None])
    assert tuple(prob.shape) == rp.shape == (1, 96 // grid[0], 128 // grid[1])
    assert np.max(np.abs(prob.cpu().numpy() - rp)) <= 1e-5 and np.max(np.abs(dist.cpu().numpy() - rd)) <= 1e-5 * max(1e-3, np.max(np.abs(rd))) + 1e-7
    pthr = pipeline2d.quantile_prob_thresh(model, img, 0.9)
    labels, res = model.predict_instances(img, prob_thresh=pthr, nms_thresh=0.3)
    ref_labels, ref = pipeline2d.predict_instances(cfg, model.weights, img, pthr, 0.3, cand_from=model)
    assert len(res['prob']) > 0 and np.array_equal(res['points'], ref['points']) and np.array_equal(labels, ref_labels)


def test_unnormalised_input_does_not_overflow_silently(sd):
    """raw 16-bit input drives activations past the fp16 range of the tensor-core representation; the pass must be
    repeated on the fp32 kernels (with a warning) and give the finite maps of the fp32 reference network"""
    import torch, warnings
    cfg = sd.Config2D(n_rays=32)
    model = sd.StarDist2D(cfg, name=None, basedir=None)
    rng = np.random.default_rng(6)
    img = (rng.integers(0, 65535, (64, 96)).astype(np.float32) * 64)         # e.g. a 22-bit sensor / un-normalised float data
    with warnings.catch_warnings(record=True) as wlist:
        warnings.simplefilter("always")
        prob, dist = model.predict(img)
    assert any("fp16 range" in str(w.message) for w in wlist)
    rp, rd = unet_torch.forward(cfg, model.weights, img.astype(np.float32)[None, ..., None])
    assert np.isfinite(dist).all() and np.isfinite(prob).all()
    assert np.max(np.abs(dist - np.maximum(1e-3, rd[0]))) <= 1e-4 * np.max(np.abs(rd))
    # a normalised image afterwards runs on the tensor cores again, no warning
    with warnings.catch_warnings(record=True) as wlist:
        warnings.simplefilter("always")
        model.predict(rng.uniform(0, 1, (64, 96)).astype(np.float32))
    assert not any("fp16 range" in str(w.message) for w in wlist)


def test_device_percentile_normalisation_is_numpy_exact(sd):
    """SURVEY 8 f3: csbdeep.utils.normalize(x, pmin, pmax) on the device -- mi / ma are np.percentile's bits (exact order
    statistics by radix select + numpy's own interpolation), the normalised array equals the numpy restatement bit for bit"""
    import torch
    from stardist_b200 import prep
    from stardist_b200.utils import normalize
    rng = np.random.default_rng(7)
    for dtype, shape, valid in ((np.float32, (301, 257), (301, 257)), (np.uint16, (128, 200), (128, 200)), (np.float32, (40, 64, 72), (37, 64, 70)),
                                (np.uint8, (77, 91), (77, 91))):
        if np.dtype(dtype).kind == 'f':
            x = rng.normal(0.3, 1.0, shape).astype(dtype); x[rng.random(shape) < 0.01] *= 50
        else:
            x = rng.integers(0, np.iinfo(dtype).max, shape).astype(dtype)
        xv = x[tuple(slice(0, v) for v in valid)]
        t = torch.from_numpy(x.astype(np.float32)).cuda()
        for ps in ((1, 99.8), (2, 99.8), (0, 100), (50, 50.5), (3, 99.9)):
            got = prep.percentiles_device(t, valid, ps, x.dtype)
            want = [np.percentile(xv, p) for p in ps]
            for g, w in zip(got, want):
                assert np.asarray(g).dtype == np.asarray(w).dtype and np.array_equal(g, w), (dtype, ps, g, w)
        if valid == shape:
            t2 = t.clone()
            prep.normalize_device(t2, shape, 1, 99.8, x.dtype)
            assert np.array_equal(t2.cpu().numpy(), normalize(x, 1, 99.8))
            t3 = t.clone()
            prep.normalize_device(t3, shape, 2, 99, x.dtype, clip=True, eps=1e-3)
            assert np.array_equal(t3.cpu().numpy(), normalize(x, 2, 99, clip=True, eps=1e-3))


def test_device_zoom_and_reflect_pad_vs_scipy_numpy(sd):
    """ndi.zoom(img, scale, order=1) (stardist/models/base.py:735) and np.pad(mode='reflect') at the end on the device"""
    import torch
    from scipy import ndimage as ndi
    from stardist_b200 import prep
    rng = np.random.default_rng(8)
    worst = 0.0
    for it in range(40):
        nd = 2 if it % 3 else 3
        shp = tuple(int(v) for v in rng.integers(5, 90 if nd == 2 else 30, nd))
        sc = tuple(float(v) for v in rng.choice([0.5, 0.75, 1.3, 2.0, 1.7, 0.33, 3.0, 1.0, 0.9], nd))
        x = rng.uniform(0, 1, shp).astype(np.float32)
        want = ndi.zoom(x, sc, order=1)
        got = prep.zoom_device(torch.from_numpy(x).cuda(), sc).cpu().numpy()
        assert got.shape == want.shape
        worst = max(worst, float(np.abs(got - want).max()))
        pads = [int(v) for v in rng.integers(0, min(shp) - 1, nd)]
        out_sp = [s + p for s, p in zip(shp, pads)]
        xc = np.stack([x, 2 * x], -1)
        wantp = np.pad(xc, [(0, p) for p in pads] + [(0, 0)], mode='reflect')
        gotp = prep.pad_reflect_end_device(torch.from_numpy(xc).cuda(), out_sp).cpu().numpy()
        assert np.array_equal(gotp, wantp)
    assert worst <= 1e-6, worst       # float tolerance (bit-equal in 299 of 300 cases of the numpy emulation of this rule)
    # integer images: scipy returns the input's dtype, i.e. rounds (half up) and clips -- restated on the device
    for dt in (np.uint16, np.uint8, np.int16):
        xi = rng.integers(np.iinfo(dt).min, np.iinfo(dt).max, (57, 83)).astype(dt)
        for sc in ((1.5, 1.5), (0.75, 2.0)):
            want = ndi.zoom(xi, sc, order=1)
            got = prep.zoom_device(torch.from_numpy(xi.astype(np.float32)).cuda(), sc, dt).cpu().numpy()
            assert got.shape == want.shape and np.array_equal(got, want.astype(np.float32)), (dt, sc, int((got != want).sum()))


@pytest.mark.parametrize("dtype", [np.uint16, np.float32])
def test_predict_instances_with_device_normaliser_and_scale_equals_host_path(sd, dtype, monkeypatch):
    """normalizer=PercentileNormalizer / scale= handled in HBM give the labels of the host (numpy / scipy) preparation"""
    import bench_data
    from stardist_b200.models.base import PercentileNormalizer
    cfg = sd.Config2D(n_rays=32)
    model = sd.StarDist2D(cfg, name=None, basedir=None, weights=bench_data.bench_weights_2d(cfg))
    img, _ = bench_data.synthetic_image((250, 333), seed=4)
    raw = (np.clip(img, 0, 1.5) * 20000 + 300).astype(dtype)
    for kw in (dict(), dict(scale=1.5), dict(scale=(0.75, 1.25))):
        monkeypatch.setenv("STARDIST_B200_PREP", "host")
        lh, rh = model.predict_instances(raw, normalizer=PercentileNormalizer(1, 99.8), **kw)
        monkeypatch.setenv("STARDIST_B200_PREP", "device")
        ld, rd = model.predict_instances(raw, normalizer=PercentileNormalizer(1, 99.8), **kw)
        assert len(rh['prob']) > 20
        if 'scale' in kw:       # zoom: float tolerance 1e-6 on the input -> allow a handful of borderline candidates
            assert abs(len(rd['prob']) - len(rh['prob'])) <= 2 and np.mean((ld > 0) != (lh > 0)) < 2e-3
        else:
            assert np.array_equal(ld, lh) and np.array_equal(rd['points'], rh['points']) and np.array_equal(rd['coord'], rh['coord'])


def test_polygon_order_property_through_product(sd):
    """the reference's test_polygon_order_2D (tests/test_big.py:202-214): with nms_thresh=0 no survivor is occluded, so the
    pixels labelled i are exactly polygon i rendered on its own.  (The single-polygon raster rule itself restates
    skimage.draw.polygon, which is not installable here: 2-D label painting stays 'parity unpinned', see README / DESIGN.)"""
    import bench_data
    from stardist_b200.geometry.geom2d import polygons_to_label_coord
    cfg = sd.Config2D(n_rays=32)
    model = sd.StarDist2D(cfg, name=None, basedir=None, weights=bench_data.bench_weights_2d(cfg))
    img, _ = bench_data.synthetic_image((384, 416), seed=9)
    labels, polys = model.predict_instances(img, nms_thresh=0)
    assert len(polys['coord']) > 30
    stolen = 0
    for i, coord in enumerate(polys['coord'], start=1):
        alone = polygons_to_label_coord(coord[None], shape=labels.shape) > 0
        mine = labels == i
        assert not (mine & ~alone).any(), i                 # label i never leaves polygon i
        # nms_thresh = 0 suppresses polygons whose integer-snapped outlines overlap (Clipper area > 0); two survivors may still
        # touch in single boundary pixels of the float rendering -- those go to the polygon painted last
        lost = alone & ~mine
        assert (labels[lost] > 0).all(), i
        stolen += int(lost.sum())
    assert stolen <= 1e-3 * (labels > 0).sum()


@pytest.mark.parametrize("n,R,radius,noise,thr,seed", [(20000, 32, 8, .2, .4, 0), (3000, 32, 1.5, .9, .3, 2), (40000, 32, 10, .1, .4, 5),
                                                       (6000, 16, 9, .3, .2, 6)])
def test_nms2d_tail_kernel_equals_host_rounds_and_reference(sd, n, R, radius, noise, thr, seed):
    """frontier rounds >= 1 inside one cooperative kernel (k_tail, on-device termination) vs the host-driven rounds vs the
    reference C++: identical keep masks; the small initial pair list forces the overflow / hand-back path as well"""
    from stardist_b200 import _lib
    from stardist_b200.lib.stardist2d import c_non_max_suppression_inds
    lib = _lib.load()
    rng = np.random.default_rng(seed)
    pts = rng.integers(0, 400, (n, 2)).astype(np.float32)
    dist = np.maximum(np.float32(1e-3), (radius * (1 + noise * rng.uniform(-1, 1, (n, R)))).astype(np.float32))
    want = ref_ext.stardist2d().c_non_max_suppression_inds(dist, pts, 1, 1, 0, np.float32(thr)) if ref_ext.available() else None
    try:
        lib.sdb_nms2d_set_tail(0)
        host = c_non_max_suppression_inds(dist, pts, 1, 1, 0, np.float32(thr))
        lib.sdb_nms2d_set_tail(1)
        tail = c_non_max_suppression_inds(dist, pts, 1, 1, 0, np.float32(thr))
        lib.sdb_nms2d_set_tail(2)               # 4 blocks per SM variant
        tail4 = c_non_max_suppression_inds(dist, pts, 1, 1, 0, np.float32(thr))
        lib.sdb_nms2d_set_filter(0); lib.sdb_nms2d_set_tail(1)      # no pre-filter: every pair through the exact sweep, nothing deferred
        tail_nf = c_non_max_suppression_inds(dist, pts, 1, 1, 0, np.float32(thr)) if n <= 20000 else tail
    finally:
        lib.sdb_nms2d_set_tail(1); lib.sdb_nms2d_set_filter(1)
    assert np.array_equal(tail, host) and np.array_equal(tail4, host) and np.array_equal(tail_nf, host)
    if want is not None:
        assert np.array_equal(tail, want)
