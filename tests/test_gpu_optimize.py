"""optimize_thresholds on the device: the sparse label-overlap kernel and the threshold engine.

* sdb_label_overlap equals np.unique / np.bincount on random, blob, empty, single-label, non-sequential, > 100 k pair (retry)
  and 128x512x512 label maps; negative labels raise.
* utils.optimize_threshold (engine: one NMS, painting and overlap table per image and nms_thresh) gives, probe for probe, the
  value of the per-probe loop over the public _instances_from_prediction + matching_dataset, and the same optimum, on
  synthetic maps (2-D grid 1 and 2, 3-D 32 / 96 rays) and on the real maps of the shipped 2D_demo and 3D_demo models; and
  it reproduces the reference's own optimize_threshold on the synthetic cases probe for probe (tests/golden/optimize.npz).
* 2D_demo on its test image: prob_thresh ~ 0.5495 and nms_thresh == 0.5 (stardist tests/test_model2D.py:121-133).
* 3D_demo: tiled and untiled predictions optimise to the same thresholds (stardist tests/test_model3D.py:125-143).
* thresholds.json written by optimize_thresholds is read back by a model loaded from the folder."""
import os, sys, json
import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sd():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import stardist_b200
    return stardist_b200


def _overlap(a, b):
    import torch
    from stardist_b200.matching import label_overlap_device
    pa, ca = label_overlap_device(torch.from_numpy(np.ascontiguousarray(a, np.int32)).cuda(),
                                  torch.from_numpy(np.ascontiguousarray(b, np.int32)).cuda())
    return pa.cpu().numpy(), ca.cpu().numpy()


def _overlap_ref(a, b):
    key = a.ravel().astype(np.int64) << 32 | b.ravel().astype(np.int64)
    k, c = np.unique(key, return_counts=True)
    return np.stack([k >> 32, k & 0xffffffff], 1).astype(np.int32), c.astype(np.int64)


def _blobs(rng, shape, n, rmax=12):
    lab = np.zeros(shape, np.int32)
    grids = np.ogrid[tuple(slice(0, s) for s in shape)]
    for i in range(1, n + 1):
        c = rng.integers(0, shape); r = rng.integers(2, rmax)
        lab[sum((g - ci) ** 2 for g, ci in zip(grids, c)) <= r * r] = i
    return lab


OVERLAP_CASES = ["random", "blobs", "zeros", "one_label", "nonsequential", "many_pairs"]


@pytest.mark.parametrize("case", OVERLAP_CASES)
def test_label_overlap_kernel(sd, case):
    rng = np.random.default_rng(OVERLAP_CASES.index(case))
    shape = (301, 517)
    if case == "random":
        a, b = rng.integers(0, 50, shape), rng.integers(0, 70, shape)
    elif case == "blobs":
        a, b = _blobs(rng, shape, 200), _blobs(rng, shape, 150)
    elif case == "zeros":
        a = b = np.zeros(shape, np.int32)
    elif case == "one_label":
        a, b = np.full(shape, 7), np.zeros(shape, np.int32)
    elif case == "nonsequential":
        a, b = _blobs(rng, shape, 100) * 1000003, _blobs(rng, shape, 90).astype(np.int64) * 17 + (2 ** 31 - 1 - 17 * 90)
    else:                                              # > 100 k distinct pairs: the first capacity guess is too small
        a, b = rng.integers(0, 2 ** 31 - 1, shape), rng.integers(0, 3, shape)
    got = _overlap(a, b)
    want = _overlap_ref(a, b)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
    if case == "many_pairs":
        assert len(want[1]) > 100_000


def test_label_overlap_kernel_volume_and_errors(sd):
    import torch
    from stardist_b200.matching import label_overlap_device
    rng = np.random.default_rng(0)
    a = _blobs(rng, (128, 128, 128), 300, rmax=16)
    vol_a = np.tile(a, (1, 4, 4)); vol_b = np.roll(vol_a, 5, axis=2) * 3
    got = _overlap(vol_a, vol_b)
    want = _overlap_ref(vol_a, vol_b)
    assert vol_a.shape == (128, 512, 512) and np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
    x = torch.zeros((64, 64), dtype=torch.int32, device='cuda'); y = x.clone(); y[3, 4] = -2
    with pytest.raises(ValueError):
        label_overlap_device(x, y)
    with pytest.raises(ValueError):
        label_overlap_device(x, x[:32])


def _loop_value(model, Y, Yhat, t, nms_thresh, iou_threshs, measure='accuracy'):
    """the reference's fn(thr) body (stardist/utils.py:287-290) over the product's public functions"""
    from stardist_b200.matching import matching_dataset
    inst = [model._instances_from_prediction(y.shape, *pd, prob_thresh=t, nms_thresh=nms_thresh)[0] for y, pd in zip(Y, Yhat)]
    stats = matching_dataset(Y, inst, thresh=iou_threshs, show_progress=False, parallel=True)
    return np.mean([s._asdict()[measure] for s in stats])


def _run_and_compare(model, Y, Yhat, nms_threshs, iou_threshs, **kw):
    """optimize_threshold per nms_thresh, every probe checked against the per-probe loop; returns [(nms, x, value, n_probes)]"""
    from stardist_b200 import optimize as E
    from stardist_b200.utils import optimize_threshold
    out = []
    for nms in nms_threshs:
        probes = []
        orig = E.dataset_matching

        def spy(tables, t, iou, criterion='iou'):
            st = orig(tables, t, iou, criterion)
            probes.append((t, np.mean([s._asdict()['accuracy'] for s in st])))
            return st
        E.dataset_matching = spy
        try:
            x, v = optimize_threshold(Y, Yhat, model, nms, iou_threshs=iou_threshs, verbose=0, **kw)
        finally:
            E.dataset_matching = orig
        assert len(probes) >= 3
        for t, val in probes:
            want = _loop_value(model, Y, [tuple(m.cpu().numpy() if hasattr(m, 'cpu') else m for m in pd) for pd in Yhat], t, nms, iou_threshs)
            assert val == want, (nms, t, val, want)
        out.append((nms, x, v, len(probes)))
    return out


def _model(sd, ndim, grid, n_rays):
    if ndim == 2:
        return sd.StarDist2D(sd.Config2D(n_rays=n_rays, grid=grid), name=None, basedir=None)
    return sd.StarDist3D(sd.Config3D(rays=sd.Rays_GoldenSpiral(n_rays), grid=grid), name=None, basedir=None)


@pytest.mark.parametrize("name", ["2d_grid1", "2d_grid2", "3d_r32", "3d_r96"])
def test_engine_reproduces_reference_search(sd, name):
    """the engine's search == the reference's own optimize_threshold (tests/golden/optimize.npz): the same probes in the same
    order with the same scalar type, the same values, the same opt.x and -opt.fun, bit for bit"""
    import optimize_cases
    from stardist_b200 import optimize as E
    from stardist_b200.utils import optimize_threshold
    want = json.loads(bytes(np.load(os.path.join(ROOT, "tests", "golden", "optimize.npz"))["results"]).decode())[name]
    ndim, grid, n_rays, Y, Yhat = optimize_cases.inputs(name)
    model = _model(sd, ndim, grid, n_rays)
    for nms in optimize_cases.NMS_THRESHS:
        probes = []
        orig = E.dataset_matching

        def spy(tables, t, iou, criterion='iou'):
            st = orig(tables, t, iou, criterion)
            probes.append([[float(t), type(t).__name__], float(np.mean([s.accuracy for s in st]))])
            return st
        E.dataset_matching = spy
        try:
            x, v = optimize_threshold(Y, Yhat, model, nms, iou_threshs=list(optimize_cases.IOU_THRESHS), verbose=0)
        finally:
            E.dataset_matching = orig
        w = want[str(nms)]
        assert probes == w["probes"], nms
        assert (float(x), type(x).__name__, float(v)) == (w["x"], w["x_type"], w["value"])


@pytest.mark.parametrize("name", ["2d_grid1", "2d_grid2", "3d_r32", "3d_r96"])
def test_engine_equals_per_probe_loop(sd, name):
    import optimize_cases
    ndim, grid, n_rays, Y, Yhat = optimize_cases.inputs(name)
    _run_and_compare(_model(sd, ndim, grid, n_rays), Y, Yhat, optimize_cases.NMS_THRESHS, optimize_cases.IOU_THRESHS)


def _demo2d(sd):
    import demo2d
    from stardist_b200.utils import normalize
    kwargs, weights, thr, img, mask = demo2d.load()
    model = sd.StarDist2D(sd.Config2D(**kwargs), name=None, basedir=None, weights=weights)
    return model, normalize(img, 1, 99.8), mask


def test_engine_on_2d_demo_maps_and_reference_optimum(sd, capsys):
    """real network maps: every probe equals the per-probe loop; the optimum is the reference's pinned one"""
    model, x, mask = _demo2d(sd)
    Yhat = [model._predict_device(x)[:2]]                      # device maps, used in place
    res = _run_and_compare(model, [mask], Yhat, [0.3, 0.5], [0.3, 0.5], tol=1e-1)
    print("2D_demo probes:", res)
    opt = model.optimize_thresholds([x], [mask], nms_threshs=[.3, .5], iou_threshs=[.3, .5], optimize_kwargs=dict(tol=1e-1),
                                    save_to_json=False)
    assert 'Using optimized values' in capsys.readouterr().out
    assert np.isclose(opt['prob'], 0.549501654040, atol=1e-3) and opt['nms'] == 0.5, opt
    assert model.thresholds.prob == opt['prob'] and model.thresholds.nms == 0.5


def test_3d_demo_tiled_equals_untiled(sd):
    """stardist tests/test_model3D.py:125-143: on 3D_demo, tiled and untiled predictions optimise to the same thresholds;
    every probe on the real maps equals the per-probe loop"""
    import demo3d
    from stardist_b200.utils import normalize
    from stardist_b200.rays3d import rays_from_json
    rays_json, kwargs, weights, thr, img, mask = demo3d.load()
    model = sd.StarDist3D(sd.Config3D(rays=rays_from_json(rays_json), **kwargs), name=None, basedir=None, weights=weights)
    x = normalize(img, 1, 99.8)
    _run_and_compare(model, [mask], [model._predict_device(x)[:2]], [0.3, 0.5], [0.3, 0.5, 0.7])
    kw = dict(nms_threshs=[0.3, 0.5], iou_threshs=[0.3, 0.5, 0.7], optimize_kwargs=dict(tol=1e-1), save_to_json=False)
    a = model.optimize_thresholds([x], [mask], predict_kwargs=dict(n_tiles=(1, 1, 1)), **kw)
    b = model.optimize_thresholds([x], [mask], predict_kwargs=dict(n_tiles=(1, 2, 2)), **kw)
    assert a == b


def test_thresholds_json_round_trip(sd, tmp_path):
    model, x, mask = _demo2d(sd)
    folder = tmp_path / "demo"; folder.mkdir()
    cfg = model.config
    json.dump({k: v for k, v in vars(cfg).items() if isinstance(v, (int, float, str, bool, list, tuple, type(None), dict))},
              open(folder / "config.json", "w"))
    model.save_weights(folder / "weights.npz")
    m = sd.StarDist2D(None, name="demo", basedir=str(tmp_path))
    assert m._guess_n_tiles(x) == (1, 1)
    opt = m.optimize_thresholds([x[:256, :256]], [mask[:256, :256]], nms_threshs=[0.4], iou_threshs=[0.5],
                                optimize_kwargs=dict(tol=1e-1))
    saved = json.load(open(folder / "thresholds.json"))
    assert saved == {'prob': float(opt['prob']), 'nms': 0.4}
    m2 = sd.StarDist2D(None, name="demo", basedir=str(tmp_path))
    assert m2.thresholds.prob == float(opt['prob']) and m2.thresholds.nms == 0.4
