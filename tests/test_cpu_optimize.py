"""Evaluation API and threshold-engine host half, without a GPU.

* matching (tuple thresholds, report_matches), matching_dataset (by_image both ways) and label_overlap equal the reference's
  own results frozen in tests/golden/matching.npz (make_matching.py), value and scalar type.
* ImageTables.probe_overlap (stardist_b200/optimize.py) equals the overlap matrix `matching` builds from the label image the
  probe stands for, where(L_floor <= k(t), L_floor, 0), on seeded label maps and survivor scores."""
import os, sys, json
import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))


@pytest.fixture(scope="module")
def golden():
    z = np.load(os.path.join(ROOT, "tests", "golden", "matching.npz"))
    return json.loads(bytes(z["results"]).decode()), z


def _encode(t):
    import make_matching
    return json.loads(json.dumps(make_matching.encode(t)))


@pytest.mark.parametrize("crit", ["iou", "iot", "iop"])
def test_matching_equals_reference(golden, crit):
    import make_matching
    from stardist_b200.matching import matching
    res, _ = golden
    for i, (a, b) in enumerate(make_matching.pairs()):
        got = matching(a, b, thresh=make_matching.THRESHS, criterion=crit, report_matches=True)
        assert isinstance(got, tuple) and len(got) == len(make_matching.THRESHS)
        assert [_encode(m) for m in got] == res["matching/%s/%d" % (crit, i)]
        assert _encode(matching(a, b, thresh=0.5, criterion=crit, report_matches=True)) == res["matching_scalar/%s/%d" % (crit, i)]


@pytest.mark.parametrize("crit", ["iou", "iot", "iop"])
@pytest.mark.parametrize("by_image", [False, True])
def test_matching_dataset_equals_reference(golden, crit, by_image):
    import make_matching
    from stardist_b200.matching import matching_dataset, matching_dataset_lazy
    res, _ = golden
    data = make_matching.pairs()
    want = res["dataset/%s/%d" % (crit, by_image)]
    got = matching_dataset([a for a, b in data], [b for a, b in data], thresh=make_matching.THRESHS, criterion=crit,
                           by_image=by_image, show_progress=False, parallel=True)
    assert [_encode(m) for m in got] == want
    lazy = matching_dataset_lazy(iter(data), thresh=make_matching.THRESHS[2], criterion=crit, by_image=by_image)
    assert _encode(lazy) == want[2]


def test_label_overlap_equals_reference(golden):
    import make_matching
    from stardist_b200.matching import label_overlap, relabel_sequential
    _, z = golden
    a, b = make_matching.pairs()[0]
    ov = label_overlap(relabel_sequential(a)[0], relabel_sequential(b)[0])
    assert str(ov.dtype) == bytes(z["overlap_dtype"]).decode() and np.array_equal(ov, z["overlap"])
    with pytest.raises(ValueError):
        label_overlap(a, b + 1000)                         # not sequential
    with pytest.raises(ValueError):
        label_overlap(a, b[:-1])


def test_matching_rejects_bad_input():
    from stardist_b200.matching import matching
    a = np.zeros((8, 8), np.int32)
    with pytest.raises(ValueError):
        matching(a, a - 1)
    with pytest.raises(ValueError):
        matching(a, a, criterion='dice')


def _random_floor_map(rng, shape, n_surv):
    """label map with ids 1..n_surv painted as overlapping discs (some hidden completely), 0 = background"""
    lab = np.zeros(shape, np.int32)
    yy, xx = np.ogrid[:shape[0], :shape[1]]
    for i in rng.permutation(n_surv) + 1:
        c = rng.integers(0, shape); r = rng.integers(2, 8)
        lab[(yy - c[0]) ** 2 + (xx - c[1]) ** 2 <= r * r] = i
    return lab


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_probe_overlap_equals_matching_matrix(seed):
    """the probe matrix is the matrix `matching` builds from where(L_floor <= k(t), L_floor, 0), for every probe, including
    survivors that painted nothing, a ground truth with non-sequential ids and thresholds on both sides of every score"""
    from stardist_b200.optimize import ImageTables, dataset_matching
    from stardist_b200.matching import _overlap_matrix, relabel_sequential, matching_dataset
    rng = np.random.default_rng(seed)
    shape = (64, 80)
    n_surv = 40
    lab = _random_floor_map(rng, shape, n_surv)
    gt = _random_floor_map(rng, shape, 30) * 7                   # ids 7, 14, ...
    surv_prob = np.sort(rng.uniform(0.3, 0.9, n_surv).astype(np.float32))[::-1]
    gt_seq, _, _ = relabel_sequential(gt)
    n_true = int(gt_seq.max())
    flat = gt_seq.ravel().astype(np.int64) * (n_surv + 1) + lab.ravel()
    keys, counts = np.unique(flat, return_counts=True)
    pairs = np.stack([keys // (n_surv + 1), keys % (n_surv + 1)], 1)
    tab = ImageTables.from_pairs(n_true, surv_prob, pairs, counts)
    probes = [np.float64(0.29), np.float64(0.95)] + [np.float64(p) for p in surv_prob[::3]] + list(rng.uniform(0.3, 0.9, 8))
    for t in probes:
        k = int(np.count_nonzero(surv_prob.astype(np.float64) > t))
        lab_t = np.where(lab <= k, lab, 0)
        want = _overlap_matrix(gt_seq, relabel_sequential(lab_t)[0])
        got = tab.probe_overlap(t)
        assert got.dtype == want.dtype and np.array_equal(got, want), t
        st = dataset_matching([tab, tab], t, (0.3, 0.5, 0.7))
        ref = matching_dataset([gt, gt], [lab_t, lab_t], thresh=(0.3, 0.5, 0.7), show_progress=False)
        assert st == ref


def test_float32_floor_selects_a_superset():
    from stardist_b200.optimize import float32_at_or_below
    rng = np.random.default_rng(5)
    for t in list(rng.uniform(0, 1, 200)) + [0.5, np.float32(0.3), 0.549501654040]:
        f = float32_at_or_below(t)
        assert isinstance(f, np.float32) and float(f) <= float(t)
        assert float(np.nextafter(f, np.float32(np.inf))) > float(t)       # the largest such float32


def _ref_or_skip():
    from oracle import ref_ext
    if not ref_ext.available():
        pytest.skip("oracle/_ref not built (make -C oracle ref)")
    return ref_ext


@pytest.mark.parametrize("name", ["r32_356x299", "r11_114x217"])
def test_prefix_facts_2d_against_reference(name):
    """facts 2-3 of stardist_b200/optimize.py with the reference's own NMS (oracle/_ref): the keep mask at the floor restricted to
    prob > t equals the reference NMS run on the candidates above t, and the label map painted from the survivors at t equals
    the floor map masked to ids <= k(t) (painting: the oracle restatement of polygons_to_label)"""
    import cases
    from oracle import geom2d_np
    ref = _ref_or_skip()
    d, p, s, thr = cases.nms2d_inputs(name)
    d, p, s = d[:400], p[:400], s[:400]                  # a prefix of the score order is itself a floor candidate set
    nms = lambda k: ref.stardist2d().c_non_max_suppression_inds(d[:k], p[:k], 1, 1, 0, thr)
    keep = nms(len(s))
    shape = tuple(int(v) + 8 for v in p.max(0))
    surv = np.flatnonzero(keep)
    lab = geom2d_np.polygons_to_label(d[surv], p[surv], shape, prob=s[surv])
    for t in np.quantile(s.astype(np.float64), [0.1, 0.35, 0.6, 0.85]):
        k = int(np.count_nonzero(s.astype(np.float64) > t))
        assert np.array_equal(nms(k), keep[:k]), t
        n_kept = int(np.count_nonzero(keep[:k]))
        st = surv[:n_kept]
        lab_t = geom2d_np.polygons_to_label(d[st], p[st], shape, prob=s[st])
        assert np.array_equal(lab_t, np.where(lab <= n_kept, lab, 0)), t


@pytest.mark.parametrize("name", ["r32_noise01_thr01", "r96_noise02_thr03"])
def test_prefix_facts_3d_against_reference(name):
    """facts 2-3 in 3-D with the reference's own NMS and polyhedron_to_label (oracle/_ref): survivors painted first cover wins
    in descending score order with ids = survivor index + 1"""
    import cases
    ref = _ref_or_skip()
    d, p, s, rays, thr, shape = cases.nms3d_inputs(name)
    d, p, s = d[:300], p[:300], s[:300]
    v, f = np.ascontiguousarray(rays.vertices, np.float32), np.ascontiguousarray(rays.faces, np.int32)
    nms = lambda k: ref.stardist3d().c_non_max_suppression_inds(d[:k], p[:k], v, f, s[:k], 1, 1, 0, thr)

    def paint(idx):
        ids = np.arange(1, len(idx) + 1, dtype=np.int32)
        return ref.stardist3d().c_polyhedron_to_label(d[idx], p[idx], v, f, ids, np.int32(0), np.int32(0), np.int32(0), np.int32(0), shape)
    keep = nms(len(s))
    surv = np.flatnonzero(keep)
    lab = paint(surv)
    for t in np.quantile(s.astype(np.float64), [0.1, 0.5, 0.9]):
        k = int(np.count_nonzero(s.astype(np.float64) > t))
        assert np.array_equal(nms(k), keep[:k]), t
        n_kept = int(np.count_nonzero(keep[:k]))
        assert np.array_equal(paint(surv[:n_kept]), np.where(lab <= n_kept, lab, 0)), t
