"""edt_prob and fill_label_holes without a GPU: the numpy restatement of their definitions (tests/labelprep_emu.py) equals
the reference's own functions on seeded random maps, bit for bit, and reproduces the golden fixture; the argument checks
raise before anything reaches the device; the product refuses to run without CUDA."""
import os, sys, json, warnings
import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
import labelprep_emu as E
import label_prep_cases as C
from oracle import ref_ext

needs_ref = pytest.mark.skipif(not (ref_ext.available() and os.path.isdir("/root/reference/stardist")),
                               reason="the reference package or oracle/_ref is not available")

RANDOM = [((40, 37), None), ((33, 41), 1.0), ((30, 30), (2, 1)), ((31, 29), (1.7, 0.9)), ((9, 14, 15), None),
          ((10, 12, 13), (2, 1, 1)), ((9, 11, 12), (1.73, 1, 1))]


@pytest.fixture(scope="module")
def ref():
    import make_label_prep as M
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return M.reference_utils()


@needs_ref
@pytest.mark.parametrize("case", range(len(RANDOM)))
@pytest.mark.parametrize("seed", range(3))
def test_restatement_equals_reference_on_random_maps(ref, case, seed):
    shape, aniso = RANDOM[case]
    rng = np.random.default_rng(100 * case + seed)
    lbl = E.random_labels(rng, shape, negative=seed == 2)
    p_ref = ref.edt_prob(lbl, anisotropy=aniso)
    assert np.array_equal(E.edt_prob_brute(lbl, aniso), p_ref)
    assert np.array_equal(E.edt_prob_boxes(lbl, aniso), p_ref)
    from scipy.ndimage import generate_binary_structure
    for c in range(1, lbl.ndim + 1):
        f_ref = ref.fill_label_holes(lbl, structure=generate_binary_structure(lbl.ndim, c))
        assert np.array_equal(E.fill_label_holes_def(lbl, c), f_ref), c


def _golden():
    g = np.load(os.path.join(HERE, "golden", "label_prep.npz"))
    return g, json.loads(g["meta"].tobytes().decode())


def test_restatement_reproduces_fixture():
    """every stored case, from the restatement alone (no reference needed)"""
    from star_dist_cases import sha
    g, meta = _golden()
    cases = [(k, lambda m=m, a=a: E.edt_prob_boxes(m, a)) for k, (m, a) in C.edt_cases().items()]
    cases += [(k, lambda m=m, c=c: E.fill_label_holes_def(m, c)) for k, (m, c) in C.fill_cases().items()]
    assert len(cases) == len(meta["hashes"]) + len(g.files) - 1
    for key, fn in cases:
        r = fn()
        if key in meta["hashes"]:
            assert [sha(r), list(r.shape), str(r.dtype)] == meta["hashes"][key], key
        else:
            assert r.dtype == g[key].dtype and np.array_equal(r, g[key]), key
    assert meta["warned"] == sorted(k for k in C.edt_cases() if "/constant/" in k)


def test_brute_force_matches_boxes_on_fixture_edge_maps():
    for name, m in C.maps_2d().items():
        if m.size <= 1500:
            for a in C.ANISO_2D.values():
                assert np.array_equal(E.edt_prob_brute(m, a), E.edt_prob_boxes(m, a)), (name, a)


def test_argument_errors_without_gpu():
    from stardist_b200 import edt_prob, fill_label_holes
    m = C.hole_smaller()
    for bad in (m.astype(np.float32), m.astype(bool), m[0], m[None, None], list(m)):
        with pytest.raises(ValueError):
            edt_prob(bad)
        with pytest.raises(ValueError):
            fill_label_holes(bad)
    big = m.astype(np.int64); big[0, 0] = 2 ** 30
    with pytest.raises(ValueError):
        edt_prob(big)
    with pytest.raises(ValueError):
        fill_label_holes(big.astype(np.uint64))
    for a in ((1, 2, 3), (1,), (0, 1), (-1, 1), np.inf):
        with pytest.raises(ValueError):
            edt_prob(m, anisotropy=a)
    with pytest.raises(ValueError):
        edt_prob(np.zeros((0, 4), np.int32))
    with pytest.raises(NotImplementedError):
        fill_label_holes(m, structure=np.ones((5, 5)))
    with pytest.raises(NotImplementedError):
        fill_label_holes(m, structure=np.array([[0, 1, 0], [0, 1, 0], [0, 1, 0]]))
    with pytest.raises(ValueError):
        fill_label_holes(m, structure=np.ones((3, 3, 3)))
    with pytest.raises(NotImplementedError):
        fill_label_holes(m, origin=1)
    with pytest.raises(NotImplementedError):
        fill_label_holes(m, output=np.zeros(m.shape, bool))
    with pytest.raises(TypeError):
        fill_label_holes(m, foo=1)
    assert fill_label_holes(np.zeros((0, 3), np.uint16)).dtype == np.uint16


def test_product_raises_without_cuda():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is visible")
    import stardist_b200 as sd
    m = C.hole_smaller()
    for call in (lambda: sd.edt_prob(m), lambda: sd.fill_label_holes(m)):
        with pytest.raises(sd._lib.StarDistB200Error):
            call()
