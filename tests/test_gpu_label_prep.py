"""edt_prob and fill_label_holes on the device: every golden case of the reference's own functions (tests/golden/label_prep.npz)
through the numpy and the device API, seeded random maps and benchmark-size maps against the restatement of the
definitions (tests/labelprep_emu.py), the C entry points, invariants at 128x512x512, and argument errors that launch nothing.

Bit for bit throughout, except where the anisotropy is not dyadic: there two features whose float64 distances tie to the
last bit may round differently, so at most 1 float32 ulp is allowed and the number of such pixels is reported."""
import os, sys, json, warnings, ctypes
import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
sys.path.insert(0, os.path.dirname(HERE))
import labelprep_emu as E
import label_prep_cases as C
from star_dist_cases import sha

pytestmark = pytest.mark.gpu


def _golden():
    g = np.load(os.path.join(HERE, "golden", "label_prep.npz"))
    return g, json.loads(g["meta"].tobytes().decode())


G, META = _golden()


def _same(key, r, exp, non_dyadic):
    assert r.shape == exp.shape and r.dtype == exp.dtype, key
    if non_dyadic and r.dtype == np.float32:
        ulp = np.abs(r.view(np.int32).astype(np.int64) - exp.view(np.int32).astype(np.int64))
        n = int(np.count_nonzero(ulp))
        if n:
            print("%s: %d pixels differ by %d ulp at most" % (key, n, ulp.max()))
        assert ulp.max() <= 1, key
    else:
        assert np.array_equal(r, exp), key


def _check_golden(key, r):
    if key in META["hashes"]:
        assert [sha(r), list(r.shape), str(r.dtype)] == META["hashes"][key], key
    else:
        _same(key, r, G[key], key.rsplit("/", 1)[1] in C.NON_DYADIC)


def _to_cuda(m):
    import torch
    return torch.from_numpy(np.ascontiguousarray(m)).cuda()


@pytest.mark.parametrize("key", sorted(C.edt_cases()))
def test_edt_prob_golden(key):
    import stardist_b200 as sd
    from stardist_b200.labelprep import edt_prob_device
    m, a = C.edt_cases()[key]
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        r = sd.edt_prob(m, anisotropy=a)
    assert any("constant label image" in str(x.message) for x in w) == (key in META["warned"])
    _check_golden(key, r)
    if True:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            d = edt_prob_device(_to_cuda(m), a)
        assert d.is_cuda and d.dtype.is_floating_point
        _check_golden(key, d.cpu().numpy())


@pytest.mark.parametrize("key", sorted(C.fill_cases()))
def test_fill_label_holes_golden(key):
    import stardist_b200 as sd
    from scipy.ndimage import generate_binary_structure
    from stardist_b200.labelprep import fill_label_holes_device
    m, c = C.fill_cases()[key]
    st = generate_binary_structure(m.ndim, c)
    r = sd.fill_label_holes(m, structure=st)
    assert r.dtype == m.dtype and r.shape == m.shape
    _check_golden(key, r)
    if c == 1:
        _check_golden(key, sd.fill_label_holes(m))
    d = fill_label_holes_device(_to_cuda(m), structure=st)
    assert d.is_cuda and str(d.dtype).endswith(str(m.dtype))
    _check_golden(key, d.cpu().numpy())


RANDOM = [((40, 37), None), ((33, 41), 1.0), ((30, 30), (2, 1)), ((31, 29), (1.7, 0.9)), ((9, 14, 15), None),
          ((10, 12, 13), (2, 1, 1)), ((9, 11, 12), (1.73, 1, 1)), ((1, 64), None), ((48, 1), (3, 1))]


@pytest.mark.parametrize("case", range(len(RANDOM)))
@pytest.mark.parametrize("seed", range(4))
def test_random_maps_against_restatement(case, seed):
    import stardist_b200 as sd
    shape, aniso = RANDOM[case]
    rng = np.random.default_rng(1000 + 10 * case + seed)
    lbl = E.random_labels(rng, shape, density=0.02 + 0.03 * (seed % 2), negative=seed == 3)
    nd = aniso is not None and np.any(np.log2(np.atleast_1d(aniso)) % 1 != 0)
    _same("edt", sd.edt_prob(lbl, anisotropy=aniso), E.edt_prob_brute(lbl, aniso), nd)
    from scipy.ndimage import generate_binary_structure
    for c in range(1, lbl.ndim + 1):
        assert np.array_equal(sd.fill_label_holes(lbl, structure=generate_binary_structure(lbl.ndim, c)), E.fill_label_holes_def(lbl, c))


def test_largest_supported_label():
    import stardist_b200 as sd
    m = C.hole_larger().astype(np.int64)
    m[m == 90] = 2 ** 30 - 1
    assert np.array_equal(sd.fill_label_holes(m), E.fill_label_holes_def(m))
    assert np.array_equal(sd.edt_prob(m), E.edt_prob_boxes(m))


def test_c_entry_points():
    from stardist_b200 import _lib as L
    lib = L.require_cuda()
    for key in ("edt2/hole_smaller/none", "edt2/int8_negative/2,1", "edt3/shell/none", "edt2/constant/none"):
        m, a = C.edt_cases()[key]
        src = np.ascontiguousarray(m, np.int32)
        out = np.empty(m.shape, np.float32)
        s = None if a is None else np.ascontiguousarray(np.broadcast_to(np.asarray(a, np.float64), (m.ndim,)))
        lib._LIB_edt_prob(L.ptr(src), m.ndim, L.iarr(m.shape), L.ptr(s), L.ptr(out))
        assert lib.sdb_last_error() == b""
        _check_golden(key, out)
    for key in ("fill2/hole_larger/2", "fill3/shell/1", "fill2/int8_negative/1", "fill2/big_labels/1"):
        m, c = C.fill_cases()[key]
        src = np.ascontiguousarray(m, np.int32)
        out = np.empty(m.shape, np.int32)
        lib._LIB_fill_label_holes(L.ptr(src), m.ndim, L.iarr(m.shape), c, L.ptr(out))
        assert lib.sdb_last_error() == b""
        _check_golden(key, out.astype(m.dtype))
    bad = np.full((4, 5), 7, np.int32)
    lib._LIB_fill_label_holes(L.ptr(src), 4, L.iarr((2, 2, 2, 2)), 1, L.ptr(bad))
    assert lib.sdb_last_error() != b""
    big = np.full((4, 5), 2 ** 31 - 1, np.int32)
    lib._LIB_fill_label_holes(L.ptr(big), 2, L.iarr(big.shape), 1, L.ptr(bad))
    assert lib.sdb_last_error() != b"" and not bad.any()


def test_benchmark_ground_truth_2d():
    import bench_data
    import stardist_b200 as sd
    lbl = bench_data.ellipse_labels((1024, 1024), seed=0)
    assert np.array_equal(sd.edt_prob(lbl), E.edt_prob_boxes(lbl))
    assert np.array_equal(sd.fill_label_holes(lbl), E.fill_label_holes_def(lbl))


def test_ellipsoid_volume_3d():
    import bench_data
    import stardist_b200 as sd
    vol = bench_data.ellipsoid_labels((64, 256, 256), seed=0)
    assert np.array_equal(sd.edt_prob(vol), E.edt_prob_boxes(vol))
    assert np.array_equal(sd.edt_prob(vol, anisotropy=(2, 1, 1)), E.edt_prob_boxes(vol, (2, 1, 1)))
    assert np.array_equal(sd.fill_label_holes(vol), E.fill_label_holes_def(vol))


def test_invariants_128x512x512():
    import torch
    import bench_data
    from stardist_b200.labelprep import edt_prob_device, fill_label_holes_device
    vol = bench_data.ellipsoid_labels((128, 512, 512), seed=0)
    d = _to_cuda(vol)
    p = edt_prob_device(d)
    f = fill_label_holes_device(d)
    obj = d > 0
    n = int(d.max()) + 1
    pmax = torch.zeros(n, dtype=torch.float32, device=d.device).scatter_reduce(0, d[obj].long(), p[obj], "amax")
    present = torch.bincount(d[obj].long(), minlength=n) > 0
    expect = np.float32(np.sqrt(1.0) / (np.sqrt(1.0) + 1e-10))   # any object's maximum: sqrt(m) / (sqrt(m) + 1e-10) rounds to 1
    assert torch.all(pmax[present] == float(expect)).item()
    assert torch.all(p[~obj] == 0).item() and torch.all(p[obj] > 0).item()
    assert torch.all(f[obj] >= d[obj]).item() and torch.all((f > 0) | ~obj).item()
    assert torch.all((f == d) | (f > 0)).item()


def test_argument_errors_launch_nothing():
    import torch
    import stardist_b200 as sd
    from stardist_b200 import _lib as L
    from stardist_b200.labelprep import edt_prob_device, fill_label_holes_device
    m = C.hole_smaller()
    d = _to_cuda(m)
    L.launch_count(reset=True)
    bad_calls = [lambda: sd.edt_prob(m.astype(np.float64)), lambda: sd.edt_prob(m[None, None]), lambda: sd.edt_prob(m, anisotropy=(1, 2, 3)),
                 lambda: sd.fill_label_holes(m.astype(np.float32)), lambda: sd.fill_label_holes(m, structure=np.ones((5, 5))),
                 lambda: sd.fill_label_holes(m, origin=(1, 0)), lambda: sd.fill_label_holes(m, output=np.zeros(m.shape, bool)),
                 lambda: sd.edt_prob(np.full((4, 4), 2 ** 30, np.int64)), lambda: edt_prob_device(d.float()),
                 lambda: edt_prob_device(d[None, None]), lambda: edt_prob_device(d, anisotropy=(0, 1)),
                 lambda: fill_label_holes_device(d, structure=np.ones((3, 3, 3))), lambda: fill_label_holes_device(m),
                 lambda: edt_prob_device(torch.full((3, 3), 2 ** 30, dtype=torch.int64, device="cuda"))]
    for call in bad_calls:
        with pytest.raises((ValueError, NotImplementedError)):
            call()
    assert L.launch_count() == 0
