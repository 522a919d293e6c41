"""tests/golden/label_prep.npz: the reference's own edt_prob (stardist/utils.py:71-125) and fill_label_holes (utils.py:137-153)
on the maps of label_prep_cases.py, run from /root/reference through tests/golden/_refpkg.py.  The `edt` package is not a
reference dependency and not installed, so edt_prob is the scipy variant; this is asserted.

Stored: results as arrays where label_prep_cases.stored_as_array says so, otherwise sha256 (key -> [sha, shape, dtype]) as
JSON; the warning edt_prob gave for each case (the constant-image warning).
Run in the build container: python tests/golden/make_label_prep.py"""
import os, sys, json, warnings
import numpy as np
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import label_prep_cases as C
from star_dist_cases import sha


def reference_utils():
    import _refpkg, importlib
    _refpkg.setup()
    ut = importlib.import_module("stardist.utils")
    assert ut._edt_available is False, "the reference would use the edt package; the fixture is for its scipy variant"
    return ut


def main():
    ut = reference_utils()
    hashes, arrays, warned = {}, {}, []
    results = []
    for key, (m, a) in C.edt_cases().items():
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            r = ut.edt_prob(m, anisotropy=a)
        if any("constant label image" in str(x.message) for x in w):
            warned.append(key)
        results.append((key, r))
    for key, (m, c) in C.fill_cases().items():
        from scipy.ndimage import generate_binary_structure
        r = ut.fill_label_holes(m, structure=generate_binary_structure(m.ndim, c))
        assert r.dtype == m.dtype
        results.append((key, r))
    for key, r in results:
        if C.stored_as_array(key, r):
            arrays[key] = r
        else:
            hashes[key] = [sha(r), list(r.shape), str(r.dtype)]
    meta = {"hashes": hashes, "warned": sorted(warned)}
    np.savez_compressed(os.path.join(HERE, "label_prep.npz"), meta=np.frombuffer(json.dumps(meta, sort_keys=True).encode(), np.uint8),
                        **arrays)
    print("wrote label_prep.npz: %d arrays, %d hashes, warned: %s" % (len(arrays), len(hashes), warned))


if __name__ == "__main__":
    main()
