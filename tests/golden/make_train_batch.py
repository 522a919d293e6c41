"""tests/golden/train_batch.npz: the reference's own StarDistData2D / StarDistData3D (stardist/models/model2d.py:29-120,
model3d.py:30-127) on the cases of train_batch_cases.py, run from /root/reference through tests/golden/_refpkg.py.

csbdeep is not installed: its RollingSequence and choice come from stardist_b200.models.data (the product's restatement,
borrowed like _raise).  star_dist is the reference's compiled extension from oracle/_ref; edt_prob is its scipy variant
(the `edt` package is not installed; asserted).  sample_patches is wrapped to record the position drawn for every item.

Stored (meta JSON): per case and batch the image indices, positions, the output shapes / dtypes / sha256, and how many
constant-image warnings were raised; arrays for the cases of train_batch_cases.ulp_cases().
Run in the build container: python tests/golden/make_train_batch.py"""
import os, sys, json, warnings, importlib
import numpy as np
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import train_batch_cases as C


def reference_generators():
    import _refpkg
    _refpkg.load_models()
    from stardist_b200.models.data import RollingSequence, choice
    sys.modules["csbdeep.internals.train"].RollingSequence = RollingSequence
    sys.modules["csbdeep.utils"].choice = choice
    for m in ("stardist.models.model2d", "stardist.models.model3d", "stardist.models.base", "stardist.sample_patches"):
        sys.modules.pop(m, None)
    ut = importlib.import_module("stardist.utils")
    assert ut._edt_available is False, "the reference would use the edt package; the fixture is for its scipy variant"
    sp = importlib.import_module("stardist.sample_patches")
    m2, m3 = importlib.import_module("stardist.models.model2d"), importlib.import_module("stardist.models.model3d")
    rays = importlib.import_module("stardist.rays3d").Rays_GoldenSpiral
    return m2, m3, sp, rays


def main():
    m2, m3, sp, Rays = reference_generators()
    positions = []
    orig_sample, orig_choice = m2.sample_patches, sp.choice

    def recording_sample_patches(datas, patch_size, n_samples, valid_inds=None, verbose=False):
        drawn = []
        sp.choice = lambda *a, **k: drawn.append(orig_choice(*a, **k)) or drawn[-1]
        try:
            res = orig_sample(datas, patch_size, n_samples, valid_inds=valid_inds, verbose=verbose)
        finally:
            sp.choice = orig_choice
        positions.append([int(v[drawn[0][0]]) for v in valid_inds])
        return res
    m2.sample_patches = m3.sample_patches = recording_sample_patches

    meta, arrays = {}, {}
    ulp = C.ulp_cases()
    for name, (dim, X, Y, kw, seed, batches) in C.cases().items():
        np.random.seed(seed)
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            gen = (m2.StarDistData2D if dim == 2 else m3.StarDistData3D)(X, Y, **C.make_kwargs(kw, Rays))
        entry = {"init_warnings": sorted({str(x.message) for x in w}), "batches": []}
        for i in batches:
            positions.clear()
            idx = gen.batch(i)          # the index map is cached: __getitem__ sees the same indices
            with warnings.catch_warnings(record=True) as w:
                warnings.simplefilter("always")
                (x,), outs = gen[i]
            b = {"index": [int(v) for v in idx], "positions": list(positions), "n_constant": sum("constant label image" in str(m.message) for m in w),
                 "outputs": [[list(a.shape), str(a.dtype), C.sha(a)] for a in (x,) + tuple(outs)]}
            if name in ulp:
                arrays["%s/%d/prob" % (name, i)] = outs[0].copy()                  # the 3-D generator reuses its buffers
                arrays["%s/%d/dist_mask" % (name, i)] = outs[1][..., -1].copy()
            entry["batches"].append(b)
        meta[name] = entry
    np.savez_compressed(os.path.join(HERE, "train_batch.npz"), meta=np.frombuffer(json.dumps(meta, sort_keys=True).encode(), np.uint8),
                        **arrays)
    print("wrote train_batch.npz: %d cases, %d arrays" % (len(meta), len(arrays)))


if __name__ == "__main__":
    main()
