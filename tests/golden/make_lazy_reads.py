"""tests/golden/lazy_reads.npz: the reference's own StarDistData2D / StarDistData3D (stardist/models/base.py:129-217,
model2d.py:29-120, model3d.py:30-127) over the lazy, read-logging sequences of lazy_reads_cases.py, loaded as
make_train_batch.py loads them.

Stored (meta JSON): per case the reads made at construction, and per batch the image indices, the reads made for it in
order ('Y3' is Y[3]), the sha256 of numpy's global random state after it, the output shapes / dtypes / sha256 and the number
of constant-image warnings.
Run in the build container: python tests/golden/make_lazy_reads.py"""
import os, sys, json, warnings
import numpy as np
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import lazy_reads_cases as C
import train_batch_cases as T
from make_train_batch import reference_generators


def main():
    m2, m3, _, Rays = reference_generators()
    meta = {}
    for name, (dim, X, Y, kw, seed, batches, random) in C.cases().items():
        log = []
        Xl, Yl = C.lazy(X, Y, log, random)
        np.random.seed(seed)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            gen = (m2.StarDistData2D if dim == 2 else m3.StarDistData3D)(Xl, Yl, **T.make_kwargs(kw, Rays))
        entry = {"init_reads": list(log), "batches": []}
        for i in batches:
            log.clear()
            with warnings.catch_warnings(record=True) as w:
                warnings.simplefilter("always")
                (x,), outs = gen[i]
            entry["batches"].append({"index": [int(v) for v in gen.batch(i)], "reads": list(log), "state": C.state_sha(),
                                     "n_constant": sum("constant label image" in str(m.message) for m in w),
                                     "outputs": [[list(a.shape), str(a.dtype), T.sha(a)] for a in (x,) + tuple(outs)]})
        meta[name] = entry
    np.savez_compressed(os.path.join(HERE, "lazy_reads.npz"), meta=np.frombuffer(json.dumps(meta, sort_keys=True).encode(), np.uint8))
    print("wrote lazy_reads.npz: %d cases" % len(meta))


if __name__ == "__main__":
    main()
