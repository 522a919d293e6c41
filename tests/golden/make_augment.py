"""tests/golden/augment.npz: the reference's own StarDistData2D / StarDistData3D (through make_train_batch.reference_generators())
with the augmenter of the reference's training notebooks, on the cases of augment_cases.py.  The augmenter functions are read
from the reference's examples/2D/2_training.ipynb and examples/3D/2_training.ipynb when this runs; nothing of them is stored.

Stored (meta JSON): per case and batch the image indices, positions, the sha256 of every output (X as float32, which is what
the generators return: the reference's X is float64 after the noise add) and the np.random state afterwards (sha256 of the
key, pos, has_gauss, gauss).  Run in the build container: python tests/golden/make_augment.py"""
import json, os, sys, warnings
import numpy as np
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import augment_cases as A
import train_batch_cases as T
from make_train_batch import reference_generators

REF = "/root/reference/examples"


def notebook_functions(dim):
    """the code cells of the reference's training notebook that define the augmenter, executed into a namespace"""
    nb = json.load(open(os.path.join(REF, "%dD" % dim, "2_training.ipynb")))
    ns = {"np": np}
    for c in nb["cells"]:
        src = "".join(c["source"])
        if c["cell_type"] == "code" and ("def random_fliprot" in src or "def augmenter" in src):
            exec(src, ns)
    return ns


def augmenters():
    nb2, nb3 = notebook_functions(2), notebook_functions(3)

    def aug_3d_noise(x, y):
        x, y = nb3["random_fliprot"](x, y, axis=(1, 2))
        x = nb3["random_intensity_change"](x)
        sig = 0.02 * np.random.uniform(0, 1)             # the 2-D notebook's noise
        x = x + sig * np.random.normal(0, 1, x.shape)
        return x, y
    return {"2d": nb2["augmenter"], "3d": nb3["augmenter"], "3d_noise": aug_3d_noise}


def state_record():
    name, key, pos, has_gauss, gauss = np.random.get_state()
    return [T.sha(np.asarray(key, np.uint32)), int(pos), int(has_gauss), float(gauss).hex()]


def main():
    m2, m3, sp, Rays = reference_generators()
    augs = augmenters()
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

    meta = {}
    for name, (dim, X, Y, kw, seed, batches, _, nb) in A.cases().items():
        np.random.seed(seed)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            gen = (m2.StarDistData2D if dim == 2 else m3.StarDistData3D)(X, Y, augmenter=augs[nb], **T.make_kwargs(kw, Rays))
        entry = []
        for i in batches:
            positions.clear()
            idx = gen.batch(i)
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                (x,), outs = gen[i]
            outs = (np.asarray(x, np.float32),) + tuple(outs)
            entry.append({"index": [int(v) for v in idx], "positions": list(positions), "state": state_record(),
                          "outputs": [[list(a.shape), str(a.dtype), T.sha(a)] for a in outs]})
        meta[name] = entry
    np.savez_compressed(os.path.join(HERE, "augment.npz"), meta=np.frombuffer(json.dumps(meta, sort_keys=True).encode(), np.uint8))
    print("wrote augment.npz: %d cases" % len(meta))


if __name__ == "__main__":
    main()
