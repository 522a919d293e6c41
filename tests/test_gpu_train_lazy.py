"""Training batches over lazy X / Y on the device: every case of tests/golden/train_batch.npz through a lazy wrapper, the
reads, random stream and outputs of tests/golden/lazy_reads.npz (random loaders included), the device memory of lazy
generators on large volumes, and train() on lazy data against train() on the same data as lists."""
import json, os, sys, warnings
import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
sys.path.insert(0, os.path.dirname(HERE))
import lazy_reads_cases as LC
import train_batch_cases as C

pytestmark = pytest.mark.gpu


def _meta(name):
    z = np.load(os.path.join(HERE, "golden", name))
    return json.loads(bytes(z["meta"]).decode())


def _make(dim, X, Y, kw, seed):
    from stardist_b200.models import StarDistData2D, StarDistData3D
    from stardist_b200.rays3d import Rays_GoldenSpiral
    np.random.seed(seed)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return (StarDistData2D if dim == 2 else StarDistData3D)(X, Y, **C.make_kwargs(kw, Rays_GoldenSpiral))


def _run(gen, batches):
    out = []
    for i in batches:
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            (x,), outs = gen[i]
        out.append(((x,) + tuple(outs), sum("constant label image" in str(m.message) for m in w), gen.last_positions.cpu().numpy().tolist()))
    return out


def _run_device(gen, batches):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return [[t.cpu().numpy() for t in ((x,) + tuple(outs))] for (x,), outs in (gen.batch_device(i) for i in batches)]


@pytest.mark.parametrize("name", sorted(C.cases()))
def test_fixture_batches_through_lazy_sequences(name):
    """byte for byte the reference's batches (the recorded hashes) and the resident path's, for gen[i] and batch_device(i)"""
    rec = _meta("train_batch.npz")[name]
    dim, X, Y, kw, seed, batches = C.cases()[name]
    lazy = _run(_make(dim, LC.Recording(X, "X", []), LC.Recording(Y, "Y", []), kw, seed), batches)
    resident = _run(_make(dim, X, Y, kw, seed), batches)
    for i, b, (arrs, n_const, pos), (want, n_want, pos_want) in zip(batches, rec["batches"], lazy, resident):
        assert pos == b["positions"] == pos_want and n_const == b["n_constant"] == n_want
        for k, (a, r, (shape, dtype, h)) in enumerate(zip(arrs, want, b["outputs"])):
            assert list(a.shape) == shape and str(a.dtype) == dtype
            assert a.tobytes() == r.tobytes(), "output %d of batch %d differs from the resident path" % (k, i)
            if not (name in C.ulp_cases() and k in (1, 2)):
                assert C.sha(a) == h, "output %d of batch %d differs from the reference" % (k, i)
    dev = _run_device(_make(dim, LC.Recording(X, "X", []), LC.Recording(Y, "Y", []), kw, seed), batches)
    for (arrs, _, _), d in zip(lazy, dev):
        assert all(a.tobytes() == b.tobytes() for a, b in zip(arrs, d))


@pytest.mark.parametrize("name", sorted(LC.cases()))
def test_lazy_reads_fixture(name):
    """the reference's reads, random stream and outputs over logging (and randomly drawing) sequences"""
    rec = _meta("lazy_reads.npz")[name]
    dim, X, Y, kw, seed, batches, random = LC.cases()[name]
    for device in (False, True):
        log = []
        gen = _make(dim, *LC.lazy(X, Y, log, random), kw, seed)
        assert log == rec["init_reads"]
        for i, b in zip(batches, rec["batches"]):
            log.clear()
            if device:
                with warnings.catch_warnings():
                    warnings.simplefilter("ignore")
                    (x,), outs = gen.batch_device(i)
                arrs = [t.cpu().numpy() for t in (x,) + tuple(outs)]
            else:
                with warnings.catch_warnings(record=True) as w:
                    warnings.simplefilter("always")
                    (x,), outs = gen[i]
                arrs = (x,) + tuple(outs)
                assert sum("constant label image" in str(m.message) for m in w) == b["n_constant"]
            assert log == b["reads"] and LC.state_sha() == b["state"], (i, device)
            assert [int(v) for v in gen.last_index] == b["index"]
            for k, (a, (shape, dtype, h)) in enumerate(zip(arrs, b["outputs"])):
                assert list(a.shape) == shape and str(a.dtype) == dtype and C.sha(a) == h, (i, k, device)


# ------------------------------------------------------------------------------------------------ device memory
class _Volumes:
    """n volumes of `shape`, made when read: a labelled block tiled over the volume (the mask), or its float32 image"""

    def __init__(self, n, shape, image):
        self.n, self.shape, self.image = n, shape, image
        tile = C._blobs((32, 64, 64), 12, 5, radius=(4, 10))
        self.tile = tile.astype(np.float32) * 0.01 if image else tile

    def __len__(self):
        return self.n

    def __getitem__(self, k):
        return np.tile(self.tile, [s // t for s, t in zip(self.shape, self.tile.shape)])


def _patch_bytes(gen, B):
    """a generous bound of everything a batch allocates besides its images: inputs, targets, labels and their workspaces"""
    P = int(np.prod(gen.patch_size))
    C1 = 1 if gen.n_channel is None else gen.n_channel
    return B * P * (4 * C1 + 4 * 4 + 2) + 2 * B * P * (gen.n_rays + 2) * 4 + (32 << 20)


@pytest.mark.parametrize("cache", (False, True))
def test_lazy_memory_on_large_volumes(cache):
    """8 volumes of 160x512x512: the resident path would hold 8 * 42M voxels * 12 bytes = 4.0 GB on the device"""
    import torch
    from stardist_b200.models import StarDistData3D
    from stardist_b200.rays3d import Rays_GoldenSpiral
    shape, B = (160, 512, 512), 2
    X, Y = _Volumes(8, shape, True), _Volumes(8, shape, False)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    np.random.seed(0)
    gen = StarDistData3D(X, Y, batch_size=B, rays=Rays_GoldenSpiral(96), length=8, patch_size=(64, 128, 128), grid=(1, 2, 2),
                         foreground_prob=0.5, sample_ind_cache=cache)
    assert torch.cuda.memory_allocated() == base
    V = int(np.prod(shape))
    rows = int(np.prod([s - p + 1 for s, p in zip(shape[:-1], gen.patch_size[:-1])]))
    after = None
    for i in range(4):
        held = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        outs = gen.batch_device(i)
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() - held
        # per item: X float32, Y int32, its relabelling, a foreground mask; one mask read in flight for the valid positions
        bound = B * (4 + 4 + 4 + 1) * V + 4 * V + B * 8 * rows + _patch_bytes(gen, B)
        print("batch %d: peak %.1f MB over %.1f MB held, bound %.1f MB" % (i, peak / 2 ** 20, (held - base) / 2 ** 20, bound / 2 ** 20))
        assert peak <= bound, (i, peak, bound)
        del outs
        torch.cuda.synchronize()
        now = torch.cuda.memory_allocated() - base
        if not cache:
            if after is None:
                after = now
                assert after <= 512                        # gen.last_positions
            assert now == after, (i, now, after)
    if cache:
        n_cached = len(gen._lazy.cache[True])
        per = 512 * (-(-V // 512)) + 512 * (-(-(rows + 1) * 8 // 512))
        assert now <= 512 + n_cached * per, (now, n_cached)


# ------------------------------------------------------------------------------------------------ train()
class _Lazy:
    def __init__(self, items):
        self.items = items

    def __len__(self):
        return len(self.items)

    def __getitem__(self, k):
        return self.items[k]


def test_train_on_lazy_data_equals_lists():
    from stardist_b200 import Config2D, StarDist2D
    from oracle import synth
    Y = [synth.ellipse_labels((96, 96), seed=10 + i, rmin=5, rmax=9) for i in range(6)]
    X = [synth.image_from_labels(y, seed=10 + i) for i, y in enumerate(Y)]
    config = Config2D(n_rays=16, unet_n_depth=2, grid=(2, 2), train_patch_size=(64, 64), train_batch_size=2, train_epochs=2,
                      train_steps_per_epoch=6, train_n_val_patches=3, train_foreground_only=0.5)
    runs = []
    for lazy in (False, True):
        wrap = _Lazy if lazy else list
        model = StarDist2D(config, name=None, basedir=None)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            hist = model.train(wrap(X[:4]), wrap(Y[:4]), validation_data=(wrap(X[4:]), wrap(Y[4:])), seed=3)
        runs.append((model.weights, hist.history))
    (w0, h0), (w1, h1) = runs
    assert h0 == h1
    assert w0.keys() == w1.keys()
    for n in w0:
        assert all(a.tobytes() == b.tobytes() for a, b in zip(w0[n], w1[n])), n
