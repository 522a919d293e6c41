"""The device augmenter (stardist_b200.models.Augmenter, csrc/augment.cu) on the GPU: the Gaussian generator against
np.random.normal, the reference's generators with the notebook augmenter (tests/golden/augment.npz), the host path fed the
same augmentation (tests/augment_emu.py's aug_emu as a plain callable) on resident and lazy datasets, and train()."""
import json, os, sys, warnings
import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import augment_cases as A
import augment_emu as E
import train_batch_cases as T

pytestmark = pytest.mark.gpu


def _ulp(a, b):
    a, b = np.asarray(a, np.float64).view(np.int64), np.asarray(b, np.float64).view(np.int64)
    return np.abs(a - b)


@pytest.mark.parametrize("pos,has_gauss", [(0, 0), (0, 1), (623, 0), (623, 1), (624, 0), (624, 1), (300, 1)])
@pytest.mark.parametrize("n", (0, 1, 2, 7, 1001, 4 * 256 * 256, 2 * 128 ** 3))
def test_generator_against_numpy(pos, has_gauss, n):
    from stardist_b200.models.augment import normal_device
    np.random.seed(pos + 11 * has_gauss)
    state = ("MT19937", np.random.get_state()[1], pos, has_gauss, 1.25 if has_gauss else 0.0)
    np.random.set_state(state)
    want = np.random.normal(0, 1, n)
    st_want = np.random.get_state()
    np.random.set_state(state)
    got = normal_device(n).cpu().numpy()
    st = np.random.get_state()
    assert np.array_equal(st[1], st_want[1]) and st[2:4] == st_want[2:4]
    u = _ulp(got, want)
    assert u.max(initial=0) <= 4
    if st[3]:
        assert _ulp(st[4], st_want[4]) <= 4
    else:
        assert st[4] == st_want[4] == 0.0
    print("n=%d pos=%d has_gauss=%d: %d of %d values not identical (max %d ulp)" % (n, pos, has_gauss, int((u > 0).sum()), n,
                                                                                   int(u.max(initial=0))))


def _meta():
    z = np.load(os.path.join(HERE, "golden", "augment.npz"))
    return json.loads(bytes(z["meta"]).decode())


class _Lazy:
    def __init__(self, items):
        self.items = items

    def __len__(self):
        return len(self.items)

    def __getitem__(self, k):
        return self.items[k]


def _make(name, augmenter=None, lazy=False):
    from stardist_b200.models import Augmenter, StarDistData2D, StarDistData3D
    from stardist_b200.rays3d import Rays_GoldenSpiral
    dim, X, Y, kw, seed, batches, akw, _ = A.cases()[name]
    if augmenter is None:
        augmenter = Augmenter(**akw)
    if lazy:
        X, Y = _Lazy(X), _Lazy(Y)
    np.random.seed(seed)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        gen = (StarDistData2D if dim == 2 else StarDistData3D)(X, Y, augmenter=augmenter, **T.make_kwargs(kw, Rays_GoldenSpiral))
    return gen, batches


def _state():
    _, key, pos, hg, gauss = np.random.get_state()
    return [T.sha(np.asarray(key, np.uint32)), int(pos), int(hg), float(gauss).hex()]


@pytest.mark.parametrize("name", sorted(A.cases()))
def test_fixture_batches_and_states(name):
    rec = _meta()[name]
    gen, batches = _make(name)
    for i, b in zip(batches, rec):
        assert [int(v) for v in gen.batch(i)] == b["index"]
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            (x,), outs = gen[i]
        assert gen.last_positions.cpu().numpy().tolist() == b["positions"]
        assert _state() == b["state"], "np.random state after batch %d" % i
        arrs = (x,) + tuple(outs)
        assert len(arrs) == len(b["outputs"])
        for k, (a, (shape, dtype, h)) in enumerate(zip(arrs, b["outputs"])):
            assert list(a.shape) == shape and str(a.dtype) == dtype
            assert T.sha(a) == h, "output %d of batch %d differs" % (k, i)


def _host_augmenter(name):
    akw = A.cases()[name][6]
    return lambda x, y: E.aug_emu(x, y, **akw)


def _run(gen, batches, device):
    out = []
    for i in batches:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            if device:
                (x,), outs = gen.batch_device(i)
                arrs = [a.cpu().numpy() for a in (x,) + tuple(outs)]
            else:
                (x,), outs = gen[i]
                arrs = [np.array(a) for a in (x,) + tuple(outs)]
        out.append((arrs, _state()))
    return out


@pytest.mark.parametrize("name", sorted(A.cases()))
@pytest.mark.parametrize("lazy", (False, True))
@pytest.mark.parametrize("device", (False, True))
def test_device_augmenter_equals_host_path(name, lazy, device):
    """the device augmenter and the host path with the same augmentation as a plain callable: byte-identical batches and the
    same np.random state, through __getitem__ and batch_device"""
    gen, batches = _make(name, lazy=lazy)
    got = _run(gen, batches, device)
    gen, batches = _make(name, augmenter=_host_augmenter(name), lazy=lazy)
    want = _run(gen, batches, device)
    for i, ((a, sa), (b, sb)) in enumerate(zip(got, want)):
        assert sa == sb, "state after batch %d" % i
        assert len(a) == len(b)
        for k, (u, v) in enumerate(zip(a, b)):
            assert u.shape == v.shape and u.dtype == v.dtype and u.tobytes() == v.tobytes(), "output %d of batch %d" % (k, i)


def _train(augmenter):
    from stardist_b200 import Config2D, StarDist2D
    from oracle import synth
    Y = [synth.ellipse_labels((96, 96), seed=30 + i, rmin=5, rmax=9) for i in range(6)]
    X = [synth.image_from_labels(y, seed=30 + i) for i, y in enumerate(Y)]
    config = Config2D(n_rays=16, unet_n_depth=2, grid=(2, 2), train_patch_size=(64, 64), train_batch_size=2, train_epochs=3,
                      train_steps_per_epoch=8, train_n_val_patches=3, train_foreground_only=0.5)
    model = StarDist2D(config, name=None, basedir=None)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        hist = model.train(X[:4], Y[:4], validation_data=(X[4:], Y[4:]), augmenter=augmenter, seed=5)
    return model.weights, hist.history


def _same_weights(w0, w1):
    return w0.keys() == w1.keys() and all(all(a.tobytes() == b.tobytes() for a, b in zip(w0[n], w1[n])) for n in w0)


def test_train_with_augmenter():
    from stardist_b200.models import Augmenter
    w0, h0 = _train(Augmenter())
    w1, h1 = _train(Augmenter())
    assert h0 == h1 and _same_weights(w0, w1)
    w2, h2 = _train(lambda x, y: E.aug_emu(x, y))
    assert h0 == h2 and _same_weights(w0, w2)
    print("val_loss per epoch:", h0["val_loss"])
    assert h0["val_loss"][-1] < h0["val_loss"][0]
