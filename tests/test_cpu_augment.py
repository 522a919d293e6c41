"""CPU checks of the device augmenter (stardist_b200.models.Augmenter): the numpy restatement of np.random.normal's legacy
generator (tests/augment_emu.py) against numpy itself, the host-side draw order against the reference's notebook augmenter
(tests/golden/augment.npz), argument errors raised before the device, and the robustness of every fixture noise value: its
float32 result does not move when the Gaussian value moves by 4 ulp either way (the device's double log may differ from the
C library's by a few ulp)."""
import json, os, sys, warnings
import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
sys.path.insert(0, HERE)
import augment_cases as A
import augment_emu as E
import traindata_emu as TE
from stardist_b200 import _lib
from stardist_b200.models import Augmenter
from stardist_b200.models.data import RollingSequence, plan_batch
from stardist_b200.utils import grid_divisible_patch_size


def _same_state(s, t):
    return s[0] == t[0] and np.array_equal(s[1], t[1]) and int(s[2]) == int(t[2]) and int(s[3]) == int(t[3]) and float(s[4]) == float(t[4])


@pytest.mark.parametrize("pos", (0, 623, 624))
@pytest.mark.parametrize("has_gauss", (0, 1))
@pytest.mark.parametrize("n", (0, 1, 2, 7, 1000, 10 ** 6))
def test_normal_emu_equals_numpy(pos, has_gauss, n):
    np.random.seed(pos + 7 * has_gauss)
    key = np.random.get_state()[1]
    state = ("MT19937", key, pos, has_gauss, -0.8125 if has_gauss else 0.0)
    np.random.set_state(state)
    want = np.random.normal(0, 1, n)
    got, after = E.normal_emu(state, n)
    assert np.array_equal(got, want)
    assert _same_state(after, np.random.get_state())


def test_twist_equals_numpy():
    np.random.seed(3)
    key = np.random.get_state()[1]
    np.random.set_state(("MT19937", key, 624, 0, 0.0))
    np.random.random_sample()                          # two words, the first after one twist
    assert np.array_equal(np.random.get_state()[1], E.twist(key))


@pytest.fixture
def no_device(monkeypatch):
    monkeypatch.setattr(_lib, "require_cuda", lambda: pytest.fail("device touched"))


@pytest.mark.parametrize("dim,patch,aug,word", [
    (2, (32, 32), Augmenter(axis=(0, 0)), "distinct"),
    (2, (32, 32), Augmenter(axis=(0, 2)), "axes of the"),
    (2, (32, 32), Augmenter(axis=(0.5,)), "axes of the"),
    (2, (32, 48), Augmenter(), "differs"),
    (3, (16, 32, 32), Augmenter(), "differs"),
    (3, (16, 32, 48), Augmenter(axis=(1, 2)), "differs"),
    (2, (32, 32), Augmenter(noise=-0.01), "noise"),
    (2, (32, 32), Augmenter(scale=(1,)), "scale"),
])
def test_argument_errors_before_the_device(dim, patch, aug, word, no_device):
    from stardist_b200.models import StarDistData2D, StarDistData3D
    from stardist_b200.rays3d import Rays_GoldenSpiral
    shape = tuple(2 * p for p in patch)
    X, Y = [np.zeros(shape, np.float32)], [np.zeros(shape, np.int32)]
    with pytest.raises(ValueError, match=word):
        if dim == 2:
            StarDistData2D(X, Y, batch_size=1, n_rays=8, length=1, patch_size=patch, augmenter=aug)
        else:
            StarDistData3D(X, Y, batch_size=1, rays=Rays_GoldenSpiral(8), length=1, patch_size=patch, augmenter=aug)


def test_anisotropic_patch_accepted_along_equal_axes(no_device):
    assert Augmenter(axis=(1, 2)).checked_axis((16, 32, 32)) == (1, 2)
    assert Augmenter(axis=(-1, -2)).checked_axis((16, 32, 32)) == (2, 1)
    assert Augmenter(noise=None).checked_axis((33, 33)) == (0, 1)


def _meta():
    z = np.load(os.path.join(HERE, "golden", "augment.npz"))
    return json.loads(bytes(z["meta"]).decode())


def _replay(name):
    """the fixture case on the host: per batch the planner's draws, then per item the product's Augmenter draws and numpy's
    own Gaussian values -> [(batch record, [(intensity-changed float32 patch, sigma, noise float64)] per item, state)]"""
    dim, X, Y, kw, seed, batches, akw, _ = A.cases()[name]
    grid = kw.get("grid", (1,) * dim)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        p = grid_divisible_patch_size(kw["patch_size"], grid)
    aug = Augmenter(**akw)
    axis = aug.checked_axis(p)
    seq = RollingSequence(len(X), kw["batch_size"], kw["length"])
    cache = {}

    def n_valid(k, fg):
        if (k, fg) not in cache:
            cache[(k, fg)] = TE.valid_positions(np.asarray(Y[k]), p, p if fg else None)
        return len(cache[(k, fg)])

    np.random.seed(seed)
    out = []
    for i, rec in zip(batches, _meta()[name]):
        idx, plan = plan_batch(seq, i, kw.get("foreground_prob", 0), n_valid)
        assert [int(v) for v in idx] == rec["index"]
        items = []
        for k, fg, r in plan:
            c = cache[(k, fg)][r]
            x = X[k][tuple(slice(int(v) - q // 2, int(v) - q // 2 + q) for v, q in zip(c, p))]
            row, sig = aug.draw(axis, dim)
            s, t = (np.int32(v).view(np.float32) for v in row[6:8])
            n = None if sig is None else np.random.normal(0, 1, x.shape)
            items.append((E.intensity(x, s, t), sig, n))
        out.append((rec, items, np.random.get_state()))
    return out


@pytest.mark.parametrize("name", sorted(A.cases()))
def test_draw_order_leaves_the_notebook_state(name):
    """the product's host draws (Augmenter.draw) with numpy's Gaussian values leave np.random where the reference's generator
    with the notebook augmenter left it, batch after batch"""
    for rec, _, st in _replay(name):
        key_sha, pos, hg, gauss = rec["state"]
        assert A.sha(np.asarray(st[1], np.uint32)) == key_sha
        assert (int(st[2]), int(st[3]), float(st[4]).hex()) == (pos, hg, gauss)


def _moved(n, k):
    """n moved by k ulp (k may be negative), float64"""
    v = n.copy()
    for _ in range(abs(k)):
        v = np.nextafter(v, np.inf if k > 0 else -np.inf)
    return v


@pytest.mark.parametrize("name", sorted(k for k, v in A.cases().items() if v[6].get("noise", 0.02) is not None))
def test_noise_values_are_robust_to_4_ulp(name):
    total = 0
    for _, items, _ in _replay(name):
        for x32, sig, n in items:
            want = E.noise_add(x32, sig, n)
            for k in (-4, -3, -2, -1, 1, 2, 3, 4):
                assert np.array_equal(E.noise_add(x32, sig, _moved(n, k)), want), (name, k)
            total += n.size
    assert total > 0
    print("%s: %d noise values, each stable under +-4 ulp" % (name, total))
