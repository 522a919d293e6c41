"""CPU checks of the training-batch generators (stardist_b200.models.data): the foreground mask restatement, scipy's order-0
zoom index rule, and the host sampling planner against every position recorded in tests/golden/train_batch.npz."""
import json, os, sys, warnings
import numpy as np
import pytest
from scipy.ndimage import maximum_filter, zoom

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
sys.path.insert(0, HERE)
import train_batch_cases as C
import traindata_emu as E
from stardist_b200.models.data import RollingSequence, plan_batch, zoom_order0_index
from stardist_b200.utils import grid_divisible_patch_size


@pytest.mark.parametrize("ndim", (2, 3))
def test_fg_mask_equals_maximum_filter(ndim):
    rng = np.random.default_rng(ndim)
    for trial in range(60):
        shape = tuple(int(v) for v in rng.integers(1, 24 if ndim == 2 else 10, ndim))
        y = rng.integers(-3, 4, shape) * (rng.random(shape) < rng.choice([0.02, 0.2, 0.8]))
        size = tuple(int(v) for v in rng.integers(1, 2 * max(shape) + 3, ndim))      # even, odd and larger than the image
        want = maximum_filter(y, size, mode='constant') > 0
        assert np.array_equal(E.fg_mask(y, size), want), (shape, size)


def test_zoom_order0_index_equals_scipy():
    for g in range(1, 9):
        for n in range(1, 513):
            n_out, ix = zoom_order0_index(n, 1 / g)
            src = np.arange(n, dtype=np.float32) + 1
            want = zoom(src, 1 / g, order=0)
            assert want.shape == (n_out,), (n, g)
            assert np.array_equal(np.where(ix >= 0, src[ix], 0), want), (n, g)


def test_grid_divisible_patch_size_warns():
    with pytest.warns(UserWarning, match="increasing patch_size"):
        assert grid_divisible_patch_size((30, 27), (2, 4)) == (30, 28)
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        assert grid_divisible_patch_size((32, 28), (2, 4)) == (32, 28)


def _meta():
    z = np.load(os.path.join(HERE, "golden", "train_batch.npz"))
    return json.loads(bytes(z["meta"]).decode())


@pytest.mark.parametrize("name", sorted(C.cases()))
def test_planner_reproduces_recorded_positions(name):
    """the random stream without a GPU: the product's planner, fed the n_valid of the numpy restatement, draws the recorded
    image indices and positions (an augmenter's own draws are replayed on dummy patches of the same shape)"""
    dim, X, Y, kw, seed, batches = C.cases()[name]
    rec = _meta()[name]
    grid = kw.get("grid", (1,) * dim)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        p = grid_divisible_patch_size(kw["patch_size"], grid)
    maxf = kw.get("maxfilter_patch_size") or p
    fp = kw.get("foreground_prob", 0)
    seq = RollingSequence(len(X), kw["batch_size"], kw["length"])
    cache = {}

    def n_valid(k, fg):
        key = (k, fg)
        if key not in cache:
            cache[key] = E.valid_positions(np.asarray(Y[k]), p, maxf if fg else None)
        return len(cache[key])

    np.random.seed(seed)
    for i, b in zip(batches, rec["batches"]):
        idx, plan = plan_batch(seq, i, fp, n_valid)
        assert [int(v) for v in idx] == b["index"]
        got = [[int(v) for v in cache[(k, fg)][r]] for k, fg, r in plan]
        assert got == b["positions"], (i, got, b["positions"])
        aug = kw.get("augmenter")
        if aug is not None:
            ch = () if np.asarray(X[0]).ndim == dim else (np.asarray(X[0]).shape[-1],)
            for _ in plan:
                aug(np.zeros(p + ch, np.float32), np.zeros(p, np.int32))
