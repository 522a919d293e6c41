"""CPU checks of the training-batch generators over lazy X / Y (stardist_b200.models.data.LazyReads): the reads of every
case of tests/golden/lazy_reads.npz, in order and number, and numpy's global random state after every batch, with the
device's foreground count replaced by the numpy restatement of tests/traindata_emu.py; and the per-read errors."""
import json, os, sys, warnings
import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
sys.path.insert(0, HERE)
import lazy_reads_cases as C
import train_batch_cases as T
import traindata_emu as E
from stardist_b200 import _lib
from stardist_b200.models import StarDistData2D, StarDistData3D
from stardist_b200.rays3d import Rays_GoldenSpiral


def _meta():
    z = np.load(os.path.join(HERE, "golden", "lazy_reads.npz"))
    return json.loads(bytes(z["meta"]).decode())


def _host_gen(dim, X, Y, kw):
    """a generator over lazy X / Y whose foreground count is the numpy restatement: planning needs no device"""
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        gen = (StarDistData2D if dim == 2 else StarDistData3D)(X, Y, **T.make_kwargs(kw, Rays_GoldenSpiral))
    maxf = tuple(int(v) for v in np.broadcast_to(np.asarray(kw.get("maxfilter_patch_size") or gen.patch_size), (dim,)))
    gen._lazy.fg_index = lambda y: (len(E.valid_positions(y, gen.patch_size, maxf)), None)
    return gen


@pytest.fixture
def no_device(monkeypatch):
    monkeypatch.setattr(_lib, "require_cuda", lambda: None)


@pytest.mark.parametrize("name", sorted(C.cases()))
def test_read_schedule_equals_reference(name, no_device):
    dim, X, Y, kw, seed, batches, random = C.cases()[name]
    rec = _meta()[name]
    log = []
    np.random.seed(seed)
    gen = _host_gen(dim, *C.lazy(X, Y, log, random), kw)
    assert log == rec["init_reads"]
    aug = kw.get("augmenter")
    for i, b in zip(batches, rec["batches"]):
        log.clear()
        idx, plan, items = gen._lazy.plan(gen, i, gen.foreground_prob)
        assert [int(v) for v in idx] == b["index"]
        if aug is not None:          # the augmenter's own draws, replayed on patches of the same shape
            for x, y, _ in items:
                aug(np.zeros(gen.patch_size + x.shape[dim:], np.float32), np.zeros(gen.patch_size, np.int32))
        assert log == b["reads"], (i, log, b["reads"])
        assert C.state_sha() == b["state"], i


def test_construction_reads_channels_twice(no_device):
    log = []
    _, X, Y, kw, _, _, _ = C.cases()["x2ch"]
    _host_gen(2, *C.lazy(X, Y, log, False), kw)
    assert log == ["X0", "X0"]


class _Seq:
    def __init__(self, items):
        self.items = items

    def __len__(self):
        return len(self.items)

    def __getitem__(self, k):
        return self.items[k]


@pytest.mark.parametrize("bad, exc", [
    ((np.zeros((40, 40), np.float32), np.zeros((40, 41), np.int32)), ValueError),          # shapes differ
    ((np.zeros((20, 40), np.float32), np.zeros((20, 40), np.int32)), ValueError),          # smaller than the patch
    ((np.zeros((40, 40, 2), np.float32), np.zeros((40, 40), np.int32)), ValueError),       # channel axis where X[0] has none
    ((np.zeros((40, 40), np.float32), np.zeros((40, 40), np.float32)), ValueError),        # a float mask
    ((np.zeros((40, 40), np.float32), np.full((40, 40), 2 ** 30, np.int64)), ValueError),  # a label above 2^30 - 1
])
def test_malformed_item_raises_when_planned(bad, exc, no_device):
    good = (np.zeros((40, 40), np.float32), np.ones((40, 40), np.int32))
    X, Y = _Seq([good[0], bad[0]]), _Seq([good[1], bad[1]])
    gen = _host_gen(2, X, Y, dict(n_rays=8, patch_size=(32, 32), batch_size=2, length=1))
    with pytest.raises(exc):
        gen._lazy.plan(gen, 0, 0)


def test_channel_count_checked_per_item(no_device):
    X = _Seq([np.zeros((40, 40, 2), np.float32), np.zeros((40, 40, 3), np.float32)])
    Y = _Seq([np.ones((40, 40), np.int32)] * 2)
    gen = _host_gen(2, X, Y, dict(n_rays=8, patch_size=(32, 32), batch_size=2, length=1))
    with pytest.raises(AssertionError):
        gen._lazy.plan(gen, 0, 0)


def test_mask_read_for_valid_positions_must_match(no_device):
    """the reference samples positions from one read of Y[k] and crops another: both must have the item's shape"""
    reads = []

    class Shrinking(_Seq):
        def __getitem__(self, k):
            reads.append(k)
            return np.ones((40, 40) if len(reads) % 2 else (48, 40), np.int32)
    gen = _host_gen(2, _Seq([np.zeros((40, 40), np.float32)]), Shrinking([None]), dict(n_rays=8, patch_size=(32, 32), batch_size=1, length=1))
    with pytest.raises(ValueError, match="corresponding shapes"):
        gen._lazy.plan(gen, 0, 0)
    assert len(reads) == 2


def test_not_a_sequence():
    with pytest.raises(ValueError):
        StarDistData2D((v for v in [np.zeros((8, 8))]), [np.zeros((8, 8), np.int32)], batch_size=1, n_rays=8, length=1, patch_size=(8, 8))
