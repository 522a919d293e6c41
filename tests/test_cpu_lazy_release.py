"""A dropped lazy generator is freed at once, without the cyclic garbage collector, so the foreground masks it caches on the
device do not outlive it (with and without the device augmenter).  No device is needed: a lazy generator uploads nothing
at construction."""
import gc, weakref
import numpy as np
import pytest

from stardist_b200 import _lib


class _Lazy:
    def __init__(self, items):
        self.items = items

    def __len__(self):
        return len(self.items)

    def __getitem__(self, k):
        return self.items[k]


@pytest.mark.parametrize("augment", (False, True))
def test_dropped_lazy_generator_is_freed_without_gc(augment, monkeypatch):
    from stardist_b200.models import Augmenter, StarDistData2D
    monkeypatch.setattr(_lib, "require_cuda", lambda: None)
    X, Y = _Lazy([np.zeros((64, 64), np.float32)]), _Lazy([np.zeros((64, 64), np.int32)])
    enabled = gc.isenabled()
    gc.disable()
    try:
        gen = StarDistData2D(X, Y, batch_size=1, n_rays=8, length=1, patch_size=(32, 32), augmenter=Augmenter() if augment else None)
        ref = weakref.ref(gen)
        del gen
        assert ref() is None
    finally:
        if enabled:
            gc.enable()
