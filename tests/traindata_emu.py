"""numpy restatement of the sampling of the training-batch generators (stardist/sample_patches.py get_valid_inds, with the
foreground filter of base.py:198-210), for the CPU tests of tests/test_cpu_train_batch.py."""
import numpy as np


def fg_mask(y, size):
    """maximum_filter(y, size, mode='constant') > 0 as a separable box dilation of y > 0: along each axis, output i is set
    when some input of [i - size//2, i + size-1-size//2] is (outside the image counts as unset)"""
    m = np.asarray(y) > 0
    size = np.broadcast_to(np.asarray(size), (m.ndim,))
    for a, f in enumerate(size):
        f = int(f)
        lo, hi = f // 2, f - 1 - f // 2
        c = np.cumsum(np.moveaxis(m, a, 0).astype(np.int64), axis=0)
        c = np.concatenate([np.zeros((1,) + c.shape[1:], np.int64), c])
        n = m.shape[a]
        i = np.arange(n)
        top, bot = np.minimum(i + hi + 1, n), np.maximum(i - lo, 0)
        m = np.moveaxis((c[top] - c[bot]) > 0, 0, a)
    return m


def valid_positions(y, patch_size, filter_size=None):
    """int [n, ndim]: the valid patch centres in the reference's order (C order over the box [p//2, s-p+p//2]; with a filter
    size, only where fg_mask is set)"""
    box = tuple(slice(p // 2, s - p + p // 2 + 1) for p, s in zip(patch_size, y.shape))
    if filter_size is None:
        keep = np.ones(tuple(b.stop - b.start for b in box), bool)
    else:
        keep = fg_mask(y, filter_size)[box]
    return np.stack([v + b.start for v, b in zip(np.nonzero(keep), box)], axis=1)
