"""Inputs of the group_matching_labels fixture (make_group_matching.py -> group_matching.npz): small seeded time-lapse stacks
in 2-D and 3-D, as arrays and as lists, in uint16 / int32 / int64, with non-sequential and large ids (up to 2^31 - 1), empty
frames, frames whose objects are all new, identical frames, shifted frames whose objects split or merge, and equal-score
alternatives in the assignment.  Every case is run under each (criterion, thresh) of RUNS."""
import numpy as np

RUNS = (('iou', 1e-10), ('iou', 0.5), ('iou', 1.0), ('iot', 1e-10), ('iot', 0.5), ('iop', 0.5))
INT32_MAX = 2 ** 31 - 1


def _blobs(rng, shape, n):
    """label image with up to n random boxes / ellipsoids painted in order (later ones on top), ids 1..n"""
    y = np.zeros(shape, np.int32)
    grids = np.meshgrid(*[np.arange(s) for s in shape], indexing='ij')
    for k in range(1, n + 1):
        c = [rng.uniform(0, s) for s in shape]
        r = [rng.uniform(1.5, max(2.0, s / 6)) for s in shape]
        d = sum(((g - ci) / ri) ** 2 for g, ci, ri in zip(grids, c, r))
        y[(d <= 1) if rng.uniform() < 0.6 else (np.maximum.reduce([np.abs(g - ci) / ri for g, ci, ri in zip(grids, c, r)]) <= 1)] = k
    return y


def _renumber(rng, y, lo=1, hi=1000):
    """the labels of y mapped to distinct random ids in [lo, hi] (0 stays 0)"""
    u = np.unique(y[y > 0])
    new = rng.choice(np.arange(lo, hi + 1, dtype=np.int64), size=len(u), replace=False) if hi - lo < 10 ** 6 else \
        np.unique(rng.integers(lo, hi + 1, size=4 * len(u) + 8, dtype=np.int64))[:len(u)]
    rng.shuffle(new)
    lut = np.zeros(int(y.max()) + 1 if y.size else 1, np.int64)
    lut[u] = new
    return lut[y]


def _movie(rng, shape, T, n, drop=0.15, hi=1000):
    """frames moving by small shifts, each relabelled at random; some objects vanish, some appear"""
    base = _blobs(rng, shape, n)
    frames = []
    for t in range(T):
        y = np.roll(base, tuple(int(v) for v in rng.integers(-2, 3, len(shape))), axis=tuple(range(len(shape))))
        keep = rng.uniform(size=n + 1) >= drop
        keep[0] = True
        y = np.where(keep[y], y, 0)
        extra = _blobs(rng, shape, 2)
        y = np.where((y == 0) & (extra > 0), extra + n, y)
        frames.append(_renumber(rng, y, hi=hi))
        base = np.roll(base, 1, axis=len(shape) - 1)
    return frames


def _ties():
    """equal-score alternatives whose order differs between the original and the grouped ids: frame 0 holds two equal
    boxes L (id 10) and R (id 20); frame 1 the same boxes with L = 2, R = 1 (so R comes first by label, L by grouped id);
    frame 2 one box overlapping both by the same amount, frame 3 the two boxes again with the labels of frame 1, swapped"""
    y = np.zeros((4, 12, 20), np.int32)
    y[0, 2:6, 2:8] = 10; y[0, 2:6, 12:18] = 20
    y[1, 2:6, 2:8] = 2; y[1, 2:6, 12:18] = 1
    y[2, 2:6, 5:15] = 7
    y[3, 2:6, 2:8] = 1; y[3, 2:6, 12:18] = 2
    y[:, 8:10, 2:4] = np.array([3, 5, 4, 6])[:, None, None]        # one more object per frame that matches its own
    return y


def _split_merge(rng):
    """object A of frame 0 splits into two in frame 1, which merge back in frame 2; B and C merge in frame 1"""
    y = np.zeros((3, 16, 24), np.int32)
    y[0, 2:8, 2:10] = 4; y[0, 10:14, 2:8] = 6; y[0, 10:14, 8:14] = 9
    y[1, 2:8, 3:6] = 1; y[1, 2:8, 6:11] = 3; y[1, 10:14, 3:14] = 2
    y[2, 2:8, 3:11] = 8; y[2, 10:14, 4:9] = 5; y[2, 10:14, 9:15] = 3
    return y


def cases():
    """name -> list of frames (a case whose name ends in '_list' is passed as a list, the others as one stacked array)"""
    rng = np.random.default_rng(7)
    out = {}
    out['2d_int32'] = np.stack(_movie(rng, (40, 56), 5, 14)).astype(np.int32)
    out['2d_uint16_list'] = [f.astype(np.uint16) for f in _movie(rng, (36, 48), 4, 12, hi=60000)]
    out['2d_int64_list'] = [f.astype(np.int64) for f in _movie(rng, (32, 40), 4, 10)]
    big = _movie(rng, (32, 40), 3, 10, hi=INT32_MAX)
    big[0] = np.where(big[0] > 0, big[0] % 1000 + INT32_MAX - 2000, 0)   # next_id just below 2^31 - 1000: room for the new ids
    big[1][big[1] == big[1].max()] = INT32_MAX
    out['2d_large_ids_int64'] = np.stack(big).astype(np.int64)
    out['3d_int32'] = np.stack(_movie(rng, (8, 20, 24), 4, 10)).astype(np.int32)
    out['3d_uint16_list'] = [f.astype(np.uint16) for f in _movie(rng, (6, 16, 20), 3, 8)]
    e = _movie(rng, (30, 30), 5, 8)
    e[1][:] = 0; e[3][:] = 0; e[4][:] = 0
    out['empty_frames'] = np.stack(e).astype(np.int32)
    z = np.zeros((3, 30, 30), np.int32)
    z[0, 2:10, 2:10] = 5; z[0, 15:20, 3:9] = 2
    z[1, 20:28, 20:28] = 5; z[1, 2:6, 20:25] = 1; z[1, 12:14, 12:26] = 3     # nothing overlaps frame 0: all new
    z[2] = z[1]
    out['all_new'] = z
    f = _renumber(rng, _blobs(rng, (28, 36), 9))
    out['identical'] = np.stack([f, f, f]).astype(np.int32)
    out['split_merge'] = _split_merge(rng)
    out['ties'] = _ties()
    return out


def shuffle_labels(y, rng):
    """stardist/matching.py _shuffle_labels with an explicit generator: the non-zero labels of y permuted at random"""
    ids = np.unique(y[y > 0])
    lut = np.zeros(int(y.max()) + 1, y.dtype)
    lut[ids] = rng.permutation(ids)
    return lut[y]


def grouping_frames(y0, seed=0):
    """the frames of the reference's test_grouping (tests/test_matching.py:35-54): y0, then 5 frames each the previous one
    with shuffled labels, rolled by 15"""
    rng = np.random.default_rng(seed)
    ys = [y0]
    for _ in range(5):
        ys.append(np.roll(shuffle_labels(ys[-1], rng), 15))
    return ys
