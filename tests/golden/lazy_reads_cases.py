"""Cases of tests/golden/lazy_reads.npz (make_lazy_reads.py): training-batch generators over lazy X / Y that log every
read.  Shared by the generator (which runs the reference's StarDistData2D / StarDistData3D) and the tests (which run
stardist_b200's).  Everything is built from fixed seeds; nothing here needs a GPU or the reference."""
import hashlib
import numpy as np
import train_batch_cases as T


class Recording:
    """a lazy X or Y over a list of arrays: every read appends '<tag><k>' to log; draw(a), when given, transforms the array
    read and may draw from np.random (as a random loader does)"""

    def __init__(self, data, tag, log, draw=None):
        self.data, self.tag, self.log, self.draw = data, tag, log, draw

    def __len__(self):
        return len(self.data)

    def __getitem__(self, k):
        self.log.append("%s%d" % (self.tag, int(k)))
        a = self.data[int(k)]
        return a if self.draw is None else self.draw(a)


def random_shift(y):
    """a different mask at every read: rolled along the last axis by a random amount"""
    return np.roll(y, np.random.randint(0, 7), axis=-1)


def random_offset(x):
    return x + np.float32(np.random.uniform(-0.25, 0.25))


def state_sha(state=None):
    """sha256 of numpy's global random state"""
    st = np.random.get_state() if state is None else state
    return hashlib.sha256(np.asarray(st[1]).tobytes() + repr(tuple(st[2:])).encode()).hexdigest()


def cases():
    """name -> (dim, X list, Y list, kwargs, seed, batch indices, random loader)"""
    C = {}
    shapes = [(64, 80), (72, 64), (96, 96)]
    Y3 = [T._blobs(s, 6, 10 + i) for i, s in enumerate(shapes)]
    X3 = [T._img(s, 20 + i) for i, s in enumerate(shapes)]
    base = dict(n_rays=16, patch_size=(32, 32), grid=(1, 1), batch_size=3, length=4)
    for fp in (0, 0.5, 1):
        for cache in (True, False):
            C["fg%g_%s" % (fp, "cache" if cache else "nocache")] = (
                2, X3, Y3, dict(base, foreground_prob=fp, sample_ind_cache=cache), 1, [0, 1, 2, 3], False)
    empty = [np.zeros((64, 64), np.int32), Y3[0]]
    Xe = [T._img((64, 64), 3), X3[0]]
    for cache in (True, False):
        C["empty_%s" % ("cache" if cache else "nocache")] = (
            2, Xe, empty, dict(base, batch_size=2, length=3, foreground_prob=1, sample_ind_cache=cache), 2, [0, 1, 2], False)
        C["dup_b5_%s" % ("cache" if cache else "nocache")] = (
            2, X3, Y3, dict(base, batch_size=5, length=3, foreground_prob=0.5, sample_ind_cache=cache), 6, [0, 1, 2], False)
        C["random_%s" % ("cache" if cache else "nocache")] = (
            2, X3, Y3, dict(base, foreground_prob=0.5, sample_ind_cache=cache), 17, [0, 1, 2, 3], True)
    C["x2ch"] = (2, [T._img(s, 30 + i, 2) for i, s in enumerate(shapes)], Y3, dict(base, length=2, foreground_prob=0.5, grid=(2, 2)),
                 7, [0, 1], False)
    C["classes"] = (2, X3, Y3, dict(base, length=2, n_classes=2, classes=[{i: 1 + i % 2 for i in range(1, 7)}] * 3, grid=(1, 2),
                                    foreground_prob=0.5), 13, [0, 1], False)
    C["augmenter"] = (2, X3, Y3, dict(base, length=2, augmenter=T.flip_noise_augmenter, foreground_prob=0.5), 11, [0, 1], True)
    s3 = [(24, 40, 36), (20, 36, 40)]
    Y33 = [T._blobs(s, 8, 60 + i, radius=(3, 7)) for i, s in enumerate(s3)]
    X33 = [T._img(s, 70 + i) for i, s in enumerate(s3)]
    for cache in (True, False):
        C["vol_%s" % ("cache" if cache else "nocache")] = (
            3, X33, Y33, dict(rays=("golden", 96), grid=(1, 2, 2), patch_size=(16, 32, 32), batch_size=3, length=3, foreground_prob=0.5,
                              sample_ind_cache=cache), 15, [0, 1, 2], False)
    C["vol_random"] = (3, X33, Y33, dict(rays=("golden", 96), grid=(1, 2, 2), anisotropy=(2, 1, 1), patch_size=(16, 32, 32), batch_size=2,
                                         length=3, foreground_prob=0.7), 18, [0, 1, 2], True)
    return C


def lazy(X, Y, log, random):
    """(X, Y) as Recording sequences sharing one log"""
    return (Recording(X, "X", log, random_offset if random else None), Recording(Y, "Y", log, random_shift if random else None))
