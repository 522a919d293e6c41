"""Training batches on the device: StarDistData2D / StarDistData3D (stardist/models/base.py:129-225, model2d.py:29-120,
model3d.py:30-127), the data generators a StarDist training loop consumes.

X / Y given as lists, tuples or arrays are uploaded once at construction and stay resident.  Any other X / Y with len()
and integer __getitem__ returning arrays (a keras.utils.Sequence-like loader, a list-like wrapper over files, zarr-backed
arrays) is lazy: construction reads X[0] (twice when it has a channel axis) and uploads nothing, and every batch reads
exactly what the reference's __getitem__ reads, in its order (LazyReads), so a loader that draws from np.random itself
leaves the global stream, and therefore the batches, as the reference does.  Each item read goes up through a pinned
staging buffer and is relabelled on the device; the foreground mask and prefix of an image come from the read the
reference takes its valid positions from, and are kept on the device (1 byte per pixel plus the prefix) only with
sample_ind_cache=True.  Nothing else of a lazy image outlives its batch.  The resident path's construction checks (shapes,
image size, channel count, integer masks and their label range) are made on every read, before the read is uploaded;
class tables are built per item.  A lazy X item becomes float32 like a resident one (the reference keeps its dtype).

A batch is drawn on the host (the random stream: which images, foreground or not, which rank among the valid positions)
and built on the device:
- the rank of every item becomes a patch position (csrc/traindata.cu: sdb_sample_select, over the foreground mask and
  prefix counts of sdb_fg_valid_index for the foreground-restricted draws);
- one gather copies the X channels and label crops of the whole batch, clamps negative labels and marks them at the grid
  positions (sdb_train_gather);
- star distances (sdb_star_dist_batch) and edt_prob (sdb_edt_prob_batch) run over the batch with no pass crossing items,
  and write straight into the `dist_and_mask` layout; `prob_class` is sdb_class_map.
The reference's values are those of its `cpp` / scipy path (gputools and the `edt` package give different numbers).

Labels are handled through a per-image sequential relabelling (ascending order, negative labels -> 0) made at
construction (for a lazy dataset: per item read): each item's labels are offset so that no two items share one, which
sizes edt_prob's per-label maxima and the class tables without reading anything back.  Star distances see the clamped
original labels (compared by their low 16 bits, as the reference's uint16 cast does).

Differences from the reference, all raised before anything is launched: `shape_completion=True` raises
NotImplementedError, and an X / Y without len() / __getitem__ ValueError; class ids are checked when the generator is made
(the reference checks them per batch), and a dict key 0 (which would class the background) is NotImplementedError.  Two
reads of one lazy image with different shapes (the reference would crop one at positions valid for the other) raise
ValueError.  A label of a patch that has no class in the dict raises the reference's ValueError when that batch is made.
X is returned as float32 even when an augmenter returns another float type.

An Augmenter (models/augment.py) runs on the device: after the gather (labels not clamped), sdb_augment_batch transposes, flips
and rescales every item's patch and adds its noise, which sdb_mt_normal draws from np.random's stream; the targets follow as
without augmentation.  Any other callable augmenter gets numpy patches on the host, and its results are relabelled and gathered
again.
"""
import random, threading, warnings, weakref
import numpy as np

from .. import _lib as L
from ..utils import _raise, grid_divisible_patch_size

_MAX_LABEL = 2 ** 30 - 1
_CLASS_NONE, _CLASS_MISSING = -1, -2
_CONSTANT_WARNING = "EDT of constant label image is ill-defined. (Assuming background around it.)"


# ---------------------------------------------------------------------------------------------------- csbdeep, restated
# The random stream of the generators is csbdeep's (csbdeep 0.8.1: csbdeep/utils/utils.py `choice` and
# csbdeep/internals/train.py `RollingSequence`), restated here; agreement with an installed csbdeep is not checked.

def choice(population, k=1, replace=True):
    """csbdeep.utils.choice: `random` seeded from np.random's global stream, its own state restored afterwards"""
    try:
        state = random.getstate()
        random.seed(np.random.randint(np.iinfo(int).min, np.iinfo(int).max))
        return random.choices(population, k=k) if replace else random.sample(population, k=k)
    finally:
        random.setstate(state)


class RollingSequence:
    """csbdeep.internals.train.RollingSequence without the keras base class: batch(i) rolls over passes through the data,
    one np.random.permutation per pass, drawn when first needed"""

    def __init__(self, data_size, batch_size, length=None, shuffle=True, rng=None, keras_kwargs=None):
        if rng is None:
            rng = np.random
        self.data_size = int(data_size)
        self.batch_size = int(batch_size)
        self.length = 2 ** 63 - 1 if length is None else int(length)
        self.shuffle = bool(shuffle)
        self.index_gen = rng.permutation if self.shuffle else np.arange
        self.index_map = {}

    def __len__(self):
        return self.length

    def _index(self, loop):
        if loop in self.index_map:
            return self.index_map[loop]
        return self.index_map.setdefault(loop, self.index_gen(self.data_size))

    def on_epoch_end(self):
        pass

    def __iter__(self):
        for i in range(len(self)):
            yield self[i]

    def batch(self, i):
        pos = i * self.batch_size
        loop = pos // self.data_size
        pos_loop = pos % self.data_size
        sl = slice(pos_loop, pos_loop + self.batch_size)
        index = self._index(loop)
        _loop = loop
        while sl.stop > len(index):
            _loop += 1
            index = np.concatenate((index, self._index(_loop)))
        return index[sl]


def plan_batch(seq, i, foreground_prob, n_valid, read=None):
    """the host side of batch i: (image indices, [(image, foreground_only, rank)]), drawing from np.random with exactly the
    calls of the reference's __getitem__ (StarDistDataBase.get_valid_inds, sample_patches).  n_valid(k, foreground_only)
    is the number of valid positions of image k; it is called once per index lookup of the reference's get_valid_inds
    (twice when an image without foreground falls back to foreground_prob=0).  read(k), when given, is called at the start
    of every item, where the reference reads Y[k] and X[k] for sample_patches."""
    idx = seq.batch(i)
    plan = []
    for k in idx:
        k = int(k)
        if read is not None:
            read(k)
        fg = bool(np.random.uniform() < foreground_prob)
        n = n_valid(k, fg)
        if fg and n == 0:
            fg = bool(np.random.uniform() < 0)             # no foreground: get_valid_inds(k, foreground_prob=0)
            n = n_valid(k, fg)
        if n == 0:
            raise ValueError("no regions to sample from!")
        rank = choice(range(n), 1, replace=(n < 1))[0]
        plan.append((k, fg, int(rank)))
    return idx, plan


def zoom_order0_index(n_in, factor):
    """scipy.ndimage.zoom(..., order=0) along one axis (grid_mode False, mode 'constant'): (output size, source index of
    every output index, -1 for the constant 0).  Output size int(round(n_in * factor)); output k maps to c = k * ((n_in - 1)
    / (n_out - 1)) (factor 1 when n_out == 1) in float64 and reads floor(c + 0.5) -- unless c lies beyond n_in - 1, which the
    rounding of the product can make happen for the last output: then it is the constant 0."""
    n_out = int(round(n_in * factor))
    z = (n_in - 1) / (n_out - 1) if n_out > 1 else 1.0
    c = np.arange(n_out, dtype=np.float64) * z
    return n_out, np.where(c > n_in - 1, -1, np.floor(c + 0.5)).astype(np.int64)


def _class_code(cls, n_classes):
    if cls is None:
        return _CLASS_NONE
    if np.issubdtype(type(cls), np.integer) and 0 <= cls <= n_classes:
        return int(cls)
    raise ValueError(f"Wrong class id '{cls}' (for n_classes={n_classes})")


def _weak_method(method):
    """a callable for a bound method that does not keep its object alive"""
    ref = weakref.WeakMethod(method)
    return lambda *args: ref()(*args)


def _is_resident(X):
    return isinstance(X, (np.ndarray, tuple, list))


def _check_mask(y):
    if not np.issubdtype(y.dtype, np.integer):
        raise ValueError("masks must be integer label images, got %s" % y.dtype)
    if y.size and (int(y.min()) < np.iinfo(np.int32).min or int(y.max()) > _MAX_LABEL):
        raise ValueError("labels must fit int32 and lie below 2^30 (labels above 2^30 - 1 are not supported)")


class LazyReads:
    """The reads of a lazy X / Y (any object with len() and integer __getitem__ returning arrays), in the reference's order
    and number, so that a sequence drawing from np.random itself leaves the global stream as the reference does.  Per item
    of a batch: Y[k], then X[k] (the arguments of sample_patches); then one more Y[k] whenever the reference's
    _ind_cache_fg / _ind_cache_all has no entry for k (StarDistDataBase.get_valid_inds), including the fallback to
    foreground_prob=0 of an image without foreground.  The key sets of those two caches are kept here, with what the
    reference would keep for them: the shape and valid-position count, and fg_index's payload for the foreground ones.

    check_item(x, y) -> (x, y) and check_mask(y) -> y make the resident path's construction checks on every read;
    fg_index(y) -> (count, payload) computes the foreground-restricted valid positions of a mask read."""

    def __init__(self, X, Y, patch_size, sample_ind_cache, check_item, check_mask, fg_index):
        self.X, self.Y = X, Y
        self.patch_size, self.sample_ind_cache = tuple(patch_size), bool(sample_ind_cache)
        self.check_item, self.check_mask, self.fg_index = check_item, check_mask, fg_index
        self.cache = {True: {}, False: {}}

    def plan(self, seq, i, foreground_prob):
        """-> (image indices, [(image, foreground_only, rank)], [[x, y, fg payload] per item]) for batch i"""
        items = []

        def read(k):
            y = self.Y[k]
            x = self.X[k]
            items.append(list(self.check_item(x, y)) + [None])

        def n_valid(k, fg):
            item = items[-1]
            cache = self.cache[fg]
            if k in cache:
                shape, n, payload = cache[k]
            else:
                y = self.check_mask(self.Y[k])
                shape = y.shape
            if shape != item[1].shape:
                raise ValueError("images and masks should have corresponding shapes/dimensions")
            if k not in cache:
                if fg:
                    n, payload = self.fg_index(y)
                else:
                    n, payload = int(np.prod([s - p + 1 for s, p in zip(shape, self.patch_size)])), None
                if self.sample_ind_cache:
                    cache[k] = (shape, n, payload)
            if fg:
                item[2] = payload
            return n

        idx, plan = plan_batch(seq, i, foreground_prob, n_valid, read)
        return idx, plan, items


# ---------------------------------------------------------------------------------------------------- the generators

class _StarDistDataDevice(RollingSequence):

    _KWARGS = ("use_gpu", "sample_ind_cache", "maxfilter_patch_size", "keras_kwargs")

    def __init__(self, ndim, X, Y, n_rays, table, grid, batch_size, patch_size, length, n_classes=None, classes=None,
                 augmenter=None, foreground_prob=0, anisotropy=None, use_gpu=False, sample_ind_cache=True,
                 maxfilter_patch_size=None, keras_kwargs=None):
        from ..geometry.distances import _check_grid, walk_bound
        from ..labelprep import _sampling
        resident = _is_resident(X) and _is_resident(Y)
        if not resident and not all(hasattr(v, "__len__") and hasattr(v, "__getitem__") for v in (X, Y)):
            raise ValueError("X and Y must be lists, tuples or arrays of images, or sequences with len() and __getitem__")
        super().__init__(data_size=len(X), batch_size=batch_size, length=length, shuffle=True, keras_kwargs=keras_kwargs)
        if resident:
            X = [np.asarray(x).astype(np.float32, copy=False) for x in X]
            Y = [np.asarray(y) for y in Y]
        len(X) == len(Y) and len(X) > 0 or _raise(ValueError("X and Y can't be empty and must have same length"))
        if classes is None:
            classes = (None,) * len(X)
        else:
            n_classes is not None or warnings.warn("Ignoring classes since n_classes is None")
        len(classes) == len(X) or _raise(ValueError("X and classes must have same length"))
        grid = _check_grid(grid, ndim)
        patch_size = grid_divisible_patch_size(patch_size, grid)
        nD = len(patch_size)
        if nD != ndim:
            raise AssertionError("patch_size must have %d values" % ndim)
        x_ndim = np.ndim(X[0])                              # a lazy X is read here, and once more for its channel count
        if x_ndim not in (nD, nD + 1):
            raise AssertionError("images must have %d or %d dimensions" % (nD, nD + 1))
        self.n_channel = None if x_ndim == nD else int(np.shape(X[0])[-1])
        self._x_ndim = x_ndim
        if resident:
            all(y.ndim == nD and x.ndim == x_ndim and x.shape[:nD] == y.shape for x, y in zip(X, Y)) or _raise(
                ValueError("images and masks should have corresponding shapes/dimensions"))
            all(all(s >= p for s, p in zip(x.shape[:nD], patch_size)) for x in X) or _raise(
                ValueError("Some images are too small for given patch_size {patch_size}".format(patch_size=patch_size)))
            if self.n_channel is not None and not all(x.shape[-1] == self.n_channel for x in X):
                raise AssertionError("all images must have the same number of channels")
        if not (0 <= foreground_prob <= 1):
            raise AssertionError("foreground_prob must lie in [0, 1]")
        from .augment import Augmenter
        self._aug_device = self._aug_axis = None
        if augmenter is None:
            self._augment = False
            augmenter = lambda *args: args
        elif isinstance(augmenter, Augmenter):
            self._augment = False
            self._aug_device, self._aug_axis = augmenter, augmenter.checked_axis(patch_size)
        else:
            callable(augmenter) or _raise(ValueError("augmenter must be None or callable"))
            self._augment = True
        if resident:
            for y in Y:
                _check_mask(y)
        self._n_classes_checked(n_classes, classes)
        maxf = patch_size if maxfilter_patch_size is None else maxfilter_patch_size
        maxf = tuple(int(v) for v in np.broadcast_to(np.asarray(maxf), (ndim,)))
        if not all(v >= 1 for v in maxf):
            raise ValueError("maxfilter_patch_size values must be >= 1")
        self._table = np.ascontiguousarray(table, np.float32)
        walk_bound(self._table, patch_size)
        self._sampling = _sampling(anisotropy, ndim)

        self.ndim, self.X_shapes = ndim, ([y.shape for y in Y] if resident else None)
        self.n_rays, self.patch_size, self.grid = int(n_rays), tuple(patch_size), tuple(grid)
        self.ss_grid = (slice(None),) + tuple(slice(0, None, g) for g in grid)
        self.n_classes, self.classes = n_classes, classes
        self.use_gpu = bool(use_gpu)
        self.augmenter, self.foreground_prob = augmenter, foreground_prob
        self.maxfilter_patch_size = maxfilter_patch_size if maxfilter_patch_size is not None else self.patch_size
        self._maxf = maxf
        self.sample_ind_cache = sample_ind_cache
        self.lock = threading.Lock()
        self.last_index = self.last_positions = None
        self._zoom = None
        if n_classes is not None:
            zs = [zoom_order0_index(p, 1 / g) for p, g in zip(self.patch_size, self.grid)]
            self._zoom_shape = tuple(n for n, _ in zs)
            self._zoom_index = np.concatenate([ix for _, ix in zs]).astype(np.int32)

        import torch
        from ..labelprep import _relabel
        L.require_cuda()
        self._X, self._Y, self._seq, self._n, self._cls = [], [], [], [], []
        self._fg = {}
        self._lazy, self._stage, self._stage_done = None, None, None
        if not resident:
            # lazy dataset: nothing is read or uploaded until a batch needs it
            # weak references back to the generator: without a reference cycle, a dropped generator frees its cached
            # foreground masks at once, not whenever the cyclic garbage collector next runs
            self._lazy = LazyReads(X, Y, self.patch_size, sample_ind_cache, *(_weak_method(m) for m in (
                self._check_item, self._check_valid_mask, self._fg_index)))
            return
        # resident dataset: X float32 [..., C], Y int32, the sequential relabelling of Y and its label count
        for k, (x, y) in enumerate(zip(X, Y)):
            xs = x if self.n_channel is not None else x[..., None]
            self._X.append(torch.from_numpy(np.ascontiguousarray(xs)).to("cuda"))
            yt = torch.from_numpy(np.ascontiguousarray(y, dtype=np.int32)).to("cuda")
            seq, n, labels, _, _ = _relabel(yt)
            self._Y.append(yt); self._seq.append(seq); self._n.append(n)
            if n_classes is not None:
                self._cls.append(self._class_table(classes[k], labels.cpu().numpy()))

    # -------------------------------------------------------------------------------------------- classes
    @staticmethod
    def _n_classes_checked(n_classes, classes):
        if n_classes is None:
            return
        if not (np.issubdtype(type(n_classes), np.integer) and n_classes >= 1):
            raise ValueError(f"n_classes is '{n_classes}' but should be a positive integer")
        for c in classes:
            if c is None or np.issubdtype(type(c), np.integer):
                _class_code(c, n_classes)
            elif isinstance(c, dict):
                for key, v in c.items():
                    _class_code(v, n_classes)
                    if np.issubdtype(type(key), np.integer) and key == 0:
                        raise NotImplementedError("a class for label 0 (the background) is not supported")
            else:
                raise ValueError("classes should be dict, single scalar, or None!")

    def _class_table(self, classes, labels):
        """int32 [n + 1]: the class code of every sequential label 1..n of an image (entry 0 unused)"""
        t = np.zeros(len(labels) + 1, np.int32)
        if classes is None or np.issubdtype(type(classes), np.integer):
            t[1:] = _class_code(classes, self.n_classes)
        else:
            t[1:] = [_class_code(classes[int(l)], self.n_classes) if int(l) in classes else _CLASS_MISSING for l in labels]
        return t

    # -------------------------------------------------------------------------------------------- sampling
    def _n_valid(self, k, foreground_only):
        shape = self.X_shapes[k]
        if not foreground_only:
            return int(np.prod([s - p + 1 for s, p in zip(shape, self.patch_size)]))
        if self.sample_ind_cache and k in self._fg:
            return self._fg[k][2]
        m = self._fg_valid_index(self._Y[k])
        with self.lock:
            self._fg[k] = m
        return m[2]

    def _fg_valid_index(self, y):
        """sdb_fg_valid_index of a CUDA int32 mask: (foreground mask uint8, int64 prefix counts per valid row, count)"""
        import ctypes, torch
        lib = L.require_cuda()
        shape = tuple(y.shape)
        rows = int(np.prod([s - p + 1 for s, p in zip(shape[:-1], self.patch_size[:-1])]))
        mask = torch.empty(shape, dtype=torch.uint8, device="cuda")
        prefix = torch.empty(rows + 1, dtype=torch.int64, device="cuda")
        n = ctypes.c_longlong(0)
        L.check(lib.sdb_fg_valid_index(L.ptr(y), self.ndim, L.iarr(shape), L.iarr(self._maxf), L.iarr(self.patch_size),
                                       L.ptr(mask), L.ptr(prefix), ctypes.byref(n), L.stream_ptr()))
        return mask, prefix, int(n.value)

    # -------------------------------------------------------------------------------------------- lazy X / Y
    def _check_item(self, x, y):
        """an item read from a lazy X / Y, with the checks the resident path makes at construction"""
        x, y = np.asarray(x), np.asarray(y)
        nD, p = self.ndim, self.patch_size
        y.ndim == nD and x.ndim == self._x_ndim and x.shape[:nD] == y.shape or _raise(
            ValueError("images and masks should have corresponding shapes/dimensions"))
        all(s >= q for s, q in zip(y.shape, p)) or _raise(
            ValueError("Some images are too small for given patch_size {patch_size}".format(patch_size=p)))
        if self.n_channel is not None and x.shape[-1] != self.n_channel:
            raise AssertionError("all images must have the same number of channels")
        _check_mask(y)
        return x, y

    def _check_valid_mask(self, y):
        """a mask read for the valid positions only (StarDistDataBase.get_valid_inds)"""
        y = np.asarray(y)
        y.ndim == self.ndim or _raise(ValueError("images and masks should have corresponding shapes/dimensions"))
        _check_mask(y)
        return y

    def _fg_index(self, y):
        mask, prefix, n = self._fg_valid_index(self._upload(y, np.int32))
        return n, (mask, prefix)

    def _upload(self, a, dtype):
        """numpy array -> new CUDA tensor of dtype (the value conversion of astype), through the pinned staging buffer"""
        import torch
        dtype = np.dtype(dtype)
        nbytes = a.size * dtype.itemsize
        if self._stage_done is not None:
            self._stage_done.synchronize()                 # the previous upload has left the buffer
        if self._stage is None or self._stage.numel() < nbytes:
            self._stage = None
            self._stage = torch.empty(max(nbytes, 1), dtype=torch.uint8, pin_memory=True)
            self._stage_done = torch.cuda.Event()
        h = self._stage[:nbytes].view(getattr(torch, dtype.name)).view(a.shape)
        np.copyto(h.numpy(), a, casting='unsafe')
        d = torch.empty(a.shape, dtype=h.dtype, device="cuda")
        d.copy_(h, non_blocking=True)
        self._stage_done.record()
        return d

    def _lazy_items(self, plan, items):
        """the uploaded items of a lazy batch, as _batch reads the resident ones: (X, Y, sequential Y, label count, class
        table, foreground mask and prefix or None) per item"""
        from ..labelprep import _relabel
        out = []
        for (k, fg, _), (x, y, fgm) in zip(plan, items):
            xt = self._upload(x if self.n_channel is not None else x[..., None], np.float32)
            yt = self._upload(y, np.int32)
            seq, n, labels, _, _ = _relabel(yt)
            cls = self._class_table(self.classes[k], labels.cpu().numpy()) if self.n_classes is not None else None
            out.append((xt, yt, seq, n, cls, fgm if fg else None))
        return out

    def _items(self, rows):
        """int64 [B][10] item table (csrc/traindata.cu) on the device"""
        import torch
        return torch.from_numpy(np.asarray(rows, np.int64).reshape(len(rows), 10)).to("cuda")

    # -------------------------------------------------------------------------------------------- one batch
    def _batch(self, i):
        """-> (X, prob, dist_and_mask, prob_class or None, status): CUDA tensors; status int32 [1 + 2B] = (missing-class flag,
        per-item label min / max) for _finish"""
        import torch
        lib = L.require_cuda()
        if self._lazy is None:
            idx, plan = plan_batch(self, i, self.foreground_prob, self._n_valid)
            res = [(self._X[k], self._Y[k], self._seq[k], self._n[k], self._cls[k] if self._cls else None, self._fg[k] if fg else None)
                   for k, fg, _ in plan]
        else:
            idx, plan, read = self._lazy.plan(self, i, self.foreground_prob)
            res = self._lazy_items(plan, read)
            del read
        B, nd, p, g = len(plan), self.ndim, self.patch_size, self.grid
        C = 1 if self.n_channel is None else self.n_channel
        pg = tuple((a - 1) // b + 1 for a, b in zip(p, g))
        P = int(np.prod(p))
        dev = "cuda"
        rows, off = [], 0
        for (k, fg, rank), (xk, yk, seqk, nk, _, m) in zip(plan, res):
            shape3 = (1,) * (3 - nd) + tuple(yk.shape)
            rows.append([xk.data_ptr(), yk.data_ptr(), seqk.data_ptr(), m[0].data_ptr() if m else 0,
                         m[1].data_ptr() if m else 0, rank, off, *shape3])
            off += nk
        items = self._items(rows)
        pos = torch.empty((B, 3), dtype=torch.int32, device=dev)
        L.check(lib.sdb_sample_select(L.ptr(items), nd, B, L.iarr(p), L.ptr(pos), L.stream_ptr()))
        self.last_index, self.last_positions = np.asarray(idx), pos[:, 3 - nd:]
        n_slots = off
        classes_on = self.n_classes is not None
        cls_table = None
        if classes_on:
            cls_table = np.concatenate([np.zeros(1, np.int32)] + [r[4][1:] for r in res])

        status = torch.zeros(1 + 2 * B, dtype=torch.int32, device=dev)
        x = torch.empty((B,) + p + (C,), dtype=torch.float32, device=dev)
        yc = torch.empty((B,) + p, dtype=torch.int32, device=dev)
        ys = torch.empty((B,) + p, dtype=torch.int32, device=dev)
        neg = torch.empty((B,) + pg, dtype=torch.uint8, device=dev)
        ye = torch.empty((B,) + pg, dtype=torch.int32, device=dev) if nd == 2 else None
        if self._augment:
            # the augmenter's contract: numpy patches in, numpy patches out (it may draw from np.random itself)
            L.check(lib.sdb_train_gather(L.ptr(items), L.ptr(pos), nd, B, L.iarr(p), C, L.iarr(g), None, L.ptr(x), L.ptr(yc), L.ptr(ys),
                                         None, L.ptr(neg), None, 0, L.stream_ptr()))
            xh, yh = x.cpu().numpy(), yc.cpu().numpy()
            xa, ya = [], []
            for b in range(B):
                xb = xh[b] if self.n_channel is not None else xh[b, ..., 0]
                xo, yo = self.augmenter(xb, yh[b])
                xo, yo = np.asarray(xo), np.asarray(yo)
                if yo.shape != p or xo.shape[:nd] != p or not np.issubdtype(yo.dtype, np.integer):
                    raise ValueError("the augmenter must return an image and an integer mask of the patch shape %s" % (p,))
                if yo.size and (int(yo.min()) < np.iinfo(np.int32).min or int(yo.max()) > _MAX_LABEL):
                    raise ValueError("labels must fit int32 and lie below 2^30 (labels above 2^30 - 1 are not supported)")
                xa.append(xo.reshape(p + (C,))); ya.append(yo)
            from ..labelprep import _relabel
            xa = torch.from_numpy(np.ascontiguousarray(np.stack(xa), dtype=np.float32)).to(dev)
            ya = torch.from_numpy(np.ascontiguousarray(np.stack(ya), dtype=np.int32)).to(dev)
            seq, n, labels, _, _ = _relabel(ya)                # one relabelling of the whole batch; slots b * n + seq
            shape3 = (1,) * (3 - nd) + p
            rows = [[xa[b].data_ptr(), ya[b].data_ptr(), seq[b].data_ptr(), 0, 0, 0, b * n, *shape3] for b in range(B)]
            items = self._items(rows)
            pos = torch.empty((B, 3), dtype=torch.int32, device=dev)
            L.check(lib.sdb_sample_select(L.ptr(items), nd, B, L.iarr(p), L.ptr(pos), L.stream_ptr()))
            n_slots = B * n
            if classes_on:
                lab = labels.cpu().numpy()
                cls_table = np.concatenate([np.zeros(1, np.int32)] + [self._class_table(self.classes[k], lab)[1:] for k, _, _ in plan])
        d_cls = torch.from_numpy(cls_table).to(dev) if classes_on else None
        if self._aug_device is not None:
            self._augment_on_device(items, pos, d_cls, status, x, yc, ys, ye, neg)
        else:
            L.check(lib.sdb_train_gather(L.ptr(items), L.ptr(pos), nd, B, L.iarr(p), C, L.iarr(g), L.ptr(d_cls), L.ptr(x), L.ptr(yc), L.ptr(ys),
                                         L.ptr(ye), L.ptr(neg), L.ptr(status), 1, L.stream_ptr()))
        del res                # a lazy batch's images are not read past the gather (their memory is reused in stream order)
        R = self.n_rays
        dam = torch.empty((B,) + pg + (R + 1,), dtype=torch.float32, device=dev)
        prob = torch.empty((B,) + pg + (1,), dtype=torch.float32, device=dev)
        L.check(lib.sdb_star_dist_batch(L.ptr(yc), nd, B, L.iarr(p), L.iarr(g), R, L.ptr(self._table), R + 1, L.ptr(dam), L.stream_ptr()))
        mm = status[1:]
        if nd == 2:      # edt_prob of the subsampled labels, no anisotropy
            L.check(lib.sdb_edt_prob_batch(L.ptr(ye), nd, B, L.iarr(pg), n_slots, None, L.iarr((1,) * nd), L.ptr(neg), L.ptr(mm), L.ptr(prob),
                                           L.ptr(dam[..., R]), R + 1, L.stream_ptr()))
        else:            # edt_prob at full resolution, then the grid positions
            L.check(lib.sdb_edt_prob_batch(L.ptr(ys), nd, B, L.iarr(p), n_slots, L.ptr(self._sampling), L.iarr(g), L.ptr(neg), L.ptr(mm),
                                           L.ptr(prob), L.ptr(dam[..., R]), R + 1, L.stream_ptr()))
        prob_class = None
        if classes_on:
            assert self._zoom_shape == pg
            if self._zoom is None:
                self._zoom = torch.from_numpy(self._zoom_index).to(dev)
            prob_class = torch.empty((B,) + self._zoom_shape + (self.n_classes + 1,), dtype=torch.float32, device=dev)
            L.check(lib.sdb_class_map(L.ptr(ys), nd, B, L.iarr(p), L.ptr(self._zoom), L.iarr(self._zoom_shape), L.ptr(d_cls), self.n_classes,
                                      L.ptr(neg), L.ptr(prob_class), L.stream_ptr()))
        return x, prob, dam, prob_class, status

    def _augment_on_device(self, items, pos, d_cls, status, x, yc, ys, ye, neg):
        """the gather and the Augmenter: x, yc, ys, ye, neg as sdb_train_gather writes them, for the augmented patches"""
        import torch
        lib = L.require_cuda()
        B, nd, p, g = x.shape[0], self.ndim, self.patch_size, self.grid
        C = x.shape[-1]
        xr, yr, sr = torch.empty_like(x), torch.empty_like(yc), torch.empty_like(ys)
        L.check(lib.sdb_train_gather(L.ptr(items), L.ptr(pos), nd, B, L.iarr(p), C, L.iarr(g), L.ptr(d_cls), L.ptr(xr), L.ptr(yr), L.ptr(sr),
                                     None, L.ptr(neg), L.ptr(status), 0, L.stream_ptr()))
        from .augment import normal_device
        aug = self._aug_device
        noise = None if aug.noise is None else torch.empty((B, xr[0].numel()), dtype=torch.float64, device="cuda")
        rows = []
        for b in range(B):             # the notebooks' draws, item after item; the noise of an item before the next item draws
            row, sig = aug.draw(self._aug_axis, nd)
            if sig is not None:
                normal_device(noise.shape[1], noise[b])
            rows.append(row)
        prm = torch.from_numpy(np.asarray(rows, np.int64)).to("cuda")
        L.check(lib.sdb_augment_batch(L.ptr(prm), nd, B, L.iarr(p), C, L.iarr(g), L.ptr(xr), L.ptr(yr), L.ptr(sr), L.ptr(noise), L.ptr(x),
                                      L.ptr(yc), L.ptr(ys), L.ptr(ye), L.ptr(neg), L.stream_ptr()))

    def _finish(self, status):
        """the host side of the batch's single read-back: the constant-patch warning per item, the missing-class error"""
        st = np.asarray(status)
        mm = st[1:].reshape(-1, 2)
        for lo, hi in mm:
            if lo == hi and hi > 0:
                warnings.warn(_CONSTANT_WARNING)
        if st[0]:
            raise ValueError("all gt labels should be present in class dict provided")

    def batch_device(self, i):
        """__getitem__(i) as CUDA tensors: ((X,), (prob, dist_and_mask[, prob_class]))"""
        x, prob, dam, pc, status = self._batch(i)
        self._finish(status.cpu().numpy())
        return (x,), ((prob, dam) if pc is None else (prob, dam, pc))

    def __getitem__(self, i):
        import torch
        x, prob, dam, pc, status = self._batch(i)
        dev = [t for t in (x, prob, dam, pc, status) if t is not None]
        host = [torch.empty(t.shape, dtype=t.dtype, pin_memory=True) for t in dev]
        for h, d in zip(host, dev):
            h.copy_(d, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        self._finish(host[-1].numpy())
        out = [h.numpy() for h in host[:-1]]
        return (out[0],), tuple(out[1:])


class StarDistData2D(_StarDistDataDevice):
    """StarDistData2D (stardist/models/model2d.py:29-120): batches ((X,), (prob, dist_and_mask[, prob_class])) as float32
    numpy arrays equal to the reference's; batch_device(i) gives the same as CUDA tensors."""

    def __init__(self, X, Y, batch_size, n_rays, length, n_classes=None, classes=None, patch_size=(256, 256), b=32, grid=(1, 1),
                 shape_completion=False, augmenter=None, foreground_prob=0, **kwargs):
        from ..geometry.distances import direction_table_2d
        if shape_completion:
            raise NotImplementedError("shape_completion=True is not supported")
        unknown = set(kwargs) - set(self._KWARGS)
        if unknown:
            raise TypeError("StarDistData2D() got an unexpected keyword argument '%s'" % sorted(unknown)[0])
        n_rays = int(n_rays)
        n_rays >= 1 or _raise(ValueError("need 'n_rays' >= 1"))
        super().__init__(2, X, Y, n_rays, direction_table_2d(n_rays), grid, batch_size, patch_size, length, n_classes=n_classes,
                         classes=classes, augmenter=augmenter, foreground_prob=foreground_prob, **kwargs)
        self.shape_completion = False
        self.b = slice(None), slice(None)
        self.sd_mode = 'cpp'


class StarDistData3D(_StarDistDataDevice):
    """StarDistData3D (stardist/models/model3d.py:30-127), as StarDistData2D; every call returns fresh arrays"""

    def __init__(self, X, Y, batch_size, rays, length, n_classes=None, classes=None, patch_size=(128, 128, 128), grid=(1, 1, 1),
                 anisotropy=None, augmenter=None, foreground_prob=0, **kwargs):
        from ..geometry.distances import rays_table_3d
        unknown = set(kwargs) - set(self._KWARGS)
        if unknown:
            raise TypeError("StarDistData3D() got an unexpected keyword argument '%s'" % sorted(unknown)[0])
        super().__init__(3, X, Y, len(rays), rays_table_3d(rays), grid, batch_size, patch_size, length, n_classes=n_classes,
                         classes=classes, augmenter=augmenter, foreground_prob=foreground_prob, anisotropy=anisotropy, **kwargs)
        self.rays, self.anisotropy = rays, anisotropy
        self.sd_mode = 'cpp'
