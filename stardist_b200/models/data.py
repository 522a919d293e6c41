"""Training batches on the device: StarDistData2D / StarDistData3D (stardist/models/base.py:129-225, model2d.py:29-120,
model3d.py:30-127), the data generators a StarDist training loop consumes.

The images and masks are uploaded once at construction and stay resident.  A batch is drawn on the host (the random
stream: which images, foreground or not, which rank among the valid positions) and built on the device:
- the rank of every item becomes a patch position (csrc/traindata.cu: sdb_sample_select, over the foreground mask and
  prefix counts of sdb_fg_valid_index for the foreground-restricted draws);
- one gather copies the X channels and label crops of the whole batch, clamps negative labels and marks them at the grid
  positions (sdb_train_gather);
- star distances (sdb_star_dist_batch) and edt_prob (sdb_edt_prob_batch) run over the batch with no pass crossing items,
  and write straight into the `dist_and_mask` layout; `prob_class` is sdb_class_map.
The reference's values are those of its `cpp` / scipy path (gputools and the `edt` package give different numbers).

Labels are handled through a per-image sequential relabelling (ascending order, negative labels -> 0) made at
construction: each item's labels are offset so that no two items share one, which sizes edt_prob's per-label maxima and
the class tables without reading anything back.  Star distances see the clamped original labels (compared by their low
16 bits, as the reference's uint16 cast does).

Differences from the reference, all raised before anything is launched: `shape_completion=True` and lazy (non-list) X / Y
raise NotImplementedError / ValueError; class ids are checked when the generator is made (the reference checks them per
batch), and a dict key 0 (which would class the background) is NotImplementedError.  A label of a patch that has no class
in the dict raises the reference's ValueError when that batch is made.  X is returned as float32 even when an augmenter
returns another float type.
"""
import random, threading, warnings
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


def plan_batch(seq, i, foreground_prob, n_valid):
    """the host side of batch i: (image indices, [(image, foreground_only, rank)]), drawing from np.random with exactly the
    calls of the reference's __getitem__ (StarDistDataBase.get_valid_inds, sample_patches).  n_valid(k, foreground_only)
    is the number of valid positions of image k."""
    idx = seq.batch(i)
    plan = []
    for k in idx:
        k = int(k)
        fg = bool(np.random.uniform() < foreground_prob)
        if fg and n_valid(k, True) == 0:
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


# ---------------------------------------------------------------------------------------------------- the generators

class _StarDistDataDevice(RollingSequence):

    _KWARGS = ("use_gpu", "sample_ind_cache", "maxfilter_patch_size", "keras_kwargs")

    def __init__(self, ndim, X, Y, n_rays, table, grid, batch_size, patch_size, length, n_classes=None, classes=None,
                 augmenter=None, foreground_prob=0, anisotropy=None, use_gpu=False, sample_ind_cache=True,
                 maxfilter_patch_size=None, keras_kwargs=None):
        from ..geometry.distances import _check_grid, walk_bound
        from ..labelprep import _sampling
        if not (isinstance(X, (np.ndarray, tuple, list)) and isinstance(Y, (np.ndarray, tuple, list))):
            raise ValueError("X and Y must be lists, tuples or arrays of images (lazy sequences are not supported)")
        super().__init__(data_size=len(X), batch_size=batch_size, length=length, shuffle=True, keras_kwargs=keras_kwargs)
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
        x_ndim = X[0].ndim
        if x_ndim not in (nD, nD + 1):
            raise AssertionError("images must have %d or %d dimensions" % (nD, nD + 1))
        all(y.ndim == nD and x.ndim == x_ndim and x.shape[:nD] == y.shape for x, y in zip(X, Y)) or _raise(
            ValueError("images and masks should have corresponding shapes/dimensions"))
        all(all(s >= p for s, p in zip(x.shape[:nD], patch_size)) for x in X) or _raise(
            ValueError("Some images are too small for given patch_size {patch_size}".format(patch_size=patch_size)))
        self.n_channel = None if x_ndim == nD else X[0].shape[-1]
        if self.n_channel is not None and not all(x.shape[-1] == self.n_channel for x in X):
            raise AssertionError("all images must have the same number of channels")
        if not (0 <= foreground_prob <= 1):
            raise AssertionError("foreground_prob must lie in [0, 1]")
        if augmenter is None:
            self._augment = False
            augmenter = lambda *args: args
        else:
            callable(augmenter) or _raise(ValueError("augmenter must be None or callable"))
            self._augment = True
        for y in Y:
            if not np.issubdtype(y.dtype, np.integer):
                raise ValueError("masks must be integer label images, got %s" % y.dtype)
            if y.size and (int(y.min()) < np.iinfo(np.int32).min or int(y.max()) > _MAX_LABEL):
                raise ValueError("labels must fit int32 and lie below 2^30 (labels above 2^30 - 1 are not supported)")
        self._n_classes_checked(n_classes, classes)
        maxf = patch_size if maxfilter_patch_size is None else maxfilter_patch_size
        maxf = tuple(int(v) for v in np.broadcast_to(np.asarray(maxf), (ndim,)))
        if not all(v >= 1 for v in maxf):
            raise ValueError("maxfilter_patch_size values must be >= 1")
        self._table = np.ascontiguousarray(table, np.float32)
        walk_bound(self._table, patch_size)
        self._sampling = _sampling(anisotropy, ndim)

        self.ndim, self.X_shapes = ndim, [y.shape for y in Y]
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

        # resident dataset: X float32 [..., C], Y int32, the sequential relabelling of Y and its label count
        import torch
        from ..labelprep import _relabel
        L.require_cuda()
        self._X, self._Y, self._seq, self._n, self._cls = [], [], [], [], []
        for k, (x, y) in enumerate(zip(X, Y)):
            xs = x if self.n_channel is not None else x[..., None]
            self._X.append(torch.from_numpy(np.ascontiguousarray(xs)).to("cuda"))
            yt = torch.from_numpy(np.ascontiguousarray(y, dtype=np.int32)).to("cuda")
            seq, n, labels, _, _ = _relabel(yt)
            self._Y.append(yt); self._seq.append(seq); self._n.append(n)
            if n_classes is not None:
                self._cls.append(self._class_table(classes[k], labels.cpu().numpy()))
        self._fg = {}

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
        import ctypes, torch
        lib = L.require_cuda()
        rows = int(np.prod([s - p + 1 for s, p in zip(shape[:-1], self.patch_size[:-1])]))
        mask = torch.empty(shape, dtype=torch.uint8, device="cuda")
        prefix = torch.empty(rows + 1, dtype=torch.int64, device="cuda")
        n = ctypes.c_longlong(0)
        L.check(lib.sdb_fg_valid_index(L.ptr(self._Y[k]), self.ndim, L.iarr(shape), L.iarr(self._maxf), L.iarr(self.patch_size),
                                       L.ptr(mask), L.ptr(prefix), ctypes.byref(n), L.stream_ptr()))
        with self.lock:
            self._fg[k] = (mask, prefix, int(n.value))
        return int(n.value)

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
        idx, plan = plan_batch(self, i, self.foreground_prob, self._n_valid)
        B, nd, p, g = len(plan), self.ndim, self.patch_size, self.grid
        C = 1 if self.n_channel is None else self.n_channel
        pg = tuple((a - 1) // b + 1 for a, b in zip(p, g))
        P = int(np.prod(p))
        dev = "cuda"
        rows, off = [], 0
        for k, fg, rank in plan:
            m = self._fg[k] if fg else None
            shape3 = (1,) * (3 - nd) + tuple(self.X_shapes[k])
            rows.append([self._X[k].data_ptr(), self._Y[k].data_ptr(), self._seq[k].data_ptr(), m[0].data_ptr() if m else 0,
                         m[1].data_ptr() if m else 0, rank, off, *shape3])
            off += self._n[k]
        items = self._items(rows)
        pos = torch.empty((B, 3), dtype=torch.int32, device=dev)
        L.check(lib.sdb_sample_select(L.ptr(items), nd, B, L.iarr(p), L.ptr(pos), L.stream_ptr()))
        self.last_index, self.last_positions = np.asarray(idx), pos[:, 3 - nd:]
        n_slots = off
        classes_on = self.n_classes is not None
        cls_table = None
        if classes_on:
            cls_table = np.concatenate([np.zeros(1, np.int32)] + [self._cls[k][1:] for k, _, _ in plan])

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
        L.check(lib.sdb_train_gather(L.ptr(items), L.ptr(pos), nd, B, L.iarr(p), C, L.iarr(g), L.ptr(d_cls), L.ptr(x), L.ptr(yc), L.ptr(ys),
                                     L.ptr(ye), L.ptr(neg), L.ptr(status), 1, L.stream_ptr()))
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
