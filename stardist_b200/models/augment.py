"""The augmenter of the StarDist training notebooks (examples/2D/2_training.ipynb, examples/3D/2_training.ipynb), applied on the
device by StarDistData2D / StarDistData3D: a random axis permutation and flips, a random intensity change and Gaussian noise.

    model.train(X, Y, validation_data=(Xv, Yv), augmenter=Augmenter())                            # the 2-D notebook's
    model.train(X, Y, validation_data=(Xv, Yv), augmenter=Augmenter(axis=(1, 2), noise=None))     # the 3-D notebook's

Per augmented item the draws come from the global np.random, in the notebooks' order: np.random.permutation(axis); one
np.random.rand() per axis of `axis` (> 0.5 flips that axis of the transposed patch); s = uniform(*scale), t = uniform(*shift);
with noise, sig = noise * uniform(0, 1) and np.random.normal(0, 1, x.shape).  The scalar draws are made here, on the host; the
Gaussian values are drawn on the device (csrc/augment.cu: sdb_mt_normal) from the state np.random.get_state() gives, and the
state numpy would hold afterwards is set back before the next item draws.  The image becomes float32(float32(x * float32(s)) +
float32(t)) (numpy's float32 arithmetic with a Python float) and, with noise, float32(float64(x) + sig * n); the labels are
transposed and flipped like the image.  Validation patches are never augmented.

Difference from the notebooks, raised when the generator is made: `axis` entries that are not distinct axes of the patch, patch
extents that differ along `axis` (the notebook would return a patch of another shape, which fails only at that batch), and a
negative `noise` raise ValueError.
"""
import ctypes
import numpy as np

from .. import _lib as L


class Augmenter:
    """Augmenter(axis=None, scale=(0.6, 2), shift=(-0.2, 0.2), noise=0.02): the notebooks' random_fliprot over `axis` (axes of
    the label patch, None = all), random_intensity_change with `scale` / `shift` ranges and, unless noise is None, Gaussian
    noise of standard deviation noise * uniform(0, 1).  Pass it as `augmenter` to StarDist2D/3D.train or StarDistData2D/3D."""

    def __init__(self, axis=None, scale=(0.6, 2), shift=(-0.2, 0.2), noise=0.02):
        self.axis = None if axis is None else tuple(axis)
        self.scale, self.shift, self.noise = tuple(scale), tuple(shift), noise

    def __repr__(self):
        return "Augmenter(axis=%r, scale=%r, shift=%r, noise=%r)" % (self.axis, self.scale, self.shift, self.noise)

    def checked_axis(self, patch_size):
        """the augmented axes for a patch of patch_size (ValueError for axes that are not distinct axes of the patch, for extents
        that differ along them, for a negative noise and for scale / shift that are not two numbers)"""
        nd = len(patch_size)
        axis = tuple(range(nd)) if self.axis is None else self.axis
        if not all(np.issubdtype(type(a), np.integer) and -nd <= a < nd for a in axis):
            raise ValueError("augmenter axis %r: entries must be axes of the %d-D patch" % (self.axis, nd))
        norm = tuple(int(a) % nd for a in axis)
        if len(set(norm)) != len(norm):
            raise ValueError("augmenter axis %r: entries must be distinct axes" % (self.axis,))
        if len({patch_size[a] for a in norm}) > 1:
            raise ValueError("augmenter axis %r: the patch size %s differs along these axes, a permutation would change the patch "
                             "shape" % (self.axis, tuple(patch_size)))
        for name, v in (("scale", self.scale), ("shift", self.shift)):
            if len(v) != 2 or not all(isinstance(u, (int, float, np.integer, np.floating)) for u in v):
                raise ValueError("augmenter %s must be two numbers, got %r" % (name, v))
        if self.noise is not None and not (isinstance(self.noise, (int, float, np.integer, np.floating)) and self.noise >= 0):
            raise ValueError("augmenter noise must be None or a number >= 0, got %r" % (self.noise,))
        return norm

    def draw(self, axis, nd):
        """the scalar draws of one item from np.random -> (int64 parameter row of sdb_augment_batch, noise sigma or None); the
        Gaussian values follow, drawn by normal_device"""
        perm = np.random.permutation(axis)
        tr = np.arange(nd)
        for a, q in zip(axis, perm):
            tr[a] = q
        flips = [np.random.rand() > 0.5 for _ in axis]
        s = np.random.uniform(*self.scale)
        t = np.random.uniform(*self.shift)
        sig = None if self.noise is None else self.noise * np.random.uniform(0, 1)
        src, flip = [0, 1, 2], [0, 0, 0]
        for a in range(nd):
            src[3 - nd + a] = 3 - nd + int(tr[a])
        for a, f in zip(axis, flips):
            flip[3 - nd + a] = int(f)
        bits = lambda v: int(np.float32(v).view(np.int32))
        row = src + flip + [bits(s), bits(t), int(np.float64(0.0 if sig is None else sig).view(np.int64)), int(sig is not None), 0, 0]
        return row, sig


def normal_device(n, out=None):
    """np.random.normal(0, 1, n) as a CUDA float64 tensor, drawn on the device from the global np.random state, which is left as
    numpy would leave it (values within a few ulp of numpy's: the device's double log; the state identical)"""
    import torch
    lib = L.require_cuda()
    n = int(n)
    if out is None:
        out = torch.empty(n, dtype=torch.float64, device="cuda")
    name, key, pos, has_gauss, gauss = np.random.get_state()
    key = np.ascontiguousarray(key, np.uint32)
    key_out = np.empty(624, np.uint32)
    pos_o, hg_o, g_o = ctypes.c_int(0), ctypes.c_int(0), ctypes.c_double(0)
    L.check(lib.sdb_mt_normal(L.ptr(key), int(pos), int(has_gauss), float(gauss), n, L.ptr(out), L.ptr(key_out), ctypes.byref(pos_o),
                              ctypes.byref(hg_o), ctypes.byref(g_o), L.stream_ptr()))
    np.random.set_state((name, key_out, pos_o.value, hg_o.value, g_o.value))
    return out
