"""Cases of tests/golden/train_batch.npz (make_train_batch.py): the data, generator arguments, seed and batch indices of every
case.  Shared by the generator (which runs the reference's StarDistData2D / StarDistData3D) and the tests (which run
stardist_b200's).  Everything is built from fixed seeds; nothing here needs a GPU or the reference."""
import os
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))


def sha(a):
    import hashlib
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def _demo(name):
    z = np.load(os.path.join(HERE, name))
    return z['img'], z['mask']


def _crop(img, shape):
    return img[tuple(slice((s - m) // 2, (s - m) // 2 + m) for s, m in zip(img.shape, shape))]


def _blobs(shape, n, seed, lo=1, radius=(3, 9)):
    """label image of n random (possibly overlapping) discs / balls with labels lo, lo+1, ..."""
    rng = np.random.default_rng(seed)
    y = np.zeros(shape, np.int32)
    grid = np.indices(shape)
    for i in range(n):
        c = [rng.integers(0, s) for s in shape]
        r = rng.uniform(*radius)
        d = sum((g - cc) ** 2 for g, cc in zip(grid, c))
        y[d <= r * r] = lo + i
    return y


def _img(shape, seed, channels=None):
    rng = np.random.default_rng(seed)
    return rng.uniform(0, 1, shape + ((channels,) if channels else ())).astype(np.float32)


def flip_noise_augmenter(x, y):
    """flips both along a random axis and adds noise, all drawn from np.random"""
    ax = np.random.randint(0, y.ndim)
    x, y = np.flip(x, ax).copy(), np.flip(y, ax).copy()
    x = x + np.random.normal(0, 0.1, x.shape).astype(np.float32)
    return x, y


def cases():
    """name -> (dim, X list, Y list, kwargs, seed, batch indices)"""
    C = {}
    img, mask = _demo("demo2d.npz")
    img, mask = _crop(img, (256, 256)), _crop(mask, (256, 256))
    # the reference's own test (test_model2D.py::test_stardistdata, shape_completion False)
    for grid in ((1, 1), (1, 2), (2, 2)):
        for nc, cl in ((None, (1, 1)), (2, (1, 2))):
            tag = "demo2d_g%d%d_%s" % (grid + ("mc" if nc else "sc",))
            kw = dict(grid=grid, n_classes=nc, classes=cl, batch_size=2, n_rays=32, length=1, patch_size=(30, 41))
            C[tag] = (2, [img, img], [mask, mask], kw, 42, [0])
            m = mask[tuple(slice(0, (s // g) * g) for s, g in zip(mask.shape, grid))]
            im = img[tuple(slice(0, (s // g) * g) for s, g in zip(img.shape, grid))]
            ids = np.unique(m)[1:]
            neg = np.isin(m, ids[::2])
            mn = m.astype(np.int32)
            mn[neg] *= -1
            kw = dict(kw, patch_size=mn.shape)
            C[tag + "_neg"] = (2, [im, im], [mn, mn], kw, 42, [0])
    # sampling
    shapes = [(64, 80), (72, 64), (96, 96)]
    Y3 = [_blobs(s, 6, 10 + i) for i, s in enumerate(shapes)]
    X3 = [_img(s, 20 + i) for i, s in enumerate(shapes)]
    base = dict(n_rays=16, patch_size=(32, 32), grid=(1, 1))
    for fp in (0, 0.5, 1):
        C["fg%g" % fp] = (2, X3, Y3, dict(base, batch_size=3, length=4, foreground_prob=fp), 1, [0, 1, 2, 3])
    empty = [np.zeros((64, 64), np.int32), Y3[0]]
    C["fg1_empty"] = (2, [_img((64, 64), 3), X3[0]], empty, dict(base, batch_size=2, length=3, foreground_prob=1), 2, [0, 1, 2])
    C["maxfilter"] = (2, X3, Y3, dict(base, batch_size=3, length=2, foreground_prob=1, maxfilter_patch_size=(9, 4)), 3, [0, 1])
    C["odd_patch"] = (2, X3, Y3, dict(base, patch_size=(31, 27), batch_size=2, length=3, foreground_prob=0.7), 4, [0, 1, 2])
    C["not_divisible"] = (2, X3, Y3, dict(base, patch_size=(30, 27), grid=(2, 4), batch_size=2, length=2, foreground_prob=0.5), 5, [0, 1])
    # stream: batches wrapping more than one pass over 3 images of different shapes
    for bs in (1, 3, 5):
        for cache in (True, False):
            C["stream_b%d_%s" % (bs, "cache" if cache else "nocache")] = (
                2, X3, Y3, dict(base, batch_size=bs, length=5, foreground_prob=0.5, sample_ind_cache=cache), 6 + bs, [0, 1, 2, 3, 4])
    # inputs
    C["x2ch"] = (2, [_img(s, 30 + i, 2) for i, s in enumerate(shapes)], Y3, dict(base, batch_size=2, length=2), 7, [0, 1])
    C["x3ch"] = (2, [_img(s, 40 + i, 3) for i, s in enumerate(shapes)], Y3, dict(base, batch_size=2, length=2, grid=(2, 2)), 8, [0, 1])
    y8 = [(_blobs(s, 6, 50 + i) * np.where(np.arange(s[1]) % 3 == 0, -1, 1)).astype(np.int8) for i, s in enumerate(shapes)]
    C["int8_negative"] = (2, X3, y8, dict(base, batch_size=3, length=2, grid=(2, 1), foreground_prob=0.5), 9, [0, 1])
    ybig = [np.where(y > 0, y + 65535 * (y % 2), 0).astype(np.int32) for y in Y3]
    C["labels_65536"] = (2, X3, ybig, dict(base, batch_size=3, length=2), 10, [0, 1])
    C["augmenter"] = (2, X3, Y3, dict(base, batch_size=3, length=2, augmenter=flip_noise_augmenter, foreground_prob=0.5,
                                      n_classes=2, classes=[{i: 1 + i % 2 for i in range(1, 7)}] * 3), 11, [0, 1])
    # constant patches: one label filling the patch, and no label at all
    yc = np.zeros((40, 40), np.int32); yc[5:35, 5:35] = 7
    C["constant"] = (2, [_img((40, 40), 12)] * 2, [yc, np.zeros((40, 40), np.int32)], dict(n_rays=8, patch_size=(20, 20), batch_size=2,
                                                                                          length=3), 12, [0, 1, 2])
    # multi-class
    dicts = [{i: (None if i % 3 == 0 else (0 if i % 3 == 1 else 1 + i % 2)) for i in range(1, 7)} for _ in range(3)]
    C["classes_dict"] = (2, X3, Y3, dict(base, batch_size=3, length=2, n_classes=2, classes=dicts, grid=(2, 2)), 13, [0, 1])
    C["classes_none"] = (2, X3, Y3, dict(base, batch_size=3, length=2, n_classes=3, classes=None, grid=(1, 2)), 14, [0, 1])
    # 3-D
    img3, mask3 = _demo("demo3d.npz")
    for bs in (1, 2):
        for grid in ((1, 1, 1), (1, 2, 2)):
            for nc, cl in ((None, (1, 1)), (2, (1, 2))):
                tag = "demo3d_b%d_g%d%d%d_%s" % ((bs,) + grid + ("mc" if nc else "sc",))
                kw = dict(grid=grid, n_classes=nc, classes=cl, batch_size=bs, rays=("golden", 64), length=1, patch_size=(30, 40, 50))
                C[tag] = (3, [img3, img3], [mask3, mask3], kw, 42, [0])
    s3 = [(24, 40, 36), (20, 36, 40)]
    Y33 = [_blobs(s, 8, 60 + i, radius=(3, 7)) for i, s in enumerate(s3)]
    X33 = [_img(s, 70 + i) for i, s in enumerate(s3)]
    for an in (None, (2, 1, 1), (1.7, 1, 1)):
        for grid in ((1, 2, 2), (2, 2, 2)):
            tag = "vol_%s_g%d%d%d" % (("iso" if an is None else "a%g" % an[0],) + grid)
            C[tag] = (3, X33, Y33, dict(rays=("golden", 96), grid=grid, anisotropy=an, patch_size=(16, 32, 32), batch_size=2, length=2,
                                        foreground_prob=0.5), 15, [0, 1])
    C["vol_classes"] = (3, X33, [(y * np.where(np.arange(y.shape[2]) % 5 == 0, -1, 1)).astype(np.int16) for y in Y33],
                        dict(rays=("golden", 96), grid=(1, 2, 2), patch_size=(16, 32, 32), batch_size=2, length=2, n_classes=2,
                             classes=[{i: 1 + i % 2 for i in range(1, 9)}] * 2), 16, [0, 1])
    return C


def ulp_cases():
    """cases whose edt_prob may differ by one float32 ulp (non-dyadic anisotropy): their prob is stored as an array"""
    return [k for k in cases() if k.startswith("vol_a1.7")]


def make_kwargs(kw, rays_cls):
    """kwargs with ('golden', n) replaced by rays_cls(n)"""
    kw = dict(kw)
    if "rays" in kw:
        kw["rays"] = rays_cls(kw["rays"][1])
    return kw
