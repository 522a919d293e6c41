"""Cases of tests/golden/augment.npz (make_augment.py): training batches with the notebooks' augmenter.  Per case: the data and
generator arguments (as train_batch_cases.cases()), the seed, the batch indices, the stardist_b200 Augmenter arguments and which
notebook augmenter the reference run composes ('2d': examples/2D/2_training.ipynb's augmenter, '3d': the 3-D notebook's,
'3d_noise': the 3-D notebook's random_fliprot(axis=(1, 2)) and random_intensity_change followed by the 2-D notebook's noise).
Everything is built from fixed seeds; nothing here needs a GPU or the reference."""
import numpy as np
import train_batch_cases as T

sha = T.sha


def cases():
    """name -> (dim, X, Y, generator kwargs, seed, batch indices, Augmenter kwargs, notebook augmenter)"""
    C = {}
    shapes = [(64, 80), (72, 64), (96, 96)]
    Y = [T._blobs(s, 6, 10 + i) for i, s in enumerate(shapes)]
    X = [T._img(s, 20 + i) for i, s in enumerate(shapes)]
    base = dict(n_rays=16, grid=(1, 1), batch_size=3, length=3, foreground_prob=0.5)
    nb2d = dict()
    C["nb2d_square"] = (2, X, Y, dict(base, patch_size=(32, 32)), 101, [0, 1, 2], nb2d, "2d")
    # 33 x 33 values per item: odd, so the Gaussian cache carries over from one item to the next
    C["nb2d_odd33"] = (2, X, Y, dict(base, patch_size=(33, 33)), 102, [0, 1, 2], nb2d, "2d")
    # two channels, grid (2, 2), negative labels
    y8 = [(T._blobs(s, 6, 50 + i) * np.where(np.arange(s[1]) % 3 == 0, -1, 1)).astype(np.int8) for i, s in enumerate(shapes)]
    X2 = [T._img(s, 30 + i, 2) for i, s in enumerate(shapes)]
    C["nb2d_x2ch_g22_neg"] = (2, X2, y8, dict(base, patch_size=(32, 32), grid=(2, 2)), 103, [0, 1], nb2d, "2d")
    # multi-class with class dicts (None, 0 and real classes)
    dicts = [{i: (None if i % 3 == 0 else (0 if i % 3 == 1 else 1 + i % 2)) for i in range(1, 7)} for _ in range(3)]
    C["nb2d_classes"] = (2, X, Y, dict(base, patch_size=(32, 32), n_classes=2, classes=dicts, grid=(2, 2)), 104, [0, 1], nb2d, "2d")
    # 3-D
    s3 = [(24, 40, 36), (20, 36, 40)]
    Y3 = [T._blobs(s, 8, 60 + i, radius=(3, 7)) for i, s in enumerate(s3)]
    X3 = [T._img(s, 70 + i) for i, s in enumerate(s3)]
    b3 = dict(rays=("golden", 96), grid=(1, 2, 2), anisotropy=(2, 1, 1), patch_size=(16, 32, 32), batch_size=2, length=2,
              foreground_prob=0.5)
    C["nb3d"] = (3, X3, Y3, b3, 105, [0, 1], dict(axis=(1, 2), noise=None), "3d")
    C["nb3d_noise"] = (3, X3, Y3, dict(b3, anisotropy=None), 106, [0, 1], dict(axis=(1, 2)), "3d_noise")
    return C
