"""Seeded label maps and ray sets of the star-distance fixtures (tests/golden/star_dist.npz, make_star_dist.py) and tests."""
import os
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))


def ellipses_2d(shape=(64, 80), n=9, seed=0):
    """n seeded ellipses with non-sequential labels, later ones painted over earlier ones"""
    rng = np.random.default_rng(seed)
    lbl = np.zeros(shape, np.int32)
    yy, xx = np.indices(shape)
    labels = rng.choice(np.arange(1, 1000), n, replace=False)
    for l in labels:
        cy, cx = rng.uniform(0, shape[0]), rng.uniform(0, shape[1])
        ry, rx = rng.uniform(3, 12, 2)
        t = rng.uniform(0, np.pi)
        u = (yy - cy) * np.cos(t) + (xx - cx) * np.sin(t)
        v = -(yy - cy) * np.sin(t) + (xx - cx) * np.cos(t)
        lbl[(u / ry) ** 2 + (v / rx) ** 2 <= 1] = l
    return lbl


def ellipsoids_3d(shape=(24, 40, 44), n=7, seed=0):
    rng = np.random.default_rng(seed)
    lbl = np.zeros(shape, np.int32)
    zz, yy, xx = np.indices(shape)
    for l in rng.choice(np.arange(1, 500), n, replace=False):
        c = [rng.uniform(0, s) for s in shape]
        r = rng.uniform(3, 9, 3)
        lbl[((zz - c[0]) / r[0]) ** 2 + ((yy - c[1]) / r[1]) ** 2 + ((xx - c[2]) / r[2]) ** 2 <= 1] = l
    return lbl


def border_2d():
    """objects touching each of the four borders and the corners, odd shape"""
    lbl = np.zeros((37, 41), np.int32)
    lbl[:6, 5:30] = 3; lbl[-4:, :] = 7; lbl[8:20, :5] = 2; lbl[10:25, -9:] = 11; lbl[:3, :3] = 5; lbl[15:22, 15:26] = 4
    return lbl


def border_3d():
    lbl = np.zeros((13, 17, 19), np.int32)
    lbl[:3, :, :] = 2; lbl[5:9, :6, 4:12] = 4; lbl[4:, 10:, -5:] = 9; lbl[-2:, 3:8, :4] = 1
    return lbl


def singles_2d():
    rng = np.random.default_rng(3)
    lbl = np.zeros((20, 23), np.int32)
    idx = rng.choice(lbl.size, 25, replace=False)
    lbl.flat[idx] = np.arange(1, 26)
    return lbl


def singles_3d():
    rng = np.random.default_rng(4)
    lbl = np.zeros((9, 10, 11), np.int32)
    lbl.flat[rng.choice(lbl.size, 20, replace=False)] = np.arange(1, 21)
    return lbl


def big_labels(lbl):
    """labels >= 65536 whose low 16 bits collide with each other (the reference compares uint16)"""
    out = lbl.astype(np.int64)
    u = np.unique(out[out > 0])
    remap = {int(l): 65536 * (1 + i % 3) + int(l) % 7 for i, l in enumerate(u)}
    for l, m in remap.items():
        out[lbl == l] = m
    return out


def negative_int8(lbl):
    """int8 map with negative values (the reference's astype(np.uint16) wraps them)"""
    out = (lbl % 200).astype(np.int16) - 100
    out[lbl == 0] = 0
    return out.astype(np.int8)


def demo_mask():
    return np.load(os.path.join(HERE, "demo2d.npz"))["mask"]


def maps_2d():
    e = ellipses_2d()
    return {"demo": demo_mask(), "ellipses": e, "ellipses_odd": ellipses_2d((31, 45), 5, seed=1), "border": border_2d(),
            "singles": singles_2d(), "empty": np.zeros((16, 16), np.int32), "constant": np.full((15, 17), 5, np.int32),
            "big_labels": big_labels(e), "int8_negative": negative_int8(e)}


def maps_3d():
    e = ellipsoids_3d()
    return {"ellipsoids": e, "border": border_3d(), "singles": singles_3d(), "empty": np.zeros((6, 7, 8), np.int32),
            "constant": np.full((5, 6, 7), 3, np.int32), "big_labels": big_labels(e), "int8_negative": negative_int8(e)}


GRIDS_2D = ((1, 1), (2, 4), (3, 1))
GRIDS_3D = ((1, 1, 1), (2, 2, 2), (1, 2, 4))


def ray_sets():
    """name -> product Rays object (vertices equal to the reference's rays3d.py, see make_rays3d.py)"""
    from stardist_b200.rays3d import Rays_GoldenSpiral, Rays_Octo, Rays_Tetra, Rays_Cartesian, Rays_Explicit
    gs = Rays_GoldenSpiral(20)
    return {"gs32": Rays_GoldenSpiral(32), "gs96": Rays_GoldenSpiral(96), "gs32_aniso": Rays_GoldenSpiral(32, anisotropy=(2, 1, 1)),
            "gs96_aniso": Rays_GoldenSpiral(96, anisotropy=(1, 1.5, 3)), "octo": Rays_Octo(1), "tetra": Rays_Tetra(2),
            "cartesian": Rays_Cartesian(), "explicit": Rays_Explicit(gs.vertices, gs.faces)}


def sha(a):
    import hashlib
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()
