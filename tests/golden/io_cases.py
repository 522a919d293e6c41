"""Seeded inputs of the ROI / OBJ writer comparisons (tests/test_io_cpu.py, tests/golden/make_io_ref.py)."""
import numpy as np

OBJ_KWARGS = (dict(), dict(single_mesh=False), dict(uv_map=True, scale=(2, 1, 0.5)), dict(scale=0.01))


def roi_cases():
    """(x, y, pos, subpixel) of 25 random polygons x 2 subpixel modes x 2 positions"""
    rng = np.random.default_rng(0)
    out = []
    for _ in range(25):
        n = int(rng.integers(3, 40)); xs = rng.uniform(-5, 300, n); ys = rng.uniform(0, 200, n)
        for sub in (True, False):
            for pos in (None, 3):
                out.append((xs, ys, pos, sub))
    return out


def obj_polys():
    """four polyhedra on a 12-ray golden spiral"""
    import stardist_b200 as sd
    rays = sd.Rays_GoldenSpiral(12)
    rng = np.random.default_rng(0)
    return dict(dist=rng.uniform(2, 6, (4, 12)).astype(np.float32), points=rng.integers(5, 40, (4, 3)),
                rays_vertices=rays.vertices, rays_faces=rays.faces)
