"""Inputs of the optimize_threshold fixtures (make_optimize.py -> optimize.npz), regenerated from seeds by the tests:
synthetic label images with their ideal prob (edt) / dist (star distances) maps (oracle/synth.py), plus seeded noise so that
scores are tie-free and no polygon / polyhedron is lattice aligned."""
import numpy as np

NMS_THRESHS = (0.3, 0.5)
IOU_THRESHS = (0.3, 0.5, 0.7)
CASES = {
    # name: (ndim, grid, n_rays, n_images)
    "2d_grid1": (2, (1, 1), 32, 3),
    "2d_grid2": (2, (2, 2), 32, 3),
    "3d_r32": (3, (1, 1, 1), 32, 2),
    "3d_r96": (3, (1, 1, 1), 96, 2),
}


def _tie_free(prob):
    """move repeated float32 values up by ulps until every value of the map is distinct"""
    flat = prob.ravel().copy()
    order = np.argsort(flat, kind='stable')
    v = flat[order]
    for i in range(1, len(v)):
        if v[i] <= v[i - 1]:
            v[i] = np.nextafter(v[i - 1], np.float32(np.inf))
    flat[order] = v
    return flat.reshape(prob.shape)


def _noisy(rng, prob, dist):
    prob = _tie_free((0.9 * prob + rng.uniform(0, 0.05, prob.shape)).astype(np.float32))
    dist = np.maximum(1e-3, dist + rng.uniform(-0.3, 0.3, dist.shape)).astype(np.float32)
    return prob, dist


def inputs(name):
    """-> (ndim, grid, n_rays, Y [label images], Yhat [(prob, dist)]) with prob / dist as predict() returns them"""
    from oracle import synth
    ndim, grid, n_rays, n_images = CASES[name]
    rng = np.random.default_rng(sorted(CASES).index(name) + 11)
    Y, Yhat = [], []
    for s in range(n_images):
        if ndim == 2:
            lbl = synth.ellipse_labels((128, 160), seed=s)
            prob, dist = synth.edt_prob(lbl), synth.star_dist(lbl, n_rays)
        else:
            from stardist_b200.rays3d import Rays_GoldenSpiral
            lbl = synth.ellipsoid_labels((24, 40, 40), seed=s)
            prob, dist = synth.edt_prob(lbl), synth.star_dist3d(lbl, Rays_GoldenSpiral(n_rays).vertices)
        sl = tuple(slice(None, None, g) for g in grid)
        prob, dist = _noisy(rng, prob[sl], dist[sl])
        Y.append(lbl.astype(np.int32)); Yhat.append((prob, dist))
    return ndim, grid, n_rays, Y, Yhat
