"""tests/golden/optimize.npz: the reference's own stardist.utils.optimize_threshold (utils.py:271-307) on the cases of
optimize_cases.py, for every nms_thresh: the sequence of evaluated (probe, value) pairs (cache misses, in call order, with the
probe's scalar type), opt.x and -opt.fun.  The model is a stand-in whose _instances_from_prediction is the reference class
method (model2d.py:512-563 / model3d.py:589-674) with the reference's compiled extensions (oracle/_ref); the 2-D painting's
skimage.draw.polygon is the oracle restatement (oracle/geom2d_np.py).  Run in the build container:
OMP_NUM_THREADS=1 python tests/golden/make_optimize.py"""
import os, sys, json, types
os.environ.setdefault("OMP_NUM_THREADS", "1")
import numpy as np
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import _refpkg, optimize_cases
sys.path.insert(0, _refpkg.ROOT)


def run(name, m2, m3, ru, rrays):
    ndim, grid, n_rays, Y, Yhat = optimize_cases.inputs(name)
    for prob, dist in Yhat:                     # tie-free scores above any bracket floor
        p = prob[prob > prob.max() / 4]
        assert len(np.unique(p)) == len(p), name
    if ndim == 2:
        cfg = m2.Config2D(n_rays=n_rays, grid=grid); cls = m2.StarDist2D
    else:
        cfg = m3.Config3D(rays=rrays.Rays_GoldenSpiral(n_rays), grid=grid); cls = m3.StarDist3D
    fake = types.SimpleNamespace(config=cfg, thresholds=types.SimpleNamespace(prob=0.5, nms=0.4))
    fake._instances_from_prediction = lambda *a, **k: cls._instances_from_prediction(fake, *a, **k)
    out = {}
    orig = ru.matching_dataset                  # the probe's value: the mean fn() takes of matching_dataset's accuracy
    for nms in optimize_cases.NMS_THRESHS:
        probes = []

        def inst(*a, **k):
            if not probes or probes[-1][1] is not None:      # first image of a new probe (the last one has its value)
                probes.append([None, None])
            t = k['prob_thresh']
            probes[-1][0] = [float(t), type(t).__name__]
            return cls._instances_from_prediction(fake, *a, **k)
        fake._instances_from_prediction = inst
        ru.matching_dataset = lambda Yt, Yp, thresh, **kw: _merge(probes, orig(Yt, Yp, thresh=thresh, **kw))
        try:
            x, v = ru.optimize_threshold(Y, Yhat, fake, nms, iou_threshs=list(optimize_cases.IOU_THRESHS), verbose=0)
        finally:
            ru.matching_dataset = orig
        out[str(nms)] = dict(probes=probes, x=float(x), x_type=type(x).__name__, value=float(v))
        print(name, nms, len(probes), x, v, flush=True)
    return out


def _merge(probes, st):
    probes[-1][1] = float(np.mean([s.accuracy for s in st]))
    return st


if __name__ == "__main__":
    from oracle import geom2d_np
    draw = _refpkg._Stub("skimage.draw"); draw.polygon = geom2d_np.polygon
    sys.modules["skimage.draw"] = draw
    m2, m3 = _refpkg.load_models()
    ru = _refpkg.load("stardist.utils")
    rrays = _refpkg.load("stardist.rays3d")
    res = {name: run(name, m2, m3, ru, rrays) for name in optimize_cases.CASES}
    np.savez_compressed(os.path.join(HERE, "optimize.npz"), results=np.frombuffer(json.dumps(res).encode(), np.uint8))
    print("wrote optimize.npz")
