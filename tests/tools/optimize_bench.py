"""Timing of optimize_thresholds and of the label-overlap kernel; prints one JSON line.

* optimize_thresholds on the shipped 2D_demo model (its test image tiled 4x4, its mask as ground truth) and on 3D_demo (its
  volume tiled 2x2 in y / x): the threshold engine (utils.optimize_threshold) against the reference's per-probe loop over
  _instances_from_prediction + matching_dataset, on the same device maps, alternating, with the default search settings.
* sdb_label_overlap at 1024^2 and 128x512^2 (blob label maps): CUDA-event time and bytes/s (8 B read per pixel) against the
  3.35 TB/s of the H100 SXM data sheet.
The GPU name and power limit are read in the same run.  Usage: python tests/tools/optimize_bench.py [--reps N]"""
import os, sys, json, time, argparse, subprocess
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))


def loop_optimize(model, Y, Yhat, nms_thresh, iou_threshs, tol=1e-2, maxiter=20):
    """stardist/utils.py:271-307 with each value computed from scratch (public functions, host maps)"""
    from scipy.optimize import minimize_scalar
    from stardist_b200.matching import matching_dataset
    values = {}
    max_prob = max([np.max(p) for p, d in Yhat])
    bracket = max_prob / 2, max_prob

    def fn(thr):
        t = np.clip(thr, *bracket)
        v = values.get(t)
        if v is None:
            inst = [model._instances_from_prediction(y.shape, *pd, prob_thresh=t, nms_thresh=nms_thresh)[0] for y, pd in zip(Y, Yhat)]
            v = values[t] = np.mean([s.accuracy for s in matching_dataset(Y, inst, thresh=iou_threshs, show_progress=False)])
        return -v
    opt = minimize_scalar(fn, method='golden', bracket=bracket, tol=tol, options={'maxiter': maxiter})
    return opt.x, -opt.fun


def time_case(model, Y, Yhat_dev, reps, nms_threshs=(0.3, 0.4, 0.5), iou_threshs=(0.3, 0.5, 0.7)):
    import torch
    from stardist_b200.utils import optimize_threshold
    Yhat_host = [tuple(m.cpu().numpy() for m in pd) for pd in Yhat_dev]
    te, tl, same = [], [], True
    for _ in range(reps):
        for which in ("engine", "loop"):
            torch.cuda.synchronize(); t0 = time.perf_counter()
            if which == "engine":
                r = [optimize_threshold(Y, Yhat_dev, model, n, iou_threshs=list(iou_threshs), verbose=0) for n in nms_threshs]
            else:
                r2 = [loop_optimize(model, Y, Yhat_host, n, list(iou_threshs)) for n in nms_threshs]
            torch.cuda.synchronize(); (te if which == "engine" else tl).append(time.perf_counter() - t0)
        same = same and [tuple(map(float, a)) for a in r] == [tuple(map(float, b)) for b in r2]
    return dict(engine_s=float(np.median(te)), loop_s=float(np.median(tl)), engine_all=te, loop_all=tl, same_optimum=bool(same))


def overlap_kernel(shape, reps):
    import torch
    from oracle import synth
    from stardist_b200.matching import label_overlap_device
    rng = np.random.default_rng(0)
    base = synth.ellipse_labels((1024, 1024), seed=0) if len(shape) == 2 else synth.ellipsoid_labels((128, 128, 128), seed=0)
    a = base if len(shape) == 2 else np.tile(base, (1, 4, 4))
    b = np.roll(a, 3, axis=-1)
    assert a.shape == tuple(shape)
    da = torch.from_numpy(np.ascontiguousarray(a, np.int32)).cuda(); db = torch.from_numpy(np.ascontiguousarray(b, np.int32)).cuda()
    for _ in range(3): label_overlap_device(da, db)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps): label_overlap_device(da, db)
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    nbytes = 8 * a.size
    return dict(shape=list(shape), ms=ms, gb_per_s=nbytes / ms / 1e6, share_of_3_35_tb_s=nbytes / ms / 1e6 / 3350.0)


def tile_labels(m, reps):
    """np.tile of a label image with the ids of every copy offset, so that copies stay distinct objects"""
    t = np.tile(m.astype(np.int64), reps)
    k = np.zeros(t.shape, np.int64)
    for a, (g, r) in enumerate(zip(np.indices(t.shape), reps)):
        k = k * r + g // m.shape[a]
    return np.where(t > 0, t + k * int(m.max()), 0).astype(np.int32)


def main():
    ap = argparse.ArgumentParser(); ap.add_argument("--reps", type=int, default=3); args = ap.parse_args()
    import torch
    import stardist_b200 as sd
    import demo2d
    from stardist_b200.utils import normalize
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    out = dict(gpu=q)
    kwargs, weights, thr, img, mask = demo2d.load()
    m2 = sd.StarDist2D(sd.Config2D(**kwargs), name=None, basedir=None, weights=weights)
    x2, y2 = normalize(np.tile(img, (4, 4)), 1, 99.8), tile_labels(mask, (4, 4))
    out["2d_demo_4x4"] = time_case(m2, [y2], [m2._predict_device(x2)[:2]], args.reps)
    import demo3d
    from stardist_b200.rays3d import rays_from_json
    rays_json, kwargs, weights, thr, img, mask = demo3d.load()
    m3 = sd.StarDist3D(sd.Config3D(rays=rays_from_json(rays_json), **kwargs), name=None, basedir=None, weights=weights)
    x3, y3 = normalize(np.tile(img, (1, 2, 2)), 1, 99.8), tile_labels(mask, (1, 2, 2))
    out["3d_demo_1x2x2"] = time_case(m3, [y3], [m3._predict_device(x3)[:2]], args.reps)
    out["overlap_1024x1024"] = overlap_kernel((1024, 1024), 50)
    out["overlap_128x512x512"] = overlap_kernel((128, 512, 512), 20)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
