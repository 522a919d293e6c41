"""Cost of the map-wide helpers: one JSON line.

For each helper, medians after warm-up of
- `*_device_ms`: CUDA events around the call on device-resident input (CUDA tensors in, CUDA tensors / host results out);
- `*_host_ms`: host clock around the call on numpy input, numpy out (uploads and downloads included);
- `*_floor_ms`: the bytes the kernels must move (from the shapes) over the H100 SXM data-sheet HBM3 bandwidth, 3.35 TB/s.
Cases:
- dist_to_volume / dist_to_centroid on a random 64x256x256x96 map (Rays_GoldenSpiral(96)), and the reference extension's
  c_dist_to_volume / c_dist_to_centroid (oracle/_ref, OpenMP) on the host cores at 1, n/4, n/2 and n threads (`ref_*`, each
  in its own process, one call each);
- mask_to_categorical on the 1024^2 benchmark ground truth with 3 classes (random dict classes);
- sample_points(200, prob > 0.2, prob=prob) on a 1024^2 device predict (default Config2D, 32 rays, seeded weights).
Usage: python tests/tools/helpers_bench.py [--iters 20] [--warmup 3]"""
import argparse, json, os, subprocess, sys, time
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from train_step_bench import gpu_info

HBM = 3.35e12
DIST_SHAPE = (64, 256, 256, 96)


def dist_map():
    return np.random.default_rng(0).uniform(0.5, 12, DIST_SHAPE).astype(np.float32)


def device_ms(fn, iters, warmup):
    import torch
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def host_ms(fn, iters, warmup):
    import torch
    ts = []
    for i in range(warmup + iters):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        if i >= warmup:
            ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


def ref_child(what):
    """one timed reference call, in a process whose OMP_NUM_THREADS was set before the extension loaded"""
    from oracle import ref_ext
    from stardist_b200.rays3d import Rays_GoldenSpiral
    rays = Rays_GoldenSpiral(96)
    v = np.ascontiguousarray(rays.vertices, np.float32); f = np.ascontiguousarray(rays.faces, np.int32)
    d = dist_map()
    ext = ref_ext.stardist3d()
    t0 = time.perf_counter()
    ext.c_dist_to_volume(d, v, f) if what == "volume" else ext.c_dist_to_centroid(d, v, f, np.int32(1))
    print(json.dumps((time.perf_counter() - t0) * 1e3))


def ref_times(what):
    n = os.cpu_count() or 1
    out = {}
    for t in sorted({1, max(1, n // 4), max(1, n // 2), n}):
        env = dict(os.environ, OMP_NUM_THREADS=str(t))
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--ref-child", what], capture_output=True, text=True, env=env)
        out[t] = json.loads(r.stdout.strip().splitlines()[-1]) if r.returncode == 0 else None
    ok = {t: ms for t, ms in out.items() if ms is not None}
    best = min(ok, key=ok.get) if ok else None
    return {"ref_%s_ms_by_threads" % what: out, "ref_%s_best_ms" % what: ok.get(best), "ref_%s_best_threads" % what: best}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--ref-child", default=None)
    a = ap.parse_args()
    if a.ref_child:
        return ref_child(a.ref_child)
    import torch
    import bench_data
    from stardist_b200 import Config2D, StarDist2D
    from stardist_b200.geometry.geom3d import dist_to_volume, dist_to_centroid
    from stardist_b200.rays3d import Rays_GoldenSpiral
    from stardist_b200.utils import mask_to_categorical, sample_points
    out = {"gpu": gpu_info(), "host_cores": os.cpu_count()}

    rays = Rays_GoldenSpiral(96)
    d = dist_map()
    d_t = torch.from_numpy(d).cuda()
    n_vox = int(np.prod(DIST_SHAPE[:3]))
    out["volume_device_ms"] = device_ms(lambda: dist_to_volume(d_t, rays), a.iters, a.warmup)
    out["centroid_device_ms"] = device_ms(lambda: dist_to_centroid(d_t, rays), a.iters, a.warmup)
    out["volume_host_ms"] = host_ms(lambda: dist_to_volume(d, rays), max(3, a.iters // 4), 1)
    out["centroid_host_ms"] = host_ms(lambda: dist_to_centroid(d, rays), max(3, a.iters // 4), 1)
    out["volume_floor_ms"] = (d.nbytes + 4 * n_vox) / HBM * 1e3
    out["centroid_floor_ms"] = (d.nbytes + 12 * n_vox) / HBM * 1e3
    out["poly_faces"] = int(len(rays.faces))
    del d_t
    out.update(ref_times("volume"))
    out.update(ref_times("centroid"))

    _, y = bench_data.synthetic_image((1024, 1024), seed=0)
    labels = np.unique(y[y > 0])
    rng = np.random.default_rng(0)
    cls = {int(l): [None, 1, 2, 3][int(c)] for l, c in zip(labels, rng.integers(0, 4, len(labels)))}
    y_t = torch.from_numpy(np.ascontiguousarray(y, np.int32)).cuda()
    out["m2c_objects"] = int(len(labels))
    out["m2c_device_ms"] = device_ms(lambda: mask_to_categorical(y_t, 3, cls), a.iters, a.warmup)
    out["m2c_host_ms"] = host_ms(lambda: mask_to_categorical(y, 3, cls), a.iters, a.warmup)
    out["m2c_floor_ms"] = (4 * y.size + 4 * 4 * y.size) / HBM * 1e3

    model = StarDist2D(Config2D(n_rays=32), name=None, basedir=None)
    model.weights = bench_data.bench_weights_2d(model.config); model._net = None
    img, _ = bench_data.synthetic_image((1024, 1024), seed=0)
    prob_t = model._predict_device(img)[0].contiguous()
    prob = prob_t.cpu().numpy()
    mask_t = prob_t > 0.2
    out["sp_candidates"] = int((prob[2:-2, 2:-2] > 0.2).sum())
    out["sp_device_ms"] = device_ms(lambda: sample_points(200, mask_t, prob=prob_t), a.iters, a.warmup)
    out["sp_host_ms"] = host_ms(lambda: sample_points(200, prob > 0.2, prob=prob), a.iters, a.warmup)
    out["sp_floor_ms"] = (mask_t.numel() + 4 * out["sp_candidates"] * 3) / HBM * 1e3
    print(json.dumps(out))


if __name__ == "__main__":
    main()
