"""Per-batch time of the training-batch generators: one JSON line.

Device-resident ms per batch (batch_device, CUDA events) and host-to-host ms per batch (__getitem__), medians after
warm-up, for the 2-D workload (32 images of 1024^2, batch 8 x 256^2, 32 rays, grid (2,2), foreground_prob 0.9) and the 3-D
workload (4 volumes of 128x256x256, batch 2 x 64x128x128, 96 rays, grid (1,2,2), anisotropy (2,1,1)); and, where
oracle/_ref holds the reference's compiled extension, the reference's per-batch targets on the host (its c_star_dist /
c_star_dist3d at the best of the thread counts tried plus the scipy edt_prob restatement of tests/labelprep_emu.py) on
the same patches.
Usage: python tests/tools/train_batch_bench.py [--iters 20] [--skip-ref]"""
import argparse, json, os, subprocess, sys, time
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, power = [s.strip() for s in r.stdout.strip().splitlines()[0].split(",")]
        return name, power
    except Exception:
        return None, None


def timed(gen, iters, warmup, device):
    import torch
    ts = []
    for i in range(warmup + iters):
        if device:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            gen.batch_device(i)
            b.record()
            b.synchronize()
            t = a.elapsed_time(b)
        else:
            t0 = time.perf_counter()
            gen[i]
            t = (time.perf_counter() - t0) * 1e3
        if i >= warmup:
            ts.append(t)
    return float(np.median(ts))


def reference_ms(gen, Y, dim, iters):
    """(ms, threads): the reference's per-batch targets on the host (c_star_dist / c_star_dist3d at the best of the thread
    counts tried, plus the per-object scipy edt_prob of labelprep_emu) on `iters` patch sets drawn by the generator"""
    import ctypes
    from oracle import ref_ext
    import labelprep_emu as E
    gomp = ctypes.CDLL("libgomp.so.1")
    mod = ref_ext.stardist2d() if dim == 2 else ref_ext.stardist3d()
    patches = []
    for i in range(iters):
        gen.batch_device(1000 + i)
        pos = gen.last_positions.cpu().numpy()
        patches.append([np.maximum(Y[k][tuple(slice(r - p // 2, r - p // 2 + p) for r, p in zip(pos[b], gen.patch_size))], 0)
                        for b, k in enumerate(gen.last_index)])
    tab = None if dim == 2 else [np.ascontiguousarray(v) for v in np.asarray(gen.rays.vertices).T.astype(np.float32)]
    res = {}
    for threads in (1, 4, 16, 32):
        if threads > os.cpu_count():
            continue
        gomp.omp_set_num_threads(threads)
        ts = []
        for ps in patches:
            t0 = time.perf_counter()
            for y in ps:
                if dim == 2:
                    mod.c_star_dist(y.astype(np.uint16), gen.n_rays, *gen.grid)
                    E.edt_prob_boxes(y[gen.ss_grid[1:]])
                else:
                    mod.c_star_dist3d(y.astype(np.uint16), *tab, len(gen.rays), *gen.grid)
                    E.edt_prob_boxes(y, gen.anisotropy)[gen.ss_grid[1:]]
            ts.append((time.perf_counter() - t0) * 1e3)
        res[threads] = float(np.median(ts))
    best = min(res, key=res.get)
    return res[best], best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--skip-ref", action="store_true")
    a = ap.parse_args()
    import bench_data
    from stardist_b200.models import StarDistData2D, StarDistData3D
    from stardist_b200.rays3d import Rays_GoldenSpiral
    name, power = gpu_info()
    out = {"gpu": name, "power_limit": power}
    np.random.seed(0)
    X2, Y2 = zip(*[bench_data.synthetic_image((1024, 1024), seed=s) for s in range(32)])
    X2, Y2 = list(X2), list(Y2)
    g2 = StarDistData2D(X2, Y2, batch_size=8, n_rays=32, length=10 ** 6, patch_size=(256, 256), grid=(2, 2), foreground_prob=0.9)
    out["2d_device_ms"] = timed(g2, a.iters, a.warmup, True)
    out["2d_host_ms"] = timed(g2, a.iters, a.warmup, False)
    Y3 = [bench_data.ellipsoid_labels((128, 256, 256), seed=s) for s in range(4)]
    X3 = [y.astype(np.float32) for y in Y3]
    g3 = StarDistData3D(X3, Y3, batch_size=2, rays=Rays_GoldenSpiral(96), length=10 ** 6, patch_size=(64, 128, 128), grid=(1, 2, 2),
                        anisotropy=(2, 1, 1))
    out["3d_device_ms"] = timed(g3, a.iters, a.warmup, True)
    out["3d_host_ms"] = timed(g3, a.iters, a.warmup, False)
    if not a.skip_ref and os.path.isdir(os.path.join(ROOT, "oracle", "_ref")):
        out["2d_reference_ms"], out["2d_reference_threads"] = reference_ms(g2, Y2, 2, 5)
        out["3d_reference_ms"], out["3d_reference_threads"] = reference_ms(g3, Y3, 3, 2)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
