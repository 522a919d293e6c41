"""Timing of the star-distance kernels and the relabel functions (CUDA events, medians), against the reference's C++
(oracle/_ref c_star_dist / c_star_dist3d) on the host cores at the best thread count of a sweep.

    python tests/tools/star_dist_bench.py [--reps 5] [--json out.json]

Maps: the benchmark's 1024^2 ground truth (bench_data.ellipse_labels) with 32 rays; ellipsoid volumes
(bench_data.ellipsoid_labels) with 96 golden-spiral rays, 128x512x512 device-resident (12.9 GB of output) and 64x256x256
host to host.  The dense kernels are compared with their HBM write floor (output bytes / 3.35 TB/s, H100 SXM data sheet)."""
import argparse, ctypes, json, os, subprocess, sys, time
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
HBM_BPS = 3.35e12


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
        return q.stdout.strip().splitlines()[0]
    except Exception:
        return "unknown"


def cuda_median(fn, reps):
    import torch
    fn(); torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def wall_median(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t = time.perf_counter(); fn(); ts.append((time.perf_counter() - t) * 1e3)
    return float(np.median(ts))


def cpu_sweep(fn, reps):
    """reference C++ at every thread count of the sweep; returns (best ms, threads, all)"""
    gomp = ctypes.CDLL("libgomp.so.1")
    res = {}
    for t in (1, 4, 8, 16, 32, 64, os.cpu_count()):
        if t > os.cpu_count() or t in res: continue
        gomp.omp_set_num_threads(t)
        res[t] = wall_median(fn, max(1, reps // 2))
    best = min(res, key=res.get)
    return res[best], best, res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json", default=None)
    ap.add_argument("--no-cpu", action="store_true")
    a = ap.parse_args()
    import torch
    import bench_data
    import stardist_b200 as sd
    from stardist_b200.geometry.distances import star_dist_device, star_dist3D_device
    from oracle import ref_ext
    out = {"gpu": gpu_info(), "reps": a.reps}
    rays = sd.Rays_GoldenSpiral(96)
    lbl2 = bench_data.ellipse_labels((1024, 1024), seed=0)
    d2 = torch.from_numpy(lbl2).cuda()
    ms = cuda_median(lambda: star_dist_device(d2, 32), a.reps)
    out["star_dist_2d_1024_r32_device_ms"] = ms
    out["star_dist_2d_1024_r32_floor_ms"] = 1024 * 1024 * 32 * 4 / HBM_BPS * 1e3
    out["star_dist_2d_1024_r32_host_ms"] = wall_median(lambda: sd.star_dist(lbl2, 32), a.reps)
    out["relabel_2d_1024_r32_ms"] = wall_median(lambda: sd.relabel_image_stardist(lbl2, 32), a.reps)
    vol_big = bench_data.ellipsoid_labels((128, 512, 512), seed=0)
    d3 = torch.from_numpy(vol_big).cuda()
    del vol_big
    res = [None]

    def big():
        res[0] = None
        res[0] = star_dist3D_device(d3, rays)
    out["star_dist_3d_128x512x512_r96_device_ms"] = cuda_median(big, a.reps)
    out["star_dist_3d_128x512x512_r96_floor_ms"] = 128 * 512 * 512 * 96 * 4 / HBM_BPS * 1e3
    res[0] = None; del d3; torch.cuda.empty_cache()
    vol = bench_data.ellipsoid_labels((64, 256, 256), seed=0)
    out["star_dist_3d_64x256x256_r96_host_ms"] = wall_median(lambda: sd.star_dist3D(vol, rays), a.reps)
    out["relabel_3d_64x256x256_r96_ms"] = wall_median(lambda: sd.relabel_image_stardist3D(vol, rays), a.reps)
    if not a.no_cpu and ref_ext.available():
        r2, r3 = ref_ext.stardist2d(), ref_ext.stardist3d()
        u2 = lbl2.astype(np.uint16)
        ms, t, allr = cpu_sweep(lambda: r2.c_star_dist(u2, 32, 1, 1), a.reps)
        out["ref_cpu_star_dist_2d_1024_r32_ms"] = ms; out["ref_cpu_2d_threads"] = t; out["ref_cpu_2d_sweep"] = allr
        u3 = vol.astype(np.uint16)
        tab = [np.ascontiguousarray(x) for x in np.asarray(rays.vertices).T.astype(np.float32)]
        ms, t, allr = cpu_sweep(lambda: r3.c_star_dist3d(u3, *tab, 96, 1, 1, 1), a.reps)
        out["ref_cpu_star_dist_3d_64x256x256_r96_ms"] = ms; out["ref_cpu_3d_threads"] = t; out["ref_cpu_3d_sweep"] = allr
    print(json.dumps(out, indent=1))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
