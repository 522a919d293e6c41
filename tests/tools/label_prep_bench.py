"""Timing of edt_prob and fill_label_holes (CUDA events, medians), device-resident and host to host, against the per-object
scipy computation of the reference restated in tests/labelprep_emu.py, run on the host cores.

    python tests/tools/label_prep_bench.py [--reps 5] [--json out.json] [--no-cpu]

Maps: the benchmark's 1024^2 ground truth (bench_data.ellipse_labels) and a 128x512x512 ellipsoid volume
(bench_data.ellipsoid_labels).  Each device time is compared with its bytes-moved floor at 3.35 TB/s (H100 SXM data sheet):
edt_prob reads the int32 map and writes float32 prob; fill_label_holes reads it and writes int32."""
import argparse, json, os, subprocess, sys, time
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
HBM_BPS = 3.35e12


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0]


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json", default=None)
    ap.add_argument("--no-cpu", action="store_true")
    a = ap.parse_args()
    import torch
    import bench_data
    import labelprep_emu as E
    import stardist_b200 as sd
    from stardist_b200.labelprep import edt_prob_device, fill_label_holes_device
    out = {"gpu": gpu_info(), "reps": a.reps}
    maps = {"2d_1024": lambda: bench_data.ellipse_labels((1024, 1024), seed=0),
            "3d_128x512x512": lambda: bench_data.ellipsoid_labels((128, 512, 512), seed=0)}
    for name, make in maps.items():
        lbl = make()
        d = torch.from_numpy(lbl).cuda()
        n = lbl.size
        out["n_labels_" + name] = int(len(np.unique(lbl)) - 1)
        out["edt_prob_%s_device_ms" % name] = cuda_median(lambda: edt_prob_device(d), a.reps)
        out["edt_prob_%s_floor_ms" % name] = n * 8 / HBM_BPS * 1e3
        out["edt_prob_%s_host_ms" % name] = wall_median(lambda: sd.edt_prob(lbl), a.reps)
        out["fill_label_holes_%s_device_ms" % name] = cuda_median(lambda: fill_label_holes_device(d), a.reps)
        out["fill_label_holes_%s_floor_ms" % name] = n * 8 / HBM_BPS * 1e3
        out["fill_label_holes_%s_host_ms" % name] = wall_median(lambda: sd.fill_label_holes(lbl), a.reps)
        if not a.no_cpu:
            reps = 1 if lbl.ndim == 3 else a.reps
            out["cpu_scipy_edt_prob_%s_ms" % name] = wall_median(lambda: E.edt_prob_boxes(lbl), reps)
            out["cpu_scipy_fill_label_holes_%s_ms" % name] = wall_median(lambda: E.fill_label_holes_def(lbl), reps)
        del d
        torch.cuda.empty_cache()
    print(json.dumps(out, indent=1))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
