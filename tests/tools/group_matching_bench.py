"""Cost of group_matching_labels: one JSON line per workload.

Workloads: T = 50 frames of 1024^2 (bench_data.ellipse_labels, about 1000 objects per frame) and T = 8 volumes of
128x256x256 (bench_data.ellipsoid_labels), each frame the base shifted by a per-frame offset and relabelled at random.
Medians over --iters repeats after --warmup, host clock around work that ends in a device synchronise:
- `device_total_ms`: group_matching_labels on a CUDA int32 stack (result stays on the device);
- `device_numpy_ms`: the same from a numpy stack (upload and download included; one repeat);
- `host_total_ms`: the numpy back-end on the same stack (one repeat);
- `labels_ms`, `overlap_ms`, `remap_ms`: the three device passes (sdb_stack_labels, sdb_stack_overlap, sdb_stack_group_remap),
  each with its small table read-back; `lsa_ms`: the time inside scipy's linear_sum_assignment during one device call,
  `chain_ms`: all host work of the chaining (the assignment included);
- `*_floor_bytes` and `*_GBps`: the bytes the overlap pass (two int32 frames read per pair) and the remap pass (one read,
  one write per pixel) must move, over their time.
The results of the two back-ends are compared on every workload.
Usage: python tests/tools/group_matching_bench.py [--iters 3] [--warmup 1]"""
import argparse, json, os, sys, time
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from train_step_bench import gpu_info


def movie(base, T, seed):
    """T frames: base rolled by t * (1, 2[, 3]) and relabelled at random (ids up to 10^6)"""
    rng = np.random.default_rng(seed)
    out = []
    for t in range(T):
        y = np.roll(base, tuple(t * (k + 1) for k in range(base.ndim)), axis=tuple(range(base.ndim)))
        u = np.unique(y[y > 0])
        lut = np.zeros(int(y.max()) + 1, np.int32)
        lut[u] = rng.choice(10 ** 6, size=len(u), replace=False) + 1
        out.append(lut[y])
    return np.stack(out)


def timed(fn):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return r, (time.perf_counter() - t0) * 1e3


def phases(stack):
    """the device path of matching._group_device with each phase timed; returns (result, {phase: ms})"""
    import torch, scipy.optimize
    from stardist_b200 import matching as M, _lib as L
    lib = L.require_cuda()
    T, S = int(stack.shape[0]), stack.numel() // int(stack.shape[0])
    (ids, offsets), t_labels = timed(lambda: M.stack_labels_device(stack))
    tables, t_overlap = timed(lambda: M.stack_overlap_device(stack, ids, offsets))
    per_frame = [ids[offsets[f]:offsets[f + 1]] for f in range(T)]

    def overlap(p):
        a, b, c = tables[p]
        m = np.zeros((1 + len(per_frame[p]), 1 + len(per_frame[p + 1])), np.int64)
        m[a, b] = c
        return m
    lsa_ms = [0.0]
    lsa = scipy.optimize.linear_sum_assignment

    def lsa_timed(c):
        t0 = time.perf_counter(); r = lsa(c); lsa_ms[0] += (time.perf_counter() - t0) * 1e3
        return r
    scipy.optimize.linear_sum_assignment = lsa_timed
    try:
        luts, t_chain = timed(lambda: M._group_chain(per_frame, overlap, 1e-10, 'iou'))
    finally:
        scipy.optimize.linear_sum_assignment = lsa

    def remap():
        lut_d = torch.from_numpy(np.concatenate(luts).astype(np.int32)).cuda()
        ids_d = torch.from_numpy(np.ascontiguousarray(ids, np.int32)).cuda()
        off_d = torch.from_numpy(offsets).cuda()
        out = torch.empty_like(stack)
        L.check(lib.sdb_stack_group_remap(L.ptr(stack), T, S, L.ptr(ids_d), L.ptr(off_d), L.ptr(lut_d), L.ptr(out), L.stream_ptr()))
        return out
    out, t_remap = timed(remap)
    return out, dict(labels_ms=t_labels, overlap_ms=t_overlap, chain_ms=t_chain, lsa_ms=lsa_ms[0], remap_ms=t_remap,
                     objects_per_frame=float(np.mean(np.diff(offsets))))


def run(name, stack_h, iters, warmup):
    import torch
    from stardist_b200.matching import group_matching_labels, _group_host
    stack = torch.from_numpy(stack_h).cuda()
    T, S = stack_h.shape[0], stack_h[0].size
    for _ in range(warmup):
        phases(stack)
    dev = []
    for _ in range(iters):
        got, ms = timed(lambda: group_matching_labels(stack))
        dev.append(ms)
    got = got.cpu().numpy()
    dev_np = timed(lambda: group_matching_labels(stack_h))[1]
    ph = [phases(stack)[1] for _ in range(iters)]
    t0 = time.perf_counter()
    want = _group_host(stack_h, 1e-10, 'iou')
    host_ms = (time.perf_counter() - t0) * 1e3
    med = {k: float(np.median([p[k] for p in ph])) for k in ph[0]}
    overlap_bytes, remap_bytes = 2 * 4 * (T - 1) * S, 2 * 4 * T * S
    return dict(workload=name, T=T, frame_shape=list(stack_h.shape[1:]), device_total_ms=float(np.median(dev)),
                device_numpy_ms=dev_np, host_total_ms=host_ms, **med,
                overlap_floor_bytes=overlap_bytes, overlap_GBps=overlap_bytes / med['overlap_ms'] / 1e6,
                remap_floor_bytes=remap_bytes, remap_GBps=remap_bytes / med['remap_ms'] / 1e6,
                device_equals_host=bool(np.array_equal(got, want)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("group_matching_bench needs a CUDA device")
    import bench_data
    info = gpu_info()
    work = [("2d_50x1024^2", movie(bench_data.ellipse_labels((1024, 1024), seed=0), 50, 0)),
            ("3d_8x128x256x256", movie(bench_data.ellipsoid_labels((128, 256, 256), seed=0), 8, 1))]
    for name, stack_h in work:
        r = run(name, stack_h, a.iters, a.warmup)
        r["gpu"] = info
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
