"""Per-batch time of the training-batch generators over lazy X / Y against the resident path: one JSON line.

Milliseconds per batch_device(i), host clock around the call and a device synchronise, medians after warm-up, for
- 2-D: 32 images of 1024^2, batch 8 x 256^2, 32 rays, grid (2,2), foreground_prob 0.9;
- 3-D: 2 volumes of 256x512x512 (a 128x256x256 ellipsoid volume tiled 2x2x2), batch 2 x 64x128x128, 96 rays, grid (1,2,2),
  anisotropy (2,1,1), foreground_prob 0.5.
The lazy sequences index the same in-memory lists, so the lazy figure is the cost of reading whole images through the
generator (the per-read checks, the pinned upload, the relabelling and the foreground index) without any file I/O; a
loader that reads from disk adds its own time.  Both paths are timed with sample_ind_cache=True and False.
Usage: python tests/tools/lazy_batch_bench.py [--iters 20] [--warmup 3]"""
import argparse, json, os, sys, time
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from train_batch_bench import gpu_info


class Lazy:
    def __init__(self, items):
        self.items = items

    def __len__(self):
        return len(self.items)

    def __getitem__(self, k):
        return self.items[k]


def timed(gen, iters, warmup):
    import torch
    ts = []
    for i in range(warmup + iters):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        gen.batch_device(i)
        torch.cuda.synchronize()
        if i >= warmup:
            ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import bench_data
    from stardist_b200.models import StarDistData2D, StarDistData3D
    from stardist_b200.rays3d import Rays_GoldenSpiral
    name, power = gpu_info()
    out = {"gpu": name, "power_limit": power}
    X2, Y2 = zip(*[bench_data.synthetic_image((1024, 1024), seed=s) for s in range(32)])
    X2, Y2 = list(X2), list(Y2)
    y3 = np.tile(bench_data.ellipsoid_labels((128, 256, 256), seed=0), (2, 2, 2))
    Y3 = [y3, np.ascontiguousarray(y3[::-1])]
    X3 = [y.astype(np.float32) for y in Y3]
    for cache in (True, False):
        tag = "cache" if cache else "nocache"
        for mode, wrap in (("resident", list), ("lazy", Lazy)):
            np.random.seed(0)
            g2 = StarDistData2D(wrap(X2), wrap(Y2), batch_size=8, n_rays=32, length=10 ** 6, patch_size=(256, 256), grid=(2, 2),
                                foreground_prob=0.9, sample_ind_cache=cache)
            out["2d_%s_%s_ms" % (mode, tag)] = timed(g2, a.iters, a.warmup)
            del g2
            np.random.seed(0)
            g3 = StarDistData3D(wrap(X3), wrap(Y3), batch_size=2, rays=Rays_GoldenSpiral(96), length=10 ** 6, patch_size=(64, 128, 128),
                                grid=(1, 2, 2), anisotropy=(2, 1, 1), foreground_prob=0.5, sample_ind_cache=cache)
            out["3d_%s_%s_ms" % (mode, tag)] = timed(g3, a.iters, a.warmup)
            del g3
    print(json.dumps(out))


if __name__ == "__main__":
    main()
