"""Cost of augmentation in training: one JSON line.

Medians after warm-up, host clock around work that ends in a device synchronise, for the 2-D default (batch 4 x 256^2, 32 rays,
grid (1,1), 8 images of 1024^2) and the 3-D default (batch 1 x 128^3, 96 rays, grid (1,2,2), anisotropy (2,1,1), 2 volumes of
128x256x256), each without augmenter, with the host path (the notebook augmenter restated in numpy as a plain callable:
tests/augment_emu.py aug_emu) and with the device Augmenter (the 2-D notebook's Augmenter(); in 3-D the notebook's
Augmenter(axis=(1, 2), noise=None) and, as a second line, the same with noise):
- `*_batch_ms`: StarDistData*.batch_device(i);
- `*_step_ms`: batch_device(i) followed by UNetTrainer.step on it (one training step with its batch);
- `normal_*_ms`: the Gaussian generator alone (models.augment.normal_device) at 262 144 and 2 097 152 values, and numpy's
  np.random.normal on the host CPU at the same sizes.
Usage: python tests/tools/augment_bench.py [--iters 20] [--warmup 3]"""
import argparse, json, os, sys, time
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from train_step_bench import gpu_info


def median_ms(fn, iters, warmup):
    import torch
    ts = []
    for i in range(warmup + iters):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn(i)
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
    import augment_emu as E
    from stardist_b200 import Config2D, Config3D
    from stardist_b200.models import Augmenter, StarDistData2D, StarDistData3D
    from stardist_b200.models.augment import normal_device
    from stardist_b200.models.train import UNetTrainer
    from stardist_b200.models.weights import glorot_uniform_weights
    from stardist_b200.rays3d import Rays_GoldenSpiral
    out = {"gpu": gpu_info()}
    X2, Y2 = zip(*[bench_data.synthetic_image((1024, 1024), seed=s) for s in range(8)])
    X2, Y2 = list(X2), list(Y2)
    Y3 = [bench_data.ellipsoid_labels((128, 256, 256), seed=s) for s in range(2)]
    X3 = [y.astype(np.float32) / max(1, int(y.max())) for y in Y3]
    c2, c3 = Config2D(n_rays=32), Config3D(rays=Rays_GoldenSpiral(96), grid=(1, 2, 2), anisotropy=(2, 1, 1))
    cases = [
        ("2d", c2, lambda aug: StarDistData2D(X2, Y2, batch_size=4, n_rays=32, length=10 ** 6, patch_size=(256, 256), augmenter=aug),
         [("none", None), ("host", lambda x, y: E.aug_emu(x, y)), ("device", Augmenter())]),
        ("3d", c3, lambda aug: StarDistData3D(X3, Y3, batch_size=1, rays=Rays_GoldenSpiral(96), length=10 ** 6, patch_size=(128, 128, 128),
                                              grid=(1, 2, 2), anisotropy=(2, 1, 1), augmenter=aug),
         [("none", None), ("host", lambda x, y: E.aug_emu(x, y, axis=(1, 2), noise=None)), ("device", Augmenter(axis=(1, 2), noise=None)),
          ("host_noise", lambda x, y: E.aug_emu(x, y, axis=(1, 2))), ("device_noise", Augmenter(axis=(1, 2)))]),
    ]
    for tag, config, make, augs in cases:
        trainer = UNetTrainer(config, glorot_uniform_weights(config, seed=0))
        for name, aug in augs:
            np.random.seed(0)
            gen = make(aug)
            out["%s_%s_batch_ms" % (tag, name)] = median_ms(lambda i: gen.batch_device(i), a.iters, a.warmup)

            def step(i):
                (x,), targets = gen.batch_device(10 ** 4 + i)
                trainer.step(x, *targets)
            out["%s_%s_step_ms" % (tag, name)] = median_ms(step, a.iters, a.warmup)
            del gen
        del trainer
    for n in (262144, 2097152):
        np.random.seed(0)
        out["normal_%d_device_ms" % n] = median_ms(lambda i: normal_device(n), a.iters, a.warmup)
        out["normal_%d_numpy_ms" % n] = median_ms(lambda i: np.random.normal(0, 1, n), a.iters, a.warmup)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
