"""A/B of the tensor-core accumulation scheme (sdb_tc_set_split_acc 0 / 1): max |error| of prob / dist against a float64
evaluation of the same network, relative to the map scale, for (a) the reference's trained 2D_demo model on its test image,
(b) the seeded bench network on a 512x512 crop of the bench image, (c) a random-init 3-D U-Net.  The bar is 1e-5."""
import os, sys, json
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import torch, stardist_b200 as sd
from stardist_b200 import _lib
from stardist_b200.utils import normalize
from oracle import unet_torch
import demo2d, bench_data

lib = _lib.require_cuda()
out = {}


def errs(tag, prob, dist, rp64, rd64):
    for name, g, r in (("prob", prob, rp64), ("dist", dist, rd64)):
        g = np.asarray(g, np.float64); r = np.asarray(r, np.float64)
        scale = max(1.0, float(np.max(np.abs(r)))) if name == "prob" else float(np.max(np.abs(r)))
        e = float(np.max(np.abs(g - r)))
        out["%s/%s" % (tag, name)] = dict(max_abs=e, scale=scale, rel=e / scale, mean_abs=float(np.mean(np.abs(g - r))),
                                          mean_signed=float(np.mean(g - r)))
        print("%-34s %-5s scale %9.4g  max|err| %.3e  = %.2e of scale   mean|err| %.2e  mean err %+.2e" %
              (tag, name, scale, e, e / scale, np.mean(np.abs(g - r)), np.mean(g - r)), flush=True)


# (a) trained 2D_demo
kwargs, weights, thr, img, mask = demo2d.load()
cfg = sd.Config2D(**kwargs)
x = normalize(img, 1, 99.8)
rp64, rd64 = unet_torch.forward(cfg, weights, x[None, ..., None].astype(np.float32), dtype=torch.float64)
rd64 = np.maximum(1e-3, rd64[0]); rp64 = rp64[0]
rp32, rd32 = unet_torch.forward(cfg, weights, x[None, ..., None].astype(np.float32))
errs("2D_demo torch-cpu fp32", rp32[0], np.maximum(1e-3, rd32[0]), rp64, rd64)
# (b) bench network
cfg_b = sd.Config2D(n_rays=32)
w_b = bench_data.bench_weights_2d(cfg_b)
img_b, _ = bench_data.synthetic_image((1024, 1024), seed=0)
img_b = np.ascontiguousarray(img_b[:512, :512])
bp64, bd64 = unet_torch.forward(cfg_b, w_b, img_b[None, ..., None].astype(np.float32), dtype=torch.float64)
bd64 = np.maximum(1e-3, bd64[0]); bp64 = bp64[0]
# (c) random-init 3-D
cfg_c = sd.Config3D(rays=sd.Rays_GoldenSpiral(96))
m_c = sd.StarDist3D(cfg_c, name=None, basedir=None)
vol = np.random.default_rng(1).uniform(0, 1, (16, 64, 128)).astype(np.float32)
cp64, cd64 = unet_torch.forward(cfg_c, m_c.weights, vol[None, ..., None], dtype=torch.float64)

for split in (0, 1):
    lib.sdb_tc_set_split_acc(split)
    model = sd.StarDist2D(cfg, name=None, basedir=None, weights=weights)
    prob, dist = model.predict(x)
    errs("2D_demo tensor-core split_acc=%d" % split, prob, dist, rp64, rd64)
    model = sd.StarDist2D(cfg_b, name=None, basedir=None, weights=w_b)
    prob, dist = model.predict(img_b)
    errs("bench net tensor-core split_acc=%d" % split, prob, dist, bp64, bd64)
    xc = torch.from_numpy(vol[None, ..., None]).cuda()
    p, d = m_c.net.forward(xc)
    errs("3D random tensor-core split_acc=%d" % split, p.cpu().numpy()[0], d.cpu().numpy()[0], cp64[0], cd64[0])
    # speed of the bench forward with this setting
    xb = torch.from_numpy(bench_data.synthetic_image((1024, 1024), seed=0)[0][None, ..., None]).cuda()
    mb = sd.StarDist2D(cfg_b, name=None, basedir=None, weights=w_b)
    for _ in range(3): mb.net.forward(xb)
    a = torch.cuda.Event(enable_timing=True); b = torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize(); a.record()
    for _ in range(20): mb.net.forward(xb)
    b.record(); torch.cuda.synchronize()
    out["bench_forward_ms/split_acc=%d" % split] = a.elapsed_time(b) / 20
    print("bench U-Net forward 1024x1024, split_acc=%d: %.3f ms (L2-warm, back to back)" % (split, a.elapsed_time(b) / 20), flush=True)
lib.sdb_tc_set_split_acc(1)
print(json.dumps(out))
