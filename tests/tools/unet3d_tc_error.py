"""fp32-faithfulness of the 3-D tensor-core U-Net: max errors against a float64 evaluation, next to torch-CPU fp32's own"""
import os, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import torch, stardist_b200 as sd
from oracle import unet_torch
from stardist_b200.models.unet_device import UNetDeviceND
for shape, grid in (((16, 32, 48), (1, 1, 1)), ((8, 24, 136), (1, 2, 2))):
    cfg = sd.Config3D(rays=sd.Rays_GoldenSpiral(96), grid=grid)
    model = sd.StarDist3D(cfg, name=None, basedir=None)
    rng = np.random.default_rng(shape[2])
    vol = rng.uniform(0, 1, shape).astype(np.float32)
    x = torch.from_numpy(vol[None, ..., None]).cuda()
    prob, dist = model.net.forward(x)
    ps, ds = UNetDeviceND(cfg, model.weights).forward(x)
    rp64, rd64 = unet_torch.forward(cfg, model.weights, vol[None, ..., None], dtype=torch.float64)
    rp32, rd32 = unet_torch.forward(cfg, model.weights, vol[None, ..., None])
    for name, got, simt, r64, r32 in (("prob", prob, ps, rp64, rp32), ("dist", dist, ds, rd64, rd32)):
        g = got.cpu().numpy().astype(np.float64); s = simt.cpu().numpy().astype(np.float64)
        scale = float(np.max(np.abs(r64)))
        print(shape, grid, name, "scale %.4g | tensor-core %.3g | cuda-core fp32 %.3g | torch-cpu fp32 %.3g  (max abs error vs float64; relative to scale: %.2e / %.2e / %.2e)" %
              (scale, np.max(np.abs(g - r64)), np.max(np.abs(s - r64)), np.max(np.abs(r32 - r64)),
               np.max(np.abs(g - r64)) / scale, np.max(np.abs(s - r64)) / scale, np.max(np.abs(r32 - r64)) / scale))
