"""Per-layer timing of the tensor-core 3x3 convolutions of the bench U-Net (default Config2D, 1024x1024 image) for each
K-block choice of sdb_conv3x3_tc (variant 3: 64-channel K blocks where the channel counts allow, variant 4: 32-channel K
blocks), CUDA events over repeated launches of one layer.  Prints one JSON line per layer and the GPU's name and power limit.
GPU only:  python tests/tools/conv_layers.py"""
import json, os, subprocess, sys
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from stardist_b200 import _lib as L
from stardist_b200.models.config import Config2D
from stardist_b200.models.weights import unet_layers

lib = L.require_cuda()
print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip())
REPS = 50
h = w = 1024
for l in unet_layers(Config2D(n_rays=32)):
    if l['kind'] == 'pool': h, w = h // 2, w // 2
    if l['kind'] == 'up': h, w = h * 2, w * 2
    if l['kind'] != 'conv' or l['cin'] % 32: continue
    cin, cout = l['cin'], l['cout']
    x = torch.randn((2, 1, h, w, cin), device='cuda').to(torch.float16)
    ws = (torch.randn((2, 9, cout, cin), device='cuda') * 0.05).to(torch.float16)
    b = torch.zeros(cout, device='cuda')
    out = torch.empty((2, 1, h, w, cout), dtype=torch.float16, device='cuda')
    call = lambda: L.check(lib.sdb_conv3x3_tc(L.ptr(None), L.ptr(None), 0, L.ptr(x[0]), L.ptr(x[1]), cin, 1, h, w, L.ptr(ws[0]), L.ptr(ws[1]), 1.0,
                                              L.ptr(b), cout, 1, 0, L.ptr(out[0]), L.ptr(out[1]), L.stream_ptr()))
    row = dict(layer=l['name'], h=h, w=w, cin=cin, cout=cout)
    for variant in (3, 4):
        L.check(lib.sdb_tc_set_variant(variant))
        call(); torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(REPS): call()
        e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / REPS
        row["ms_v%d" % variant] = round(ms, 4)
        row["tflops_v%d" % variant] = round(2.0 * 9 * cin * cout * h * w / (ms / 1e3) / 1e12, 1)
    L.check(lib.sdb_tc_set_variant(0))
    L.check(lib.sdb_tc_error_check(L.stream_ptr()))
    print(json.dumps(row), flush=True)
