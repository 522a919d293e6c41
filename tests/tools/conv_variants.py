"""the conv kernel variants (one tile per CTA / persistent, 64-channel K blocks / persistent, 32-channel K blocks) against a float64 convolution of
the same split operands, and their timings on the layer shapes of the 1024x1024 forward pass"""
import sys, os, time
import numpy as np, torch, torch.nn.functional as F
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from stardist_b200 import _lib as L
from stardist_b200.models.unet_device import tc_weight_scale
lib = L.require_cuda()

def split(t):
    hi = t.to(torch.float16); lo = (t - hi.float()).to(torch.float16)
    return torch.stack([hi, lo]).contiguous()

def run(h, w, c0, c1, cout, relu, up2x, mode):
    g = torch.Generator().manual_seed(h * 131 + w + cout)
    cin = c0 + c1
    x = torch.randn((2, h, w, cin), generator=g).cuda()
    k = (torch.randn((3, 3, cin, cout), generator=g) * (2.0 / (9 * cin)) ** 0.5).cuda()
    b = (torch.randn(cout, generator=g) * 0.1).cuda()
    xs = split(x); x_eff = xs[0].double() + xs[1].double()
    ws = torch.empty((2, 9, cout, cin), dtype=torch.float16, device='cuda')
    wsc = tc_weight_scale(k.cpu().numpy())
    L.check(lib.sdb_split_weights(L.ptr(k.contiguous()), cin, cout, wsc, L.ptr(ws[0]), L.ptr(ws[1]), L.stream_ptr()))
    k_eff = ((ws[0].double() + ws[1].double()) / wsc).reshape(3, 3, cout, cin).permute(0, 1, 3, 2)
    src1 = xs[..., c0:].contiguous(); src0 = xs[..., :c0].contiguous() if c0 else None
    oh, ow = (2 * h, 2 * w) if up2x else (h, w)
    out = torch.zeros((2, 2, oh, ow, cout), dtype=torch.float16, device='cuda')
    args = (L.ptr(src0[0]) if c0 else L.ptr(None), L.ptr(src0[1]) if c0 else L.ptr(None), c0, L.ptr(src1[0]), L.ptr(src1[1]), c1,
            2, h, w, L.ptr(ws[0]), L.ptr(ws[1]), wsc, L.ptr(b), cout, relu, up2x)
    L.check(lib.sdb_tc_set_variant(-mode))
    L.check(lib.sdb_conv3x3_tc(*args, L.ptr(out[0]), L.ptr(out[1]), L.stream_ptr()))
    L.check(lib.sdb_tc_error_check(L.stream_ptr()))
    got = out[0].double() + out[1].double()
    y = F.conv2d(x_eff.permute(0, 3, 1, 2), k_eff.permute(3, 2, 0, 1), b.double(), padding=1)
    if relu: y = F.relu(y)
    want = y.permute(0, 2, 3, 1)
    if up2x: want = want.repeat_interleave(2, 1).repeat_interleave(2, 2)
    return (got - want).abs().max().item() / max(1.0, want.abs().max().item())

cases = [(16, 128, 0, 32, 32, 1, 0), (7, 300, 0, 32, 128, 1, 0), (33, 97, 0, 64, 32, 1, 1), (64, 640, 32, 32, 32, 1, 0), (40, 256, 64, 64, 64, 1, 0), (9, 200, 0, 64, 64, 1, 0), (32, 256, 0, 128, 128, 0, 0), (16, 128, 64, 64, 64, 1, 0),
         (8, 130, 0, 128, 256, 1, 1), (5, 77, 32, 32, 32, 1, 0), (64, 512, 0, 32, 128, 1, 0)]
for c in cases:
    e = [run(*c, m) for m in (-1, -3, -4)]
    print(c, "rel err  v1 %.2e | v3 %.2e | v4 %.2e" % tuple(e))

# timing of the big layers (1024^2)
def bench(h, w, c0, c1, cout, mode, reps=5):
    cin = c0 + c1
    xs = torch.randn((2, 1, h, w, cin), device='cuda').half()
    ws = torch.randn((2, 9, cout, cin), device='cuda').half()
    b = torch.zeros(cout, device='cuda')
    out = torch.empty((2, 1, h, w, cout), dtype=torch.float16, device='cuda')
    src0 = xs[..., :c0].contiguous() if c0 else None; src1 = xs[..., c0:].contiguous()
    args = (L.ptr(src0[0]) if c0 else L.ptr(None), L.ptr(src0[1]) if c0 else L.ptr(None), c0, L.ptr(src1[0]), L.ptr(src1[1]), c1,
            1, h, w, L.ptr(ws[0]), L.ptr(ws[1]), 1.0, L.ptr(b), cout, 1, 0)
    def go():
        L.check(lib.sdb_tc_set_variant(-mode))
        L.check(lib.sdb_conv3x3_tc(*args, L.ptr(out[0]), L.ptr(out[1]), L.stream_ptr()))
    for _ in range(2): go()
    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps): go()
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    fl = 2.0 * h * w * 9 * cin * cout
    return ms, fl / ms / 1e9
for (h, w, c0, c1, cout) in [(1024, 1024, 0, 32, 32), (1024, 1024, 0, 32, 128), (1024, 1024, 32, 32, 32), (512, 512, 0, 64, 64), (256, 256, 0, 128, 128), (256, 256, 128, 128, 128), (128, 128, 0, 256, 128), (512, 512, 64, 64, 64), (512, 512, 0, 64, 32), (256, 256, 0, 128, 64), (256, 256, 0, 64, 128)]:
    r1 = bench(h, w, c0, c1, cout, -1); r3 = bench(h, w, c0, c1, cout, -3); r2 = bench(h, w, c0, c1, cout, -4)
    print((h, w, c0 + c1, cout), "v1 %.3f ms (%.0f TF/s alg)  v3 %.3f ms (%.0f TF/s alg)  v4 %.3f ms (%.0f TF/s alg)" % (r1[0], r1[1], r3[0], r3[1], r2[0], r2[1]))
L.check(lib.sdb_tc_error_check(L.stream_ptr()))
L.check(lib.sdb_tc_set_variant(0))
