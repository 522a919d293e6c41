"""GPU tests of the wgmma convolution path (csrc/unet_tc.cu): single layers against a float64
torch convolution of the *same split operands*, then the whole network against torch-CPU fp32."""
import os, sys
import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


def _split(t):
    import torch
    hi = t.to(torch.float16)
    lo = (t - hi.to(torch.float32)).to(torch.float16)
    return torch.stack([hi, lo]).contiguous()


def _ref_conv(x_nhwc, k, b, relu):
    import torch, torch.nn.functional as F
    t = x_nhwc.double().permute(0, 3, 1, 2)
    kt = k.double().permute(3, 2, 0, 1)
    y = F.conv2d(t, kt, b.double(), padding=1)
    if relu: y = F.relu(y)
    return y.permute(0, 2, 3, 1)


@pytest.mark.parametrize("h,w,c0,c1,cout,relu,up2x", [
    (16, 32, 0, 64, 64, 1, 0), (8, 16, 0, 32, 32, 1, 0), (24, 40, 0, 128, 128, 0, 0), (16, 16, 0, 256, 128, 1, 0),
    (16, 32, 64, 64, 64, 1, 0), (16, 32, 32, 32, 32, 1, 0), (13, 21, 0, 64, 32, 1, 0), (8, 16, 0, 128, 256, 1, 1),
    (40, 72, 0, 32, 128, 1, 0)])
def test_conv3x3_tc_single_layer(h, w, c0, c1, cout, relu, up2x):
    import torch
    from stardist_b200 import _lib as L
    lib = L.require_cuda()
    g = torch.Generator(device='cpu').manual_seed(h * 131 + w + cout)
    cin = c0 + c1
    x = torch.randn((2, h, w, cin), generator=g).cuda()
    k = (torch.randn((3, 3, cin, cout), generator=g) * (2.0 / (9 * cin)) ** 0.5).cuda()
    b = (torch.randn(cout, generator=g) * 0.1).cuda()
    xs = _split(x)                       # [2,n,h,w,cin]
    x_eff = xs[0].double() + xs[1].double()
    ws = torch.empty((2, 9, cout, cin), dtype=torch.float16, device='cuda')
    from stardist_b200.models.unet_device import tc_weight_scale
    wsc = tc_weight_scale(k.cpu().numpy())
    L.check(lib.sdb_split_weights(L.ptr(k.contiguous()), cin, cout, wsc, L.ptr(ws[0]), L.ptr(ws[1]), L.stream_ptr()))
    k_eff = ((ws[0].double() + ws[1].double()) / wsc).reshape(3, 3, cout, cin).permute(0, 1, 3, 2)
    src1 = xs[..., c0:].contiguous(); src0 = xs[..., :c0].contiguous() if c0 else None
    oh, ow = (2 * h, 2 * w) if up2x else (h, w)
    out = torch.zeros((2, 2, oh, ow, cout), dtype=torch.float16, device='cuda')
    L.check(lib.sdb_conv3x3_tc(L.ptr(src0[0]) if c0 else L.ptr(None), L.ptr(src0[1]) if c0 else L.ptr(None), c0,
                               L.ptr(src1[0]), L.ptr(src1[1]), c1, 2, h, w, L.ptr(ws[0]), L.ptr(ws[1]), wsc, L.ptr(b), cout, relu, up2x,
                               L.ptr(out[0]), L.ptr(out[1]), L.stream_ptr()))
    L.check(lib.sdb_tc_error_check(L.stream_ptr()))
    got = (out[0].float() + out[1].float()).double()
    want = _ref_conv(x_eff, k_eff, b, relu)
    if up2x:
        want = want.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2)
    err = (got - want).abs().max().item()
    scale = want.abs().max().item()
    # fp32 accumulation over K = 9*cin terms (the tensor-core adder truncates): observed <= 5e-6 relative
    assert err <= 1e-5 * max(1.0, scale), (err, scale)


@pytest.mark.parametrize("shape,grid", [((64, 96), (1, 1)), ((48, 80), (2, 2)), ((72, 104), (1, 1))])
def test_unet_tc_vs_torch_fp32(shape, grid):
    import torch, stardist_b200 as sd
    from stardist_b200.models.unet_device import UNetDevice2DTC, UNetDevice2D
    from oracle import unet_torch
    cfg = sd.Config2D(n_rays=32, grid=grid)
    model = sd.StarDist2D(cfg, name=None, basedir=None)
    assert isinstance(model.net, UNetDevice2DTC)
    rng = np.random.default_rng(3)
    img = rng.uniform(0, 1, shape).astype(np.float32)
    x = torch.from_numpy(img[None, ..., None]).cuda()
    prob, dist = model.net.forward(x)
    rp, rd = unet_torch.forward(cfg, model.weights, img[None, ..., None])
    p, d = prob.cpu().numpy(), dist.cpu().numpy()
    assert np.max(np.abs(p - rp)) <= 1e-5 * max(1.0, np.max(np.abs(rp)))
    assert np.max(np.abs(d - rd)) <= 1e-5 * max(1e-3, np.max(np.abs(rd))) + 1e-7
    # and against the exact-fp32 CUDA-core kernels of the same library
    simt = UNetDevice2D(cfg, model.weights)
    p2, d2 = simt.forward(x)
    assert torch.max(torch.abs(p2 - prob)).item() <= 1e-5


@pytest.mark.parametrize("n_rays,fuse", [(16, "1"), (32, "0"), (64, "1"), (7, "1")])
def test_unet_tc_head_variants(n_rays, fuse, monkeypatch):
    """heads: fused into the features epilogue (n_rays <= 32, CUDA cores on the fp32 accumulators) or as the
    separate tensor-core 1x1 kernel (n_rays > 32, or STARDIST_B200_FUSE_HEADS=0) -- both against torch-CPU fp32"""
    import torch, stardist_b200 as sd
    from stardist_b200.models.unet_device import UNetDevice2DTC
    from oracle import unet_torch
    monkeypatch.setenv("STARDIST_B200_FUSE_HEADS", fuse)
    cfg = sd.Config2D(n_rays=n_rays)
    model = sd.StarDist2D(cfg, name=None, basedir=None, seed=n_rays)
    assert isinstance(model.net, UNetDevice2DTC)
    assert model.net.fuse_heads == (fuse == "1" and n_rays <= 32)
    rng = np.random.default_rng(n_rays)
    img = rng.uniform(0, 1, (56, 264)).astype(np.float32)      # 264 = 2 tiles of 128 + a ragged one
    x = torch.from_numpy(img[None, ..., None]).cuda()
    prob, dist = model.net.forward(x)
    rp, rd = unet_torch.forward(cfg, model.weights, img[None, ..., None])
    p, d = prob.cpu().numpy(), dist.cpu().numpy()
    assert p.shape == rp.shape and d.shape == rd.shape
    assert np.max(np.abs(p - rp)) <= 1e-5 * max(1.0, np.max(np.abs(rp)))
    assert np.max(np.abs(d - rd)) <= 1e-5 * max(1e-3, np.max(np.abs(rd))) + 1e-7


@pytest.mark.parametrize("variant", [1, 3, 4])
def test_conv_variants_agree(variant):
    """the conv kernel variants (one tile per CTA / persistent, 64-channel K blocks / persistent, 32-channel K blocks) on one layer"""
    import torch
    from stardist_b200 import _lib as L
    from stardist_b200.models.unet_device import tc_weight_scale
    lib = L.require_cuda()
    g = torch.Generator(device='cpu').manual_seed(11)
    h, w, cin, cout = 37, 300, 64, 64
    x = torch.randn((1, h, w, cin), generator=g).cuda()
    k = (torch.randn((3, 3, cin, cout), generator=g) * (2.0 / (9 * cin)) ** 0.5).cuda()
    b = (torch.randn(cout, generator=g) * 0.1).cuda()
    xs = _split(x); x_eff = xs[0].double() + xs[1].double()
    ws = torch.empty((2, 9, cout, cin), dtype=torch.float16, device='cuda')
    wsc = tc_weight_scale(k.cpu().numpy())
    L.check(lib.sdb_split_weights(L.ptr(k.contiguous()), cin, cout, wsc, L.ptr(ws[0]), L.ptr(ws[1]), L.stream_ptr()))
    k_eff = ((ws[0].double() + ws[1].double()) / wsc).reshape(3, 3, cout, cin).permute(0, 1, 3, 2)
    out = torch.zeros((2, 1, h, w, cout), dtype=torch.float16, device='cuda')
    try:
        L.check(lib.sdb_tc_set_variant(variant))
        L.check(lib.sdb_conv3x3_tc(L.ptr(None), L.ptr(None), 0, L.ptr(xs[0]), L.ptr(xs[1]), cin, 1, h, w, L.ptr(ws[0]), L.ptr(ws[1]), wsc,
                                   L.ptr(b), cout, 1, 0, L.ptr(out[0]), L.ptr(out[1]), L.stream_ptr()))
        L.check(lib.sdb_tc_error_check(L.stream_ptr()))
    finally:
        L.check(lib.sdb_tc_set_variant(0))
    got = (out[0].float() + out[1].float()).double()
    want = _ref_conv(x_eff, k_eff, b, 1)
    assert (got - want).abs().max().item() <= 1e-5 * max(1.0, want.abs().max().item())


@pytest.mark.parametrize("nd", [2, 3])
def test_c_unet_forward_equals_python_executor(nd):
    """_LIB_unet_forward_2d / _3d (SURVEY 8b: the network boundary as C entry points, csrc/unet_exec.cu) launch the same kernels
    in the same order as the Python executor: prob / dist maps bit-equal; the library names the layers it expects"""
    import ctypes, torch
    import stardist_b200 as sd
    from stardist_b200 import _lib as L
    lib = L.require_cuda()
    rng = np.random.default_rng(11)
    if nd == 2:
        cfg = sd.Config2D(n_rays=32)
        model = sd.StarDist2D(cfg, name=None, basedir=None)
        x = rng.uniform(0, 1, (1, 96, 160, 1)).astype(np.float32)
    else:
        cfg = sd.Config3D(rays=sd.Rays_GoldenSpiral(96))
        model = sd.StarDist3D(cfg, name=None, basedir=None)
        x = rng.uniform(0, 1, (1, 16, 32, 64, 1)).astype(np.float32)
    net, ccfg = L.c_unet_create(cfg, model.weights)
    try:
        n = lib.sdb_unet_layer_count(ctypes.byref(ccfg))
        names = [lib.sdb_unet_layer_name(ctypes.byref(ccfg), i).decode() for i in range(n)]
        assert names[0] == 'down_level_0_no_0' and names[-3:] == ['features', 'prob', 'dist'] and set(names) <= set(model.weights)
        xd = torch.from_numpy(x).cuda()
        want_p, want_d = model.net.forward(xd)
        sp = tuple(x.shape[1:-1])
        prob = torch.empty(sp, dtype=torch.float32, device='cuda')
        dist = torch.empty(sp + (cfg.n_rays,), dtype=torch.float32, device='cuda')
        if nd == 2:
            L.check(lib._LIB_unet_forward_2d(net, L.ptr(xd), sp[0], sp[1], L.ptr(prob), L.ptr(dist), L.stream_ptr()))
        else:
            L.check(lib._LIB_unet_forward_3d(net, L.ptr(xd), sp[0], sp[1], sp[2], L.ptr(prob), L.ptr(dist), L.stream_ptr()))
        torch.cuda.synchronize()
        assert torch.equal(prob, want_p[0]) and torch.equal(dist, want_d[0])
        # extents that are not multiples of 2^depth are refused (the caller pads, as StarDistPadAndCropResizer does)
        assert lib._LIB_unet_forward_2d(net, L.ptr(xd), 97, 160, L.ptr(prob), L.ptr(dist), L.stream_ptr()) != 0
    finally:
        lib.sdb_unet_destroy(net)
