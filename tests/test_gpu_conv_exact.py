"""Layer tests of every tensor-core convolution and heads instance (csrc/unet_tc.cu, k_conv_wg<N, KC, FUSE>) on exactly
representable operands (tests/convexact.py): every partial sum is exact in fp32, so each output plane must equal the float64
reference element by element, under both accumulation schemes (sdb_tc_set_split_acc) and every grid / K-block variant
(sdb_tc_set_variant).  Also: the split-format companions against exact CPU restatements, the fp16 range flag, argument
validation, random-data layer tests of the heads N = 144 and fused instances, and the 3-D network at 128 rays."""
import numpy as np
import pytest

import convexact as CX

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def lib():
    """clears the device error word before each test and restores the default variant and accumulation scheme after it"""
    from stardist_b200 import _lib as L
    lib = L.require_cuda()
    lib.sdb_tc_error_check(L.stream_ptr())
    yield lib
    lib.sdb_tc_set_variant(0)
    lib.sdb_tc_set_split_acc(1)


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _ptr(t):
    from stardist_b200 import _lib as L
    return L.ptr(t)


def _st():
    from stardist_b200 import _lib as L
    return L.stream_ptr()


def _call(lib, rc):
    """a launch that must succeed and leave the device error word clear"""
    from stardist_b200 import _lib as L
    L.check(rc)
    err = lib.sdb_tc_error_check(_st())
    assert err == 0, "sdb_tc_error_check = %d: %s" % (err, lib.sdb_last_error().decode())


def _switches(lib, case):
    from stardist_b200 import _lib as L
    L.check(lib.sdb_tc_set_variant(case["variant"]))
    L.check(lib.sdb_tc_set_split_acc(case["split"]))


def _sources(D, c0):
    xh, xl = _dev(D["x_hi"]), _dev(D["x_lo"])
    src1 = (xh[..., c0:].contiguous(), xl[..., c0:].contiguous())
    src0 = (xh[..., :c0].contiguous(), xl[..., :c0].contiguous()) if c0 else (None, None)
    return src0, src1


def _nan_planes(shape, dtype):
    import torch
    return torch.full(shape, float("nan"), dtype=dtype, device="cuda")        # elements nobody writes stay NaN


# ------------------------------------------------------------------------------------------------ exact layer tests
@pytest.mark.parametrize("case", CX.CONV2D_CASES + CX.CONV3D_CASES, ids=CX.case_id)
def test_conv_tc_exact(lib, case):
    import torch
    D = CX.gen_conv(case)
    c0, c1, cout, f = case["c0"], case["c1"], case["cout"], 2 if case["up"] else 1
    src0, src1 = _sources(D, c0)
    wh, wl, b = _dev(D["w_hi"]), _dev(D["w_lo"]), _dev(D["bias"])
    _switches(lib, case)
    if case["family"] == "conv2d":
        n, h, w = case["n"], case["h"], case["w"]
        out = _nan_planes((2, n, f * h, f * w, cout), torch.float16)
        rc = lib.sdb_conv3x3_tc(_ptr(src0[0]), _ptr(src0[1]), c0, _ptr(src1[0]), _ptr(src1[1]), c1, n, h, w, _ptr(wh), _ptr(wl),
                                D["w_scale"], _ptr(b), cout, case["relu"], case["up"], _ptr(out[0]), _ptr(out[1]), _st())
    else:
        d, h, w = case["d"], case["h"], case["w"]
        out = _nan_planes((2, f * d, f * h, f * w, cout), torch.float16)
        rc = lib.sdb_conv3x3x3_tc(_ptr(src0[0]), _ptr(src0[1]), c0, _ptr(src1[0]), _ptr(src1[1]), c1, d, h, w, _ptr(wh), _ptr(wl),
                                  D["w_scale"], _ptr(b), cout, case["relu"], case["up"], _ptr(out[0]), _ptr(out[1]), _st())
    _call(lib, rc)
    want_hi, want_lo = CX.split16(CX.conv_ref(case, D))
    got = out.cpu().numpy()
    msg = CX.first_mismatch(got[0], want_hi, "hi plane [.., c]") or CX.first_mismatch(got[1], want_lo, "lo plane [.., c]")
    assert not msg, "%s: %s" % (CX.case_id(case), msg)


@pytest.mark.parametrize("case", CX.HEADS_CASES, ids=CX.case_id)
def test_heads_tc_exact(lib, case):
    import torch
    D = CX.gen_heads(case)
    n, h, w, R = case["n"], case["h"], case["w"], case["R"]
    xh, xl = _dev(D["x_hi"]), _dev(D["x_lo"])
    wh, wl, b = _dev(D["w_hi"]), _dev(D["w_lo"]), _dev(D["bias"])
    prob = _nan_planes((n, h, w), torch.float32)
    dist = _nan_planes((n, h, w, R), torch.float32)
    _switches(lib, case)
    _call(lib, lib.sdb_heads_tc(_ptr(xh), _ptr(xl), case["cfeat"], n, h, w, _ptr(wh), _ptr(wl), D["w_scale"], _ptr(b), case["np"], R,
                                _ptr(prob), _ptr(dist), _st()))
    want_p, want_d = CX.heads_ref(D, R)
    msg = CX.first_mismatch(dist.cpu().numpy(), want_d, "dist [n, y, x, ray]") or CX.prob_mismatch(prob.cpu().numpy(), want_p)
    assert not msg, "%s: %s" % (CX.case_id(case), msg)


@pytest.mark.parametrize("case", CX.FUSED_CASES, ids=CX.case_id)
def test_conv3x3_heads_tc_exact(lib, case):
    import torch
    D = CX.gen_conv(case)
    c0, c1, n, h, w, R = case["c0"], case["c1"], case["n"], case["h"], case["w"], case["R"]
    src0, src1 = _sources(D, c0)
    wh, wl, b = _dev(D["w_hi"]), _dev(D["w_lo"]), _dev(D["bias"])
    hw, hb = _dev(D["heads_w"]), _dev(D["heads_b"])
    prob = _nan_planes((n, h, w), torch.float32)
    dist = _nan_planes((n, h, w, R), torch.float32)
    _switches(lib, case)
    _call(lib, lib.sdb_conv3x3_heads_tc(_ptr(src0[0]), _ptr(src0[1]), c0, _ptr(src1[0]), _ptr(src1[1]), c1, n, h, w, _ptr(wh), _ptr(wl),
                                        D["w_scale"], _ptr(b), case["relu"], _ptr(hw), _ptr(hb), R, _ptr(prob), _ptr(dist), _st()))
    _, want_p, want_d = CX.fused_ref(case, D)
    msg = CX.first_mismatch(dist.cpu().numpy(), want_d, "dist [n, y, x, ray]") or CX.prob_mismatch(prob.cpu().numpy(), want_p)
    assert not msg, "%s: %s" % (CX.case_id(case), msg)


@pytest.mark.parametrize("case", CX.STEM_CASES, ids=CX.case_id)
def test_stem_split_exact(lib, case):
    import torch
    D = CX.gen_stem(case)
    n, h, w, cout = case["n"], case["h"], case["w"], case["cout"]
    x, k, b = _dev(D["x"]), _dev(D["w"]), _dev(D["bias"])
    out = _nan_planes((2, n, h, w, cout), torch.float16)
    _call(lib, lib.sdb_stem_split(_ptr(x), n, h, w, case["cin"], _ptr(k), _ptr(b), cout, case["relu"], _ptr(out[0]), _ptr(out[1]), _st()))
    want_hi, want_lo = CX.split16(CX.stem_ref(D, case["relu"]))
    got = out.cpu().numpy()
    msg = CX.first_mismatch(got[0], want_hi, "hi plane") or CX.first_mismatch(got[1], want_lo, "lo plane")
    assert not msg, "%s: %s" % (CX.case_id(case), msg)


# ------------------------------------------------------------------------------------------------ split-format companions
def _mixed(rng, shape):
    """random values over some 30 binades (fp16 subnormal lo parts included), inside the fp16 range"""
    return (np.clip(rng.standard_normal(shape), -4, 4) * 10.0 ** rng.uniform(-6, 3.5, shape)).astype(np.float32)


def _bits_equal(got, want, what):
    got = np.asarray(got, np.float16).view(np.int16); want = np.asarray(want, np.float16).view(np.int16)
    bad = np.argwhere(got != want)
    assert len(bad) == 0, "%s: %d elements differ in their bits, first at %s" % (what, len(bad), tuple(bad[0]))


def test_split_f32_is_torch_half_rounding(lib):
    import torch
    x = _mixed(np.random.default_rng(1), (3, 7, 33, 64))
    out = _nan_planes((2,) + x.shape, torch.float16)
    xd = _dev(x)
    _call(lib, lib.sdb_split_f32(_ptr(xd), x.size, _ptr(out[0]), _ptr(out[1]), _st()))
    hi = torch.from_numpy(x).half()
    lo = (torch.from_numpy(x) - hi.float()).half()
    _bits_equal(out[0].cpu().numpy(), hi.numpy(), "hi"); _bits_equal(out[1].cpu().numpy(), lo.numpy(), "lo")


@pytest.mark.parametrize("nd,cin,cout", [(2, 32, 64), (2, 96, 32), (3, 64, 128), (3, 32, 32)])
def test_split_weights_transposes_and_rounds_like_torch(lib, nd, cin, cout):
    import torch
    from stardist_b200.models.unet_device import tc_weight_scale
    rng = np.random.default_rng(cin + cout + nd)
    k = (rng.standard_normal((3,) * nd + (cin, cout)) * 10.0 ** rng.uniform(-4, 0, (3,) * nd + (cin, cout))).astype(np.float32)
    sc = tc_weight_scale(k)
    taps = 3 ** nd
    out = _nan_planes((2, taps, cout, cin), torch.float16)
    fn = lib.sdb_split_weights if nd == 2 else lib.sdb_split_weights_3d
    kd = _dev(k)
    _call(lib, fn(_ptr(kd), cin, cout, sc, _ptr(out[0]), _ptr(out[1]), _st()))
    v = torch.from_numpy(k * np.float32(sc)).reshape(taps, cin, cout).transpose(1, 2)     # [tap][cout][cin]
    hi = v.half(); lo = (v - hi.float()).half()
    _bits_equal(out[0].cpu().numpy(), hi.numpy(), "w_hi"); _bits_equal(out[1].cpu().numpy(), lo.numpy(), "w_lo")


def _random_split(rng, shape):
    import torch
    x = torch.from_numpy(_mixed(rng, shape))
    hi = x.half()
    return hi.numpy(), (x - hi.float()).half().numpy()


@pytest.mark.parametrize("n,h,w,c", [(1, 2, 2, 32), (3, 10, 34, 64), (2, 6, 130, 2)])
def test_maxpool_split_2d(lib, n, h, w, c):
    import torch
    hi, lo = _random_split(np.random.default_rng(h * w + c), (n, h, w, c))
    out = _nan_planes((2, n, h // 2, w // 2, c), torch.float16)
    hd, ld = _dev(hi), _dev(lo)
    _call(lib, lib.sdb_maxpool_split(_ptr(hd), _ptr(ld), n, h, w, c, _ptr(out[0]), _ptr(out[1]), _st()))
    # images are independent: pool (1, 2, 2) over the stacked images
    want_hi, want_lo = CX.maxpool_split_ref(hi, lo, (1, 2, 2))
    got = out.cpu().numpy()
    msg = CX.first_mismatch(got[0], want_hi, "hi") or CX.first_mismatch(got[1], want_lo, "lo")
    assert not msg, msg


@pytest.mark.parametrize("pool", [(2, 2, 2), (1, 2, 2), (2, 1, 1)])
def test_maxpool3d_split(lib, pool):
    import torch
    d, h, w, c = 4, 6, 18, 32
    hi, lo = _random_split(np.random.default_rng(sum(pool)), (d, h, w, c))
    pz, py, px = pool
    out = _nan_planes((2, d // pz, h // py, w // px, c), torch.float16)
    hd, ld = _dev(hi), _dev(lo)
    _call(lib, lib.sdb_maxpool3d_split(_ptr(hd), _ptr(ld), d, h, w, c, pz, py, px, _ptr(out[0]), _ptr(out[1]), _st()))
    want_hi, want_lo = CX.maxpool_split_ref(hi, lo, pool)
    got = out.cpu().numpy()
    msg = CX.first_mismatch(got[0], want_hi, "hi") or CX.first_mismatch(got[1], want_lo, "lo")
    assert not msg, msg


def test_merge_split(lib):
    import torch
    hi, lo = _random_split(np.random.default_rng(5), (5, 13, 29, 32))
    out = _nan_planes(hi.shape, torch.float32)
    hd, ld = _dev(hi), _dev(lo)
    _call(lib, lib.sdb_merge_split(_ptr(hd), _ptr(ld), hi.size, _ptr(out), _st()))
    want = hi.astype(np.float32) + lo.astype(np.float32)
    assert np.array_equal(out.cpu().numpy().view(np.int32), want.view(np.int32))


# ------------------------------------------------------------------------------------------------ range flag, arguments
def _expect_range_flag(lib):
    rc = lib.sdb_tc_error_check(_st())
    assert rc == 2 and "fp16 overflow" in lib.sdb_last_error().decode(), (rc, lib.sdb_last_error())
    assert lib.sdb_tc_error_check(_st()) == 0, "the error word is not cleared by the check that reports it"


def test_range_flag_on_fp16_overflow(lib):
    import torch
    from stardist_b200 import _lib as L
    case = dict(CX.CONV2D_CASES[0], family="conv2d", c0=0, c1=32, cout=32, n=1, h=8, w=16, relu=0, up=0)
    D = CX.gen_conv(case)
    D["bias"][3] = 70000.0                                    # exact, and beyond the fp16 range of the hi plane
    out = torch.zeros((2, 1, 8, 16, 32), dtype=torch.float16, device="cuda")
    xh, xl, wh, wl, b = (_dev(D[k]) for k in ("x_hi", "x_lo", "w_hi", "w_lo", "bias"))
    L.check(lib.sdb_conv3x3_tc(None, None, 0, _ptr(xh), _ptr(xl), 32, 1, 8, 16, _ptr(wh), _ptr(wl), D["w_scale"], _ptr(b), 32, 0, 0,
                               _ptr(out[0]), _ptr(out[1]), _st()))
    _expect_range_flag(lib)


def test_range_flag_on_nan_input(lib):
    import torch
    from stardist_b200 import _lib as L
    x = np.ones((2, 3, 32), np.float32); x[1, 2, 5] = np.nan
    out = torch.zeros((2,) + x.shape, dtype=torch.float16, device="cuda")
    xd = _dev(x)
    L.check(lib.sdb_split_f32(_ptr(xd), x.size, _ptr(out[0]), _ptr(out[1]), _st()))
    _expect_range_flag(lib)


def test_argument_validation_launches_nothing(lib):
    import torch
    from stardist_b200 import _lib as L
    buf = torch.zeros(1 << 16, dtype=torch.float16, device="cuda")
    fb = torch.zeros(1 << 16, dtype=torch.float32, device="cuda")
    p, q = _ptr(buf), _ptr(fb)
    calls = {
        "conv cout 96": lambda: lib.sdb_conv3x3_tc(None, None, 0, p, p, 32, 1, 8, 16, p, p, 16.0, q, 96, 1, 0, p, p, _st()),
        "conv channels 48": lambda: lib.sdb_conv3x3_tc(None, None, 0, p, p, 48, 1, 8, 16, p, p, 16.0, q, 32, 1, 0, p, p, _st()),
        "conv source 0 of 16 channels": lambda: lib.sdb_conv3x3_tc(p, p, 16, p, p, 48, 1, 8, 16, p, p, 16.0, q, 32, 1, 0, p, p, _st()),
        "heads np 64": lambda: lib.sdb_heads_tc(p, p, 64, 1, 8, 16, p, p, 16.0, q, 64, 32, q, q, _st()),
        "fused R 33": lambda: lib.sdb_conv3x3_heads_tc(None, None, 0, p, p, 32, 1, 8, 16, p, p, 16.0, q, 1, q, q, 33, q, q, _st()),
        "3-D conv channels 48": lambda: lib.sdb_conv3x3x3_tc(None, None, 0, p, p, 48, 2, 8, 16, p, p, 16.0, q, 32, 1, 0, p, p, _st()),
        "3-D conv up2x 1": lambda: lib.sdb_conv3x3x3_tc(None, None, 0, p, p, 32, 2, 8, 16, p, p, 16.0, q, 32, 1, 1, p, p, _st()),
    }
    for what, call in calls.items():
        L.launch_count(reset=True)
        rc = call()
        assert rc != 0, what
        assert lib.sdb_last_error().decode(), what
        assert L.launch_count() == 0, "%s launched a kernel" % what
    torch.cuda.synchronize()
    assert lib.sdb_tc_error_check(_st()) == 0


# ------------------------------------------------------------------------------------------------ random-data layer tests
def _split_t(t):
    import torch
    hi = t.to(torch.float16)
    return torch.stack([hi, (t - hi.float()).to(torch.float16)]).contiguous()


@pytest.mark.parametrize("cf,R,shape", [(128, 143, (1, 5 * 12, 37)), (256, 128, (2, 9, 130)), (64, 112, (1, 8, 16))])
def test_heads_tc_random_vs_float64(lib, cf, R, shape):
    import torch
    from stardist_b200 import _lib as L
    from stardist_b200.models.unet_device import tc_weight_scale
    g = torch.Generator().manual_seed(cf + R)
    npd = next(v for v in (48, 80, 112, 144) if v >= R + 1)
    x = torch.relu(torch.randn(shape + (cf,), generator=g)).cuda()
    Wf = torch.zeros((npd, cf)); Wf[:R + 1] = torch.randn((R + 1, cf), generator=g) * (1.0 / cf) ** 0.5
    b = torch.zeros(npd); b[:R + 1] = torch.randn(R + 1, generator=g) * 0.1
    sc = tc_weight_scale(Wf.numpy())
    xs, ws = _split_t(x), _split_t((Wf * sc).cuda())
    bd = b.cuda()
    prob = torch.empty(shape, device="cuda"); dist = torch.empty(shape + (R,), device="cuda")
    _call(lib, lib.sdb_heads_tc(L.ptr(xs[0]), L.ptr(xs[1]), cf, *shape, L.ptr(ws[0]), L.ptr(ws[1]), sc, L.ptr(bd), npd, R,
                                L.ptr(prob), L.ptr(dist), _st()))
    z = (xs[0].double() + xs[1].double()) @ ((ws[0].double() + ws[1].double()) / sc).t() + bd.double()
    wp, wd = torch.sigmoid(z[..., 0]), z[..., 1:R + 1]
    assert (prob.double() - wp).abs().max().item() <= 1e-5
    err, scale = (dist.double() - wd).abs().max().item(), wd.abs().max().item()
    assert err <= 1e-5 * max(1.0, scale), (err, scale)


@pytest.mark.parametrize("c0,c1,R,relu,shape", [(0, 32, 32, 1, (2, 37, 70)), (32, 32, 17, 1, (1, 24, 40)), (0, 64, 7, 0, (1, 9, 130))])
def test_conv3x3_heads_tc_random_vs_float64(lib, c0, c1, R, relu, shape):
    import torch, torch.nn.functional as F
    from stardist_b200 import _lib as L
    from stardist_b200.models.unet_device import tc_weight_scale
    g = torch.Generator().manual_seed(c0 + c1 + R)
    cin = c0 + c1
    x = torch.randn(shape + (cin,), generator=g).cuda()
    k = (torch.randn((3, 3, cin, 128), generator=g) * (2.0 / (9 * cin)) ** 0.5).cuda()
    b = (torch.randn(128, generator=g) * 0.1).cuda()
    hw = torch.zeros((128, 36)); hw[:, :R] = torch.randn((128, R), generator=g) * (1.0 / 128) ** 0.5
    hw[:, 32] = torch.randn(128, generator=g) * (1.0 / 128) ** 0.5
    hb = torch.zeros(36); hb[:R] = torch.randn(R, generator=g) * 0.1; hb[32] = 0.2
    hw, hb = hw.cuda(), hb.cuda()
    xs = _split_t(x)
    sc = tc_weight_scale(k.cpu().numpy())
    ws = torch.empty((2, 9, 128, cin), dtype=torch.float16, device="cuda")
    L.check(lib.sdb_split_weights(L.ptr(k.contiguous()), cin, 128, sc, L.ptr(ws[0]), L.ptr(ws[1]), _st()))
    src1 = xs[..., c0:].contiguous(); src0 = xs[..., :c0].contiguous() if c0 else None
    prob = torch.empty(shape, device="cuda"); dist = torch.empty(shape + (R,), device="cuda")
    _call(lib, lib.sdb_conv3x3_heads_tc(L.ptr(src0[0]) if c0 else None, L.ptr(src0[1]) if c0 else None, c0, L.ptr(src1[0]), L.ptr(src1[1]),
                                        c1, *shape, L.ptr(ws[0]), L.ptr(ws[1]), sc, L.ptr(b), relu, L.ptr(hw), L.ptr(hb), R,
                                        L.ptr(prob), L.ptr(dist), _st()))
    x_eff = (xs[0].double() + xs[1].double()).permute(0, 3, 1, 2)
    k_eff = ((ws[0].double() + ws[1].double()) / sc).reshape(3, 3, 128, cin).permute(2, 3, 0, 1)
    f = F.conv2d(x_eff, k_eff, b.double(), padding=1).permute(0, 2, 3, 1)
    if relu: f = torch.relu(f)
    o = f @ hw.double() + hb.double()
    wp, wd = torch.sigmoid(o[..., 32]), o[..., :R]
    assert (prob.double() - wp).abs().max().item() <= 1e-5
    err, scale = (dist.double() - wd).abs().max().item(), wd.abs().max().item()
    assert err <= 1e-5 * max(1.0, scale), (err, scale)


# ------------------------------------------------------------------------------------------------ network level, 128 rays
def test_unet3d_tc_128_rays_vs_float64():
    """the 3-D network whose heads need the N = 144 instance (Rays_GoldenSpiral(128)) against a float64 evaluation, with the
    bounds of test_gpu_3d.py::test_unet3d_tc_vs_torch_fp32"""
    import torch
    import stardist_b200 as sd
    from oracle import unet_torch
    from stardist_b200.models.unet_device import UNetDevice3DTC
    cfg = sd.Config3D(rays=sd.Rays_GoldenSpiral(128))
    model = sd.StarDist3D(cfg, name=None, basedir=None)
    assert isinstance(model.net, UNetDevice3DTC) and model.net.heads_np == 144
    vol = np.random.default_rng(128).uniform(0, 1, (16, 32, 48)).astype(np.float32)
    prob, dist = model.net.forward(torch.from_numpy(vol[None, ..., None]).cuda())
    rp64, rd64 = unet_torch.forward(cfg, model.weights, vol[None, ..., None], dtype=torch.float64)
    p, dd = prob.cpu().numpy().astype(np.float64), dist.cpu().numpy().astype(np.float64)
    assert p.shape == rp64.shape and dd.shape == rd64.shape
    assert np.max(np.abs(p - rp64)) <= 1e-5 * max(1.0, np.max(np.abs(rp64)))
    err, scale = float(np.max(np.abs(dd - rd64))), float(np.max(np.abs(rd64)))
    assert err <= 1e-5 * max(1.0, scale) and err <= 2e-5 * scale, (err, scale)


def test_c_unet_forward_3d_128_rays_equals_python_executor(lib):
    import torch
    import stardist_b200 as sd
    from stardist_b200 import _lib as L
    cfg = sd.Config3D(rays=sd.Rays_GoldenSpiral(128))
    model = sd.StarDist3D(cfg, name=None, basedir=None)
    x = np.random.default_rng(7).uniform(0, 1, (1, 16, 32, 64, 1)).astype(np.float32)
    net, _ = L.c_unet_create(cfg, model.weights)
    try:
        xd = torch.from_numpy(x).cuda()
        want_p, want_d = model.net.forward(xd)
        sp = tuple(x.shape[1:-1])
        prob = torch.empty(sp, dtype=torch.float32, device="cuda")
        dist = torch.empty(sp + (cfg.n_rays,), dtype=torch.float32, device="cuda")
        L.check(lib._LIB_unet_forward_3d(net, L.ptr(xd), sp[0], sp[1], sp[2], L.ptr(prob), L.ptr(dist), _st()))
        torch.cuda.synchronize()
        assert torch.equal(prob, want_p[0]) and torch.equal(dist, want_d[0])
    finally:
        lib.sdb_unet_destroy(net)
