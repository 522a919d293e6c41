"""Layer tests of the fp32 CUDA-core network kernels (csrc/unet_simt.cu) on exactly representable operands
(tests/simtexact.py): every partial sum is exact in fp32, so the convolutions (tiled, stem and generic), pooling, the
residual sum and the dist head must equal their float64 references element by element.  prob must be within 4 float32 ulps
of the float64 sigmoid and prob_class within the operation-count bound of simtexact.class_head_ulps.  Every output starts
as NaN, so an element no thread writes fails.  Also: the 2-D wrappers, and argument validation that launches nothing."""
import numpy as np
import pytest

import simtexact as SX

pytestmark = pytest.mark.gpu


@pytest.fixture
def lib():
    from stardist_b200 import _lib as L
    return L.require_cuda()


def _dev(a):
    import torch
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _ptr(t):
    from stardist_b200 import _lib as L
    return L.ptr(t)


def _st():
    from stardist_b200 import _lib as L
    return L.stream_ptr()


def _nan(shape):
    import torch
    return torch.full(shape, float("nan"), dtype=torch.float32, device="cuda")


def _call(rc):
    """a launch that must succeed and complete without a device error"""
    import torch
    from stardist_b200 import _lib as L
    L.check(rc)
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ exact layer tests
def _conv3(lib, case, D):
    n, d, h, w, cout = case["n"], case["d"], case["h"], case["w"], case["cout"]
    x, lo, k, b = _dev(D["skip"]), _dev(D["lo"]), _dev(D["w"]), _dev(D["bias"])
    uz, uy, ux = case["up"]
    out = _nan((n, d, h, w, cout))
    _call(lib.sdb_conv3_nd(_ptr(x), _ptr(lo), n, d, h, w, case["cin_skip"], case["cin_lo"], uz, uy, ux, _ptr(k), _ptr(b), cout,
                           case["kz"], case["relu"], _ptr(out), _st()))
    return out.cpu().numpy()


@pytest.mark.parametrize("case", SX.CONV_CASES + SX.STEM_CASES, ids=SX.case_id)
def test_conv3_nd_exact(lib, case):
    D = SX.gen(case)
    msg = SX.first_mismatch(_conv3(lib, case, D), SX.conv3_ref(case, D), "out [n, z, y, x, c]")
    assert not msg, "%s (%s): %s" % (SX.case_id(case), SX.instance(case), msg)


@pytest.mark.parametrize("case", SX.GENERIC_CASES, ids=SX.case_id)
def test_conv_generic_nd_exact(lib, case):
    D = SX.gen(case)
    n, d, h, w, cin, cout = case["n"], case["d"], case["h"], case["w"], case["cin"], case["cout"]
    (kz, ky, kx), (sz, sy, sx) = case["k"], case["s"]
    x, k, b = _dev(D["x"]), _dev(D["w"]), _dev(D["bias"])
    out = _nan((n, -(-d // sz), -(-h // sy), -(-w // sx), cout))
    _call(lib.sdb_conv_generic_nd(_ptr(x), n, d, h, w, cin, _ptr(k), _ptr(b), cout, kz, ky, kx, sz, sy, sx, case["relu"],
                                  _ptr(out), _st()))
    msg = SX.first_mismatch(out.cpu().numpy(), SX.generic_ref(case, D), "out [n, z, y, x, c]")
    assert not msg, "%s: %s" % (SX.case_id(case), msg)


@pytest.mark.parametrize("case", SX.MAXPOOL_CASES, ids=SX.case_id)
def test_maxpool_nd_exact(lib, case):
    D = SX.gen(case)
    n, d, h, w, c = case["n"], case["d"], case["h"], case["w"], case["c"]
    pz, py, px = case["pool"]
    x = _dev(D["x"])
    out = _nan((n, d // pz, h // py, w // px, c))
    _call(lib.sdb_maxpool_nd(_ptr(x), n, d, h, w, c, pz, py, px, _ptr(out), _st()))
    msg = SX.first_mismatch(out.cpu().numpy(), SX.maxpool_ref(case, D), "out [n, z, y, x, c]")
    assert not msg, "%s: %s" % (SX.case_id(case), msg)


@pytest.mark.parametrize("case", SX.ADD_CASES, ids=SX.case_id)
def test_add_act_exact(lib, case):
    D = SX.gen(case)
    a, b = _dev(D["a"]), _dev(D["b"])
    out = _nan((case["size"],))
    _call(lib.sdb_add_act(_ptr(a), _ptr(b), case["size"], case["relu"], _ptr(out), _st()))
    msg = SX.first_mismatch(out.cpu().numpy(), SX.add_ref(case, D), "out")
    assert not msg, "%s: %s" % (SX.case_id(case), msg)


@pytest.mark.parametrize("case", SX.HEADS_CASES, ids=SX.case_id)
def test_heads_2d_exact(lib, case):
    D = SX.gen(case)
    npix, R = case["npix"], case["R"]
    f, wp, bp, wd, bd = (_dev(D[k]) for k in ("feat", "wp", "bp", "wd", "bd"))
    prob, dist = _nan((npix,)), _nan((npix, R))
    _call(lib.sdb_heads_2d(_ptr(f), npix, 128, _ptr(wp), _ptr(bp), _ptr(wd), _ptr(bd), R, _ptr(prob), _ptr(dist), _st()))
    want_p, want_d = SX.heads_ref(case, D)
    msg = SX.first_mismatch(dist.cpu().numpy(), want_d, "dist [pixel, ray]") or SX.prob_mismatch(prob.cpu().numpy(), want_p)
    assert not msg, "%s: %s" % (SX.case_id(case), msg)


@pytest.mark.parametrize("case", SX.CLASS_CASES, ids=SX.case_id)
def test_class_head_within_bound(lib, case):
    D = SX.gen(case)
    npix, cf, C = case["npix"], case["cf"], case["C"]
    f, w, b = _dev(D["feat"]), _dev(D["w"]), _dev(D["bias"])
    out = _nan((npix, C))
    _call(lib.sdb_class_head(_ptr(f), npix, cf, _ptr(w), _ptr(b), C, _ptr(out), _st()))
    msg = SX.softmax_mismatch(out.cpu().numpy(), SX.class_ref(case, D), C)
    assert not msg, "%s (bound %d ulps): %s" % (SX.case_id(case), SX.class_head_ulps(C), msg)


def test_conv3x3_2d_wrapper(lib):
    """sdb_conv3x3_2d = sdb_conv3_nd with d 1, kz 1 and a 2x2 up-sampled source"""
    case = dict(family="conv", cin_skip=16, cin_lo=8, up=(1, 2, 2), cout=96, kz=1, n=2, d=1, h=18, w=34, relu=1, seed=7100)
    D = SX.gen(case)
    x, lo, k, b = _dev(D["skip"]), _dev(D["lo"]), _dev(D["w"]), _dev(D["bias"])
    out = _nan((2, 18, 34, 96))
    _call(lib.sdb_conv3x3_2d(_ptr(x), _ptr(lo), 2, 18, 34, 16, 8, _ptr(k), _ptr(b), 96, 1, _ptr(out), _st()))
    msg = SX.first_mismatch(out.cpu().numpy(), SX.conv3_ref(case, D)[:, 0], "out [n, y, x, c]")
    assert not msg, msg


def test_maxpool2x2_2d_wrapper(lib):
    case = dict(family="maxpool", pool=(1, 2, 2), c=12, n=3, d=1, h=10, w=34, seed=7101)
    D = SX.gen(case)
    x = _dev(D["x"][:, 0])
    out = _nan((3, 5, 17, 12))
    _call(lib.sdb_maxpool2x2_2d(_ptr(x), 3, 10, 34, 12, _ptr(out), _st()))
    msg = SX.first_mismatch(out.cpu().numpy(), SX.maxpool_ref(case, D)[:, 0], "out [n, y, x, c]")
    assert not msg, msg


# ------------------------------------------------------------------------------------------------ arguments
def _zeros(n):
    import torch
    return torch.zeros(max(int(n), 1), dtype=torch.float32, device="cuda")


def _conv3_call(lib, n, d, h, w, cs, cl, up, cout, kz, lo=True):
    """sdb_conv3_nd on zero buffers as large as the call describes (so a missing check computes garbage in bounds)"""
    uz, uy, ux = up
    x, y = _zeros(n * d * h * w * cs), _zeros(n * d * h * w * cout)
    xl = _zeros(n * d * h * w * cl) if lo else None
    k, b = _zeros(max(kz, 3) * 9 * (cs + cl) * cout), _zeros(cout)
    return lambda: lib.sdb_conv3_nd(_ptr(x), _ptr(xl), n, d, h, w, cs, cl, uz, uy, ux, _ptr(k), _ptr(b), cout, kz, 1, _ptr(y), _st())


def _rejections(lib):
    calls = {
        "conv3_nd kz 2": (_conv3_call(lib, 1, 4, 8, 8, 8, 0, (1, 1, 1), 32, 2), "kz must be 1 or 3"),
        "conv3_nd kz 1 with d 2": (_conv3_call(lib, 1, 2, 8, 8, 8, 0, (1, 1, 1), 32, 1), "d == 1"),
        "conv3_nd cin_lo without in_lo": (_conv3_call(lib, 1, 1, 8, 8, 8, 8, (1, 2, 2), 32, 1, lo=False), "cin_lo without in_lo"),
        "conv3_nd stem cout 48": (_conv3_call(lib, 1, 1, 8, 8, 1, 0, (1, 1, 1), 48, 1), "stem supports cout 32 or 64"),
        "conv3_nd stem cout 128": (_conv3_call(lib, 1, 2, 8, 8, 4, 0, (1, 1, 1), 128, 3), "stem supports cout 32 or 64"),
        "conv3_nd cin_skip 12": (_conv3_call(lib, 1, 1, 8, 8, 12, 0, (1, 1, 1), 32, 1), "multiples of 8"),
        "conv3_nd cin_lo 4": (_conv3_call(lib, 1, 1, 8, 8, 8, 4, (1, 2, 2), 32, 1), "multiples of 8"),
        "conv3_nd cout 48": (_conv3_call(lib, 1, 1, 8, 8, 8, 0, (1, 1, 1), 48, 1), "multiples of 8"),
        "conv3_nd h 9 with uy 2": (_conv3_call(lib, 1, 1, 9, 8, 8, 8, (1, 2, 2), 32, 1), "not divisible by the up-sampling"),
        "conv3_nd d 3 with uz 2": (_conv3_call(lib, 1, 3, 8, 8, 8, 8, (2, 2, 2), 32, 3), "not divisible by the up-sampling"),
        "conv3_nd up factor 0": (_conv3_call(lib, 1, 1, 8, 8, 8, 8, (1, 0, 2), 32, 1), "not divisible by the up-sampling"),
        "conv3_nd 65552 z tiles": (_conv3_call(lib, 1, 4097, 1, 1, 8, 0, (1, 1, 1), 1024, 3), "grid.z too large"),
    }
    x, lo, k, b, y = _zeros(2 * 9 * 8 * 16), _zeros(9 * 4 * 8), _zeros(9 * 16 * 32), _zeros(32), _zeros(2 * 9 * 8 * 32)
    calls["conv3x3_2d odd h with up-sampled source"] = (
        lambda: lib.sdb_conv3x3_2d(_ptr(x), _ptr(lo), 2, 9, 8, 8, 8, _ptr(k), _ptr(b), 32, 1, _ptr(y), _st()), "even h, w")
    p_in, p_out = _zeros(2 * 5 * 8 * 6 * 8), _zeros(2 * 5 * 8 * 6 * 8)
    calls["maxpool_nd h 5 with py 2"] = (lambda: lib.sdb_maxpool_nd(_ptr(p_in), 2, 1, 5, 8, 8, 1, 2, 2, _ptr(p_out), _st()), "divisible")
    calls["maxpool_nd c 6"] = (lambda: lib.sdb_maxpool_nd(_ptr(p_in), 1, 2, 8, 6, 6, 2, 2, 2, _ptr(p_out), _st()), "c % 4")
    calls["maxpool_nd pool 0"] = (lambda: lib.sdb_maxpool_nd(_ptr(p_in), 1, 2, 8, 6, 8, 0, 2, 2, _ptr(p_out), _st()), "divisible")
    npix = 100
    for cf, R, what in ((64, 32, "only 128 feature channels"), (256, 32, "only 128 feature channels"), (128, 294, "n_rays too large")):
        f, wp, bp, wd, bd = _zeros(npix * cf), _zeros(cf), _zeros(1), _zeros(cf * R), _zeros(R)
        pr, di = _zeros(npix), _zeros(npix * R)
        calls["heads_2d cfeat %d R %d" % (cf, R)] = (
            lambda f=f, wp=wp, bp=bp, wd=wd, bd=bd, pr=pr, di=di, cf=cf, R=R:
            lib.sdb_heads_2d(_ptr(f), npix, cf, _ptr(wp), _ptr(bp), _ptr(wd), _ptr(bd), R, _ptr(pr), _ptr(di), _st()), what)
    for cf, C, what in ((128, 33, "[1,32]"), (128, 0, "[1,32]"), (512, 32, "weight table too large")):
        f, w, b2, o = _zeros(npix * cf), _zeros(cf * C), _zeros(C), _zeros(npix * C)
        calls["class_head cfeat %d n_out %d" % (cf, C)] = (
            lambda f=f, w=w, b2=b2, o=o, cf=cf, C=C: lib.sdb_class_head(_ptr(f), npix, cf, _ptr(w), _ptr(b2), C, _ptr(o), _st()), what)
    g = _zeros(1 << 16)
    for i, bad in enumerate(("n", "d", "h", "w", "cin", "cout", "kz", "ky", "kx", "sz", "sy", "sx")):
        args = dict(n=1, d=2, h=3, w=4, cin=2, cout=3, kz=1, ky=3, kx=3, sz=1, sy=2, sx=2)
        args[bad] = 0 if i % 2 else -1
        calls["conv_generic_nd %s %d" % (bad, args[bad])] = (
            lambda a=args: lib.sdb_conv_generic_nd(_ptr(g), a["n"], a["d"], a["h"], a["w"], a["cin"], _ptr(g), _ptr(g), a["cout"],
                                                a["kz"], a["ky"], a["kx"], a["sz"], a["sy"], a["sx"], 0, _ptr(g), _st()), "bad arguments")
    return calls


def test_argument_validation_launches_nothing(lib):
    """each rejected call returns non-zero, says why in sdb_last_error() and launches no kernel"""
    import torch
    from stardist_b200 import _lib as L
    calls = _rejections(lib)
    torch.cuda.synchronize()
    for what, (call, why) in calls.items():
        L.launch_count(reset=True)
        rc = call()
        err = lib.sdb_last_error().decode()
        assert rc != 0, what
        assert why in err, "%s: sdb_last_error() = %r" % (what, err)
        assert L.launch_count() == 0, "%s launched a kernel" % what
    torch.cuda.synchronize()
