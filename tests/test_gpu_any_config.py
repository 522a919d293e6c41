"""Models outside the default architecture family on the device (csrc/unet_any.cu and the executors' routing).

Layer level: sdb_conv_any_nd on small-integer operands (every partial sum exact in fp32, tests/any_config_oracle.py
max_partial) must equal the float64 'same' convolution element by element; every activation must be within 8 float32 ulps
of its float64 value plus the effect of one relative rounding (2^-23) of the argument; sdb_heads_any must be within the
fp32 dot-product bound (cf + 1) 2^-24 sum(|b| + |f w|).  Whole models (Glorot weights): prob, dist and prob_class within
1e-5 of the map's maximum of the float64 restatement, labels equal to the oracle pipeline on the same maps, n_tiles equal to
untiled.  Routing guard: the shipped demo models and the benchmark configurations never reach the new kernels."""
import os
import sys

import numpy as np
import pytest

import any_config_oracle as O

pytestmark = pytest.mark.gpu

NEW_ENTRY_POINTS = ('sdb_conv_any_nd', 'sdb_heads_any', 'sdb_maxpool_any_nd', 'sdb_add_act_any')


@pytest.fixture(scope="module")
def lib():
    from stardist_b200 import _lib as L
    return L.require_cuda()


def _dev(a):
    import torch
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _nan(shape):
    import torch
    return torch.full(tuple(shape), float("nan"), dtype=torch.float32, device="cuda")


def _call(rc):
    import torch
    from stardist_b200 import _lib as L
    L.check(rc)
    torch.cuda.synchronize()


def _conv_any(lib, x, lo, k, b, stride, up, act):
    """sdb_conv_any_nd on numpy operands; x [n, *sp, c_skip] (2-D or 3-D)"""
    from stardist_b200 import _lib as L
    from stardist_b200.models.unet_device import act_id
    nd = x.ndim - 2
    n = x.shape[0]
    d, h, w = ((1,) + x.shape[1:3]) if nd == 2 else x.shape[1:4]
    ks, ss, us = tuple(k.shape[:nd]), tuple(stride), tuple(up)
    if nd == 2:
        ks, ss, us = (1,) + ks, (1,) + ss, (1,) + us
    cout = k.shape[-1]
    osp = tuple(-(-s // t) for s, t in zip(x.shape[1:-1], stride))
    out = _nan((n,) + osp + (cout,))
    c_lo = 0 if lo is None else lo.shape[-1]
    xd, lod, kd, bd = _dev(x), _dev(lo), _dev(k), _dev(b)
    _call(lib.sdb_conv_any_nd(L.ptr(xd), L.ptr(lod), n, d, h, w, x.shape[-1], c_lo, *us, L.ptr(kd), L.ptr(bd), cout, *ks, *ss,
                              act_id(act), L.ptr(out), L.stream_ptr()))
    return out.cpu().numpy()


# ------------------------------------------------------------------------------------------------ layer-exact
@pytest.mark.parametrize("case", O.CONV_CASES, ids=lambda c: c['id'])
def test_conv_any_exact(lib, case):
    skip, lo, k, b = O.gen_conv(case)
    got = _conv_any(lib, skip, lo, k, b, case['s'], case['up'], case['act'])
    want = O.conv_ref(case, skip, lo, k, b)
    assert got.shape == want.shape
    bad = np.argwhere(~(got == want))
    assert len(bad) == 0, "%d mismatches, first at %s: %r != %r" % (len(bad), bad[0], got[tuple(bad[0])], want[tuple(bad[0])])


def test_maxpool_and_add_any_exact(lib):
    import torch
    from stardist_b200 import _lib as L
    rng = np.random.default_rng(5)
    for shape, pool in (((2, 1, 12, 18, 7), (1, 2, 3)), ((1, 4, 6, 8, 5), (2, 2, 2)), ((1, 1, 8, 8, 1), (1, 1, 2))):
        x = rng.integers(-50, 50, size=shape).astype(np.float32)
        n, d, h, w, c = shape
        out, xd = _nan((n, d // pool[0], h // pool[1], w // pool[2], c)), _dev(x)
        _call(lib.sdb_maxpool_any_nd(L.ptr(xd), n, d, h, w, c, *pool, L.ptr(out), L.stream_ptr()))
        want = O.maxpool(torch.from_numpy(x).double().reshape(n, d, h, w, c), pool).numpy()
        assert np.array_equal(out.cpu().numpy(), want)
    a = rng.integers(-50, 50, size=1001).astype(np.float32); bb = rng.integers(-50, 50, size=1001).astype(np.float32)
    ad, bd = _dev(a), _dev(bb)
    for act in ('relu', 'linear'):
        from stardist_b200.models.unet_device import act_id
        out = _nan((1001,))
        _call(lib.sdb_add_act_any(L.ptr(ad), L.ptr(bd), 1001, act_id(act), L.ptr(out), L.stream_ptr()))
        assert np.array_equal(out.cpu().numpy(), O.act64(act, torch.from_numpy(a + bb).double()).numpy())


def _act_inputs():
    x = np.linspace(-30, 30, 6001, dtype=np.float64)
    x = np.concatenate([x, [-1e-6, -1e-30, 0.0, 1e-30, 1e-6, -13.9423847, 13.9423847, -14.5, 14.5]])
    return x.astype(np.float32)


@pytest.mark.parametrize("act", O.ACTS)
def test_activations_vs_float64(lib, act):
    """each activation through the convolution's epilogue (1x1, weight 1, bias 0) and through the residual sum (b = 0)"""
    import torch
    from stardist_b200 import _lib as L
    from stardist_b200.models.unet_device import act_id
    x = _act_inputs()
    f = lambda v: O.act64(act, torch.from_numpy(np.asarray(v, np.float64))).numpy()
    want = f(x)
    sens = np.maximum(np.abs(f(x.astype(np.float64) * (1 + 2.0 ** -23)) - want), np.abs(f(x.astype(np.float64) * (1 - 2.0 ** -23)) - want))
    bound = 8 * np.spacing(np.abs(want).astype(np.float32)).astype(np.float64) + sens
    conv = _conv_any(lib, x.reshape(1, 1, -1, 1), None, np.ones((1, 1, 1, 1), np.float32), np.zeros(1, np.float32),
                     (1, 1), (1, 1), act).reshape(-1)
    out, xd, zd = _nan(x.shape), _dev(x), _dev(np.zeros_like(x))
    _call(lib.sdb_add_act_any(L.ptr(xd), L.ptr(zd), x.size, act_id(act), L.ptr(out), L.stream_ptr()))
    for name, got in (('conv', conv), ('add_act', out.cpu().numpy())):
        err = np.abs(got.astype(np.float64) - want)
        i = int(np.argmax(err - bound))
        assert np.all(err <= bound), "%s/%s: x=%r got %r want %r (bound %g)" % (act, name, x[i], got[i], want[i], bound[i])


@pytest.mark.parametrize("cf", [1, 32, 64, 256])
@pytest.mark.parametrize("R", [1, 17, 64, 128])
def test_heads_any_vs_float64(lib, cf, R):
    from stardist_b200 import _lib as L
    rng = np.random.default_rng(cf * 1000 + R)
    npix = 777
    f = rng.standard_normal((npix, cf)).astype(np.float32)
    wp = rng.standard_normal((cf, 1)).astype(np.float32); bp = rng.standard_normal(1).astype(np.float32)
    wd = rng.standard_normal((cf, R)).astype(np.float32); bd = rng.standard_normal(R).astype(np.float32)
    prob, dist = _nan((npix,)), _nan((npix, R))
    dev = [_dev(a) for a in (f, wp, bp, wd, bd)]          # kept alive until the launch completed
    _call(lib.sdb_heads_any(L.ptr(dev[0]), npix, cf, *[L.ptr(t) for t in dev[1:]], R, L.ptr(prob), L.ptr(dist), L.stream_ptr()))
    F64 = f.astype(np.float64)
    W = np.concatenate([wp, wd], 1).astype(np.float64); B = np.concatenate([bp, bd]).astype(np.float64)
    z = F64 @ W + B
    gamma = (cf + 1) * 2.0 ** -24 / (1 - (cf + 1) * 2.0 ** -24)
    bound = gamma * (np.abs(F64) @ np.abs(W) + np.abs(B))
    d = dist.cpu().numpy().astype(np.float64)
    assert np.all(np.abs(d - z[:, 1:]) <= bound[:, 1:])
    p = prob.cpu().numpy().astype(np.float64)
    pw = 1 / (1 + np.exp(-z[:, 0]))
    assert np.all(np.abs(p - pw) <= 0.25 * bound[:, 0] + 4 * np.spacing(pw.astype(np.float32)))


# ------------------------------------------------------------------------------------------------ whole models
def _configs():
    from stardist_b200 import Config2D, Config3D, Rays_GoldenSpiral
    r3 = dict(rays=Rays_GoldenSpiral(32))
    return {
        'base16': Config2D(unet_n_filter_base=16),
        'after0': Config2D(net_conv_after_unet=0),
        'after256': Config2D(net_conv_after_unet=256, n_rays=64, grid=(2, 2)),
        'k55_elu': Config2D(unet_kernel_size=(5, 5), unet_activation='elu', unet_last_activation='linear'),
        'cin5_swish': Config2D(n_channel_in=5, unet_n_filter_base=24, unet_activation='swish'),
        'classes3': Config2D(n_classes=3, net_conv_after_unet=64),
        '3d_k133': Config3D(unet_n_filter_base=16, unet_kernel_size=(1, 3, 3), unet_pool=(1, 2, 2), grid=(1, 2, 2), **r3),
        '3d_resnet': Config3D(backbone='resnet', resnet_n_filter_base=16, resnet_activation='elu', net_conv_after_resnet=64,
                              grid=(1, 2, 2), **r3),
    }


def _model(name):
    from stardist_b200 import StarDist2D, StarDist3D
    config = _configs()[name]
    model = (StarDist2D if config.n_dim == 2 else StarDist3D)(config, name=None, basedir=None)
    # a usable dist head for the random-init body: bias 4 -> star-convex shapes of radius ~4 pixels
    k, b = model.weights['dist']
    model.weights['dist'] = (k, b + np.float32(4.0))
    return model


def _image(config, seed=0):
    rng = np.random.default_rng(seed)
    shape = (128, 160) if config.n_dim == 2 else (12, 64, 80)
    c = () if config.n_channel_in == 1 else (config.n_channel_in,)
    return rng.uniform(0, 1, shape + c).astype(np.float32)


@pytest.mark.parametrize("name", list(_configs()))
def test_whole_model_maps_vs_float64(lib, name):
    import torch
    model = _model(name)
    img = _image(model.config)
    x = img if img.ndim == model.config.n_dim + 1 else img[..., None]
    prob, dist = model.net.forward(torch.from_numpy(x[None]).cuda())
    rp, rd, rc = O.forward(model.config, model.weights, x[None], device='cuda')
    for got, want, what in ((prob, rp, 'prob'), (dist, rd, 'dist'), (model.net.prob_class, rc, 'prob_class')):
        if want is None:
            assert got is None
            continue
        got = got.cpu().numpy()
        assert got.shape == want.shape, what
        err = np.max(np.abs(got - want))
        assert err <= 1e-5 * np.max(np.abs(want)), "%s %s: max error %g, max |map| %g" % (name, what, err, np.max(np.abs(want)))
    assert model.config.n_classes is None or model.net.prob_class is not None


@pytest.mark.parametrize("name", list(_configs()))
def test_whole_model_labels_vs_oracle_pipeline(lib, name):
    from oracle import ref_ext
    model = _model(name)
    img = _image(model.config, seed=1)
    prob = model.predict(img)[0]
    pthr = float(np.quantile(prob, 0.97))
    labels, res = model.predict_instances(img, prob_thresh=pthr, nms_thresh=0.3)
    shape = img.shape[:model.config.n_dim]
    assert labels.shape == shape and len(res['prob']) > 2
    if model.config.n_dim == 2:
        from oracle import pipeline2d
        ref_labels, ref = pipeline2d.predict_instances(model.config, model.weights, img[..., 0] if img.ndim == 3 else img, pthr, 0.3,
                                                       cand_from=model)
    else:
        if not ref_ext.available():
            pytest.skip("oracle/_ref not present")
        os.environ["OMP_NUM_THREADS"] = "1"
        from oracle import pipeline3d
        from stardist_b200.rays3d import rays_from_json
        rays = rays_from_json(model.config.rays_json)
        ref_labels, ref = pipeline3d.predict_instances(model.config, rays, img, pthr, 0.3, cand_from=model)
    assert np.array_equal(res['points'], ref['points'])
    assert np.array_equal(res['prob'], ref['prob'])
    assert np.array_equal(labels, ref_labels)


@pytest.mark.parametrize("name,n_tiles", [('k55_elu', (2, 3)), ('3d_k133', (1, 2, 2))])
def test_n_tiles_equals_untiled(lib, name, n_tiles):
    model = _model(name)
    rng = np.random.default_rng(9)
    img = rng.uniform(0, 1, (256, 224) if model.config.n_dim == 2 else (16, 128, 96)).astype(np.float32)
    p1, d1 = model.predict(img)
    p2, d2 = model.predict(img, n_tiles=n_tiles)
    assert p1.shape == p2.shape and d1.shape == d2.shape
    assert np.max(np.abs(p1 - p2)) <= 1e-5 and np.max(np.abs(d1 - d2)) <= 1e-5 * max(1e-3, np.max(np.abs(d1))) + 1e-7


# ------------------------------------------------------------------------------------------------ routing guard
@pytest.fixture
def counted(lib, monkeypatch):
    """call counts of the csrc/unet_any.cu entry points"""
    calls = {n: 0 for n in NEW_ENTRY_POINTS}
    for n in NEW_ENTRY_POINTS:
        fn = getattr(lib, n)

        def wrap(*a, _fn=fn, _n=n):
            calls[_n] += 1
            return _fn(*a)
        monkeypatch.setattr(lib, n, wrap)
    return calls


def test_demo_and_bench_models_never_reach_the_new_kernels(counted):
    import stardist_b200 as sd
    from stardist_b200.utils import normalize
    from stardist_b200.rays3d import rays_from_json
    from stardist_b200.models.unet_device import UNetDeviceND
    root = os.path.dirname(os.path.abspath(__file__))
    sys.path.insert(0, os.path.join(root, "golden"))
    sys.path.insert(0, os.path.dirname(root))
    import demo2d, demo3d, bench_data
    kwargs, weights, thr, img, _ = demo2d.load()
    m2 = sd.StarDist2D(sd.Config2D(**kwargs), name=None, basedir=None, weights=weights)
    m2.predict_instances(normalize(img, 1, 99.8), prob_thresh=thr['prob'], nms_thresh=thr['nms'])
    m2s = sd.StarDist2D(sd.Config2D(**kwargs), name=None, basedir=None, weights=weights)
    m2s._net = UNetDeviceND(m2s.config, m2s.weights)          # the CUDA-core executor too
    m2s.predict(normalize(img, 1, 99.8)[:256, :256])
    rays_json, kwargs, weights, thr, img, _ = demo3d.load()
    m3 = sd.StarDist3D(sd.Config3D(rays=rays_from_json(rays_json), **kwargs), name=None, basedir=None, weights=weights)
    m3.predict_instances(normalize(img, 1, 99.8), prob_thresh=thr['prob'], nms_thresh=thr['nms'])
    c2 = sd.Config2D(n_rays=32)
    b2 = sd.StarDist2D(c2, name=None, basedir=None, weights=bench_data.bench_weights_2d(c2))
    b2.predict_instances(bench_data.synthetic_image((256, 256), seed=0)[0], prob_thresh=0.5, nms_thresh=0.4)
    c3 = bench_data.bench_config_3d(96)
    b3 = sd.StarDist3D(c3, name=None, basedir=None, weights=bench_data.bench_weights_3d(c3))
    b3.predict_instances(bench_data.synthetic_volume((32, 96, 96), seed=0)[0], prob_thresh=0.5, nms_thresh=0.4)
    assert counted == {n: 0 for n in NEW_ENTRY_POINTS}


def test_new_configurations_reach_the_new_kernels(counted):
    """the counting itself works: configurations outside the default family call them"""
    import torch
    for name, entry in (('base16', 'sdb_conv_any_nd'), ('after0', 'sdb_heads_any')):
        model = _model(name)
        model.net.forward(torch.from_numpy(_image(model.config)[None, ..., None]).cuda())
        assert counted[entry] > 0, name
