"""Training on the device (stardist_b200/models/train.py, csrc/unet_train.cu): layer-exact backward kernels on exactly
representable data, the loss kernel against the float64 restatement, whole-network gradients against float64 torch
autograd on real StarDistData batches, Adam against its float32 numpy restatement, run-to-run determinism and an
end-to-end train() on synthetic ellipses."""
import os, sys, warnings
import numpy as np
import pytest
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import train_oracle as O
from train_cpu_cases import EXACT_WGRAD, EXACT_DECODER, int_data

pytestmark = pytest.mark.gpu


def _lib():
    from stardist_b200 import _lib as L
    return L, L.require_cuda()


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


def _to_torch_layout(k):
    nd = k.ndim - 2
    return torch.from_numpy(k.astype(np.float64)).permute(nd + 1, nd, *range(nd)).contiguous()


# ------------------------------------------------------------------------------------------------ layer-exact kernels
@pytest.mark.parametrize("case", EXACT_WGRAD, ids=lambda c: c['id'])
def test_conv_wgrad_and_dgrad_exact(case):
    """dW, db (sdb_conv_wgrad_nd) and dX (sdb_conv3_nd on the flipped kernel) bit-equal to float64 autograd"""
    L, lib = _lib()
    nd, shape, cin, cout = case['nd'], case['shape'], case['cin'], case['cout']
    x, dy, k = int_data(case)
    conv = F.conv2d if nd == 2 else F.conv3d
    xt = torch.from_numpy(x.astype(np.float64)).permute(0, nd + 1, *range(1, nd + 1)).requires_grad_(True)
    kt = _to_torch_layout(k).requires_grad_(True)
    bt = torch.zeros(cout, dtype=torch.float64, requires_grad=True)
    y = conv(xt, kt, bt, padding='same')
    y.backward(torch.from_numpy(dy.astype(np.float64)).permute(0, nd + 1, *range(1, nd + 1)))
    want_dw = kt.grad.permute(*range(2, nd + 2), 1, 0).numpy()
    want_dx = xt.grad.permute(0, *range(2, nd + 2), 1).numpy()
    d, h, w = ((1,) + shape) if nd == 2 else shape
    n = x.shape[0]
    dx_, dy_, k_ = _dev(x), _dev(dy), _dev(k)
    taps = 3 ** nd
    need = int(lib.sdb_conv_wgrad_workspace(n * d * h * w, taps, cin, cout))
    work = torch.empty(need, dtype=torch.float32, device='cuda')
    dw = torch.empty(k.shape, dtype=torch.float32, device='cuda'); db = torch.empty(cout, dtype=torch.float32, device='cuda')
    L.check(lib.sdb_conv_wgrad_nd(L.ptr(dx_), None, n, d, h, w, cin, 0, 1, 1, 1, 3 if nd == 3 else 1, 3, L.ptr(dy_), cout, cout,
                                  L.ptr(work), need, L.ptr(dw), L.ptr(db), L.stream_ptr()))
    assert np.array_equal(dw.cpu().numpy().astype(np.float64), want_dw)
    assert np.array_equal(db.cpu().numpy().astype(np.float64), bt.grad.numpy())
    if cin % 32 == 0:
        wf = torch.empty((taps, cout, cin), dtype=torch.float32, device='cuda')
        L.check(lib.sdb_conv_flip_weights(L.ptr(k_), taps, cin, cout, L.ptr(wf), L.stream_ptr()))
        zb = torch.zeros(cin, dtype=torch.float32, device='cuda')
        dx = torch.empty(x.shape, dtype=torch.float32, device='cuda')
        L.check(lib.sdb_conv3_nd(L.ptr(dy_), None, n, d, h, w, cout, 0, 1, 1, 1, L.ptr(wf), L.ptr(zb), cin, 1 if nd == 2 else 3, 0,
                                 L.ptr(dx), L.stream_ptr()))
        assert np.array_equal(dx.cpu().numpy().astype(np.float64), want_dx)


@pytest.mark.parametrize("case", EXACT_DECODER, ids=lambda c: c['id'])
def test_decoder_layer_backward_exact(case):
    """decoder convolution over [upsample(x_lo), skip]: wgrad through the loader's address math, dgrad, the decoder split
    (the backward of nearest up-sampling) and max-pool + ReLU backward of the skip's producer, bit-equal to autograd"""
    L, lib = _lib()
    nd, shape, up = case['nd'], case['shape'], case['up']
    c_lo, c_skip, cout = case['c_lo'], case['c_skip'], case['cout']
    rng = np.random.default_rng(case['seed'])
    lo_shape = tuple(s // u for s, u in zip(shape, up))
    n = 2
    skip_pre = rng.integers(-2, 3, (n,) + shape + (c_skip,)).astype(np.float32)         # pre-ReLU values of the skip
    skip = np.maximum(skip_pre, 0)
    lo = rng.integers(-2, 3, (n,) + lo_shape + (c_lo,)).astype(np.float32)
    k = rng.integers(-2, 3, (3,) * nd + (c_lo + c_skip, cout)).astype(np.float32)
    dy = rng.integers(-2, 3, (n,) + shape + (cout,)).astype(np.float32)
    pool = up
    gpool = rng.integers(-2, 3, (n,) + lo_shape + (c_skip,)).astype(np.float32)           # gradient arriving through max-pool
    conv = F.conv2d if nd == 2 else F.conv3d
    mp = F.max_pool2d if nd == 2 else F.max_pool3d
    cf = lambda a: torch.from_numpy(a.astype(np.float64)).permute(0, nd + 1, *range(1, nd + 1))
    spre = cf(skip_pre).requires_grad_(True)
    lot = cf(lo).requires_grad_(True)
    kt = _to_torch_layout(k).requires_grad_(True)
    s_ = F.relu(spre)
    cat = torch.cat([F.interpolate(lot, scale_factor=tuple(float(u) for u in up), mode='nearest'), s_], dim=1)
    y = conv(cat, kt, torch.zeros(cout, dtype=torch.float64), padding='same')
    loss = (y * cf(dy)).sum() + (mp(s_, tuple(pool)) * cf(gpool)).sum()
    loss.backward()
    d, h, w = ((1,) + shape) if nd == 2 else shape
    uz, uy, ux = ((1,) + tuple(up)) if nd == 2 else tuple(up)
    skd, lod, kd, dyd, gpd = _dev(skip), _dev(lo), _dev(k), _dev(dy), _dev(gpool)
    taps, cin = 3 ** nd, c_lo + c_skip
    need = int(lib.sdb_conv_wgrad_workspace(n * d * h * w, taps, cin, cout))
    work = torch.empty(need, dtype=torch.float32, device='cuda')
    dw = torch.empty(k.shape, dtype=torch.float32, device='cuda'); db = torch.empty(cout, dtype=torch.float32, device='cuda')
    L.check(lib.sdb_conv_wgrad_nd(L.ptr(skd), L.ptr(lod), n, d, h, w, c_skip, c_lo, uz, uy, ux, 3 if nd == 3 else 1, 3, L.ptr(dyd), cout, cout,
                                  L.ptr(work), need, L.ptr(dw), L.ptr(db), L.stream_ptr()))
    assert np.array_equal(dw.cpu().numpy().astype(np.float64), kt.grad.permute(*range(2, nd + 2), 1, 0).numpy())
    wf = torch.empty((taps, cout, cin), dtype=torch.float32, device='cuda')
    L.check(lib.sdb_conv_flip_weights(L.ptr(kd), taps, cin, cout, L.ptr(wf), L.stream_ptr()))
    zb = torch.zeros(cin, dtype=torch.float32, device='cuda')
    dcat = torch.empty((n,) + shape + (cin,), dtype=torch.float32, device='cuda')
    L.check(lib.sdb_conv3_nd(L.ptr(dyd), None, n, d, h, w, cout, 0, 1, 1, 1, L.ptr(wf), L.ptr(zb), cin, 1 if nd == 2 else 3, 0,
                             L.ptr(dcat), L.stream_ptr()))
    dlo = torch.empty(lo.shape, dtype=torch.float32, device='cuda')
    dskip = torch.empty(skip.shape, dtype=torch.float32, device='cuda')
    L.check(lib.sdb_decoder_split(L.ptr(dcat), n, d, h, w, c_lo, c_skip, uz, uy, ux, L.ptr(dlo), L.ptr(dskip), L.stream_ptr()))
    assert np.array_equal(dlo.cpu().numpy().astype(np.float64), lot.grad.permute(0, *range(2, nd + 2), 1).numpy())
    pz, py, px = ((1,) + tuple(pool)) if nd == 2 else tuple(pool)
    L.check(lib.sdb_maxpool_backward_nd(L.ptr(skd), L.ptr(gpd), n, d, h, w, c_skip, pz, py, px, 1, L.ptr(dskip), L.stream_ptr()))
    L.check(lib.sdb_relu_backward(L.ptr(dskip), L.ptr(skd), dskip.numel(), L.stream_ptr()))
    assert np.array_equal(dskip.cpu().numpy().astype(np.float64), spre.grad.permute(0, *range(2, nd + 2), 1).numpy())


# ------------------------------------------------------------------------------------------------ loss kernel
@pytest.mark.parametrize("dist_loss,lam", [('mae', 0.0), ('mae', 1e-4), ('mse', 0.0), ('mse', 1e-2)])
def test_loss_kernel_against_float64(dist_loss, lam):
    """loss terms: relative error <= 4e-6 (a few float32 ulps after the float64 accumulation); per-pixel dz and d dist:
    |err| <= 4e-6 |ref| + 1e-6 max|ref| (float32 arithmetic of a handful of operations per element)"""
    L, lib = _lib()
    rng = np.random.default_rng(5)
    npix, R = 3000, 16
    z = rng.normal(0, 4, npix)
    z[:20] = 40.0; z[20:40] = -40.0                   # the clip region at both ends
    prob = (1 / (1 + np.exp(-z))).astype(np.float32)
    prob_t = rng.uniform(0, 1, npix).astype(np.float32)
    prob_t[rng.uniform(0, 1, npix) < 0.2] = -1        # ignored pixels
    dist = rng.normal(3, 2, (npix, R)).astype(np.float32)
    dam = np.concatenate([rng.uniform(0, 8, (npix, R)), (rng.uniform(0, 1, (npix, 1)) < 0.6)], axis=1).astype(np.float32)
    p64 = torch.from_numpy(prob.astype(np.float64)).requires_grad_(True)
    d64 = torch.from_numpy(dist.astype(np.float64)).requires_grad_(True)
    tot, lp, ld = O.loss64(p64, d64, torch.from_numpy(prob_t.astype(np.float64)), torch.from_numpy(dam.astype(np.float64)),
                           dist_loss=dist_loss, lam=lam, weights=(1.0, 0.2))
    tot.backward()
    want_dz = (p64.grad * p64 * (1 - p64)).detach().numpy()       # chain rule through the sigmoid
    want_dd = d64.grad.numpy()
    work = torch.empty(int(lib.sdb_stardist_loss_workspace(npix)) // 4, dtype=torch.float32, device='cuda')
    stats = torch.empty(2, dtype=torch.float32, device='cuda')
    dhead = torch.empty((npix, R + 1), dtype=torch.float32, device='cuda')
    out = torch.empty(4, dtype=torch.float32, device='cuda')
    dev = [_dev(a) for a in (prob, dist, prob_t, dam)]          # kept alive until the kernels have run
    L.check(lib.sdb_stardist_loss(*(L.ptr(t) for t in dev), npix, R, 1 if dist_loss == 'mae' else 0,
                                  lam, 1.0, 0.2, L.ptr(work), L.ptr(stats), L.ptr(dhead), L.ptr(out), None, L.stream_ptr()))
    o = out.cpu().numpy().astype(np.float64)
    for got, ref in zip(o[:3], (tot.item(), lp.item(), ld.item())):
        assert abs(got - ref) <= 4e-6 * abs(ref), (got, ref)
    assert o[3] == 0
    dh = dhead.cpu().numpy().astype(np.float64)
    for got, ref in ((dh[:, 0], want_dz), (dh[:, 1:], want_dd)):
        err = np.abs(got - ref)
        assert np.all(err <= 4e-6 * np.abs(ref) + 1e-6 * np.abs(ref).max()), err.max()


# ------------------------------------------------------------------------------------------------ whole network
def _small_data(nd, n=4, seed=0):
    from oracle import synth
    if nd == 2:
        Y = [synth.ellipse_labels((96, 96), seed=seed + i, rmin=5, rmax=9) for i in range(n)]
        X = [synth.image_from_labels(y, seed=seed + i) for i, y in enumerate(Y)]
    else:
        # fill 0.1: a fill these volumes can reach (the default retries 400000 placements when it cannot)
        Y = [synth.ellipsoid_labels((24, 48, 48), seed=seed + i, fill=0.1, rmin=4, rmax=7) for i in range(n)]
        X = [synth.volume_from_labels(y, seed=seed + i) for i, y in enumerate(Y)]
    return X, Y


def _config(case):
    from stardist_b200 import Config2D, Config3D
    if case == '2d':
        return Config2D(n_rays=16, unet_n_depth=2, unet_n_filter_base=32, grid=(1, 1), train_patch_size=(64, 64), train_batch_size=2)
    if case == '2d_grid':
        return Config2D(n_rays=16, unet_n_depth=2, unet_n_filter_base=32, grid=(2, 2), train_patch_size=(64, 64), train_batch_size=2)
    from stardist_b200.rays3d import Rays_GoldenSpiral
    return Config3D(rays=Rays_GoldenSpiral(24), unet_n_depth=2, unet_n_filter_base=32, unet_pool=(1, 2, 2), grid=(1, 2, 2),
                    train_patch_size=(6, 16, 16), train_batch_size=1, train_background_reg=1e-4)


def _batch(config, seed=0, length=4):
    from stardist_b200.models import StarDistData2D, StarDistData3D
    X, Y = _small_data(config.n_dim, seed=seed)
    kw = dict(patch_size=config.train_patch_size, grid=config.grid, foreground_prob=config.train_foreground_only)
    np.random.seed(seed)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        if config.n_dim == 2:
            g = StarDistData2D(X, Y, batch_size=config.train_batch_size, n_rays=config.n_rays, length=length, **kw)
        else:
            from stardist_b200.rays3d import rays_from_json
            g = StarDistData3D(X, Y, batch_size=config.train_batch_size, rays=rays_from_json(config.rays_json), length=length, **kw)
        return [g.batch_device(i) for i in range(length)]


@pytest.mark.parametrize("case", ['2d', '2d_grid', '3d_pool122'])
def test_network_gradient_against_float64_autograd(case):
    """every parameter tensor's gradient within relative L2 error 1e-4 of float64 torch autograd on a real batch"""
    from stardist_b200.models.train import UNetTrainer
    from stardist_b200.models.weights import glorot_uniform_weights
    config = _config(case)
    weights = glorot_uniform_weights(config, seed=1)
    tr = UNetTrainer(config, weights)
    (x,), (p, d) = _batch(config)[0]
    got = tr.gradients(x, p, d)
    P = O.params64(weights, tr.names)
    prob, dist = O.forward64(config, P, x.cpu().double())
    tot, _, _ = O.loss64(prob, dist, p.cpu().double(), d.cpu().double(), dist_loss=config.train_dist_loss,
                         lam=float(config.train_background_reg), weights=tuple(float(v) for v in config.train_loss_weights))
    tot.backward()
    want = O.grads_keras(P)
    worst = 0.0
    for n in tr.names:
        for a, b in zip(got[n], want[n]):
            rel = np.linalg.norm(a.astype(np.float64) - b) / max(np.linalg.norm(b), 1e-30)
            worst = max(worst, rel)
            assert rel <= 1e-4, (n, rel)
    print("%s: worst relative L2 gradient error %.3g" % (case, worst))


def test_adam_bit_identical_to_numpy():
    from stardist_b200.models.train import UNetTrainer
    from stardist_b200.models.weights import glorot_uniform_weights
    config = _config('2d')
    tr = UNetTrainer(config, glorot_uniform_weights(config, seed=2))
    batches = _batch(config, seed=3)
    coef = None
    w = tr.params.cpu().numpy(); m = np.zeros_like(w); v = np.zeros_like(w)
    for t, ((x,), (p, d)) in enumerate(batches, start=1):
        tr.gradients(x, p, d)
        g = tr.grad.cpu().numpy()
        tr.step(x, p, d)
        coef = tr.coef.cpu().numpy()
        w, m, v = O.adam_np(w, g, m, v, tr.lr, coef[t - 1])
        assert np.array_equal(tr.params.cpu().numpy(), w), t
        assert np.array_equal(tr.m.cpu().numpy(), m) and np.array_equal(tr.v.cpu().numpy(), v)


def test_training_is_deterministic():
    from stardist_b200.models.train import UNetTrainer
    from stardist_b200.models.weights import glorot_uniform_weights
    config = _config('2d_grid')
    runs = []
    for _ in range(2):
        tr = UNetTrainer(config, glorot_uniform_weights(config, seed=4))
        losses = [tr.step(x, p, d).cpu().numpy().copy() for (x,), (p, d) in _batch(config, seed=5, length=5)]
        runs.append((tr.params.cpu().numpy(), np.stack(losses)))
    assert np.array_equal(runs[0][0], runs[1][0])
    assert np.array_equal(runs[0][1], runs[1][1])


def test_empty_batch_is_skipped():
    from stardist_b200.models.train import UNetTrainer
    from stardist_b200.models.weights import glorot_uniform_weights
    config = _config('2d')
    tr = UNetTrainer(config, glorot_uniform_weights(config, seed=6))
    (x,), (p, d) = _batch(config)[0]
    before = tr.params.cpu().numpy()
    out = tr.step(x, torch.full_like(p, -1.0), d).cpu().numpy()
    assert out[3] == 1
    assert np.array_equal(tr.params.cpu().numpy(), before)
    assert tr.state.cpu().numpy().tolist() == [0, 1, 1]


# ------------------------------------------------------------------------------------------------ train()
def test_train_end_to_end(tmp_path):
    from stardist_b200 import Config2D, StarDist2D
    X, Y = _small_data(2, n=6, seed=10)
    config = Config2D(n_rays=16, unet_n_depth=2, grid=(1, 1), train_patch_size=(64, 64), train_batch_size=4, train_epochs=6,
                      train_steps_per_epoch=50, train_learning_rate=1e-3)
    model = StarDist2D(config, name='m', basedir=str(tmp_path))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        hist = model.train(X[:4], Y[:4], validation_data=(X[4:], Y[4:]), seed=0)
    h = hist.history
    assert set(h) == {'loss', 'prob_loss', 'dist_loss', 'val_loss', 'val_prob_loss', 'val_dist_loss', 'lr'}
    assert all(len(v) == 6 for v in h.values())
    print("val_loss per epoch:", ["%.4f" % v for v in h['val_loss']])
    assert h['val_loss'][-1] < 0.5 * h['val_loss'][0]
    for f in ('config.json', 'weights.npz', 'weights_last.npz'):
        assert (tmp_path / 'm' / f).exists(), f
    best = int(np.argmin(h['val_loss']))
    assert h['val_loss'][best] == min(h['val_loss'])
    again = StarDist2D(None, name='m', basedir=str(tmp_path))
    for n, (k, b) in model.weights.items():
        assert np.array_equal(again.weights[n][0], k) and np.array_equal(again.weights[n][1], b), n
    img = X[5]
    l1, r1 = model.predict_instances(img)
    l2, r2 = again.predict_instances(img)
    assert np.array_equal(l1, l2) and np.array_equal(r1['points'], r2['points'])
