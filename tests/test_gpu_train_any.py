"""Training outside the default architecture family on the device: sdb_conv_wgrad_any_nd and sdb_conv_dgrad_any_nd bit-equal
to float64 autograd on exactly representable data, sdb_act_backward within the bound of tests/train_any_cases.py, the
split forward (linear convolution, then sdb_act_any) bit-equal to the fused one, whole-network gradients against float64
autograd through the any_config_oracle restatement, determinism, Adam, and an end-to-end train() of a 5x5 ELU model."""
import os, sys, warnings
import numpy as np
import pytest
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import any_config_oracle as AO
import train_any_cases as C
import train_oracle as O
import train_oracle_classes as OC

pytestmark = pytest.mark.gpu


def _lib():
    from stardist_b200 import _lib as L
    return L, L.require_cuda()


def _dev(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


def _nan(shape):
    return torch.full(tuple(shape), float('nan'), dtype=torch.float32, device='cuda')


def _dhw(nd, t):
    return ((1,) + tuple(t)) if nd == 2 else tuple(t)


# ------------------------------------------------------------------------------------------------ layer-exact kernels
@pytest.mark.parametrize("case", C.EXACT_ANY, ids=lambda c: c['id'])
def test_wgrad_and_dgrad_any_exact(case):
    """dW, db (sdb_conv_wgrad_any_nd) and dX (sdb_conv_dgrad_any_nd on the flipped kernel, then sdb_decoder_split for a
    decoder input) bit-equal to float64 autograd of any_config_oracle.conv_same"""
    L, lib = _lib()
    st = L.stream_ptr()
    skip, lo, dy, k = C.int_data(case)
    nd, n, cout = case['nd'], case['n'], case['cout']
    c_skip, c_lo = case['c_skip'], case['c_lo']
    cin = c_skip + c_lo
    t = lambda a: torch.from_numpy(a.astype(np.float64)).requires_grad_(True)
    xs, xl, kt = t(skip), (None if lo is None else t(lo)), t(k)
    bt = torch.zeros(cout, dtype=torch.float64, requires_grad=True)
    inp = xs if xl is None else torch.cat([AO.upsample(xl, case['up']), xs], dim=-1)
    (AO.conv_same(inp, kt, bt) * torch.from_numpy(dy.astype(np.float64))).sum().backward()
    d, h, w = _dhw(nd, case['shape'])
    kz, ky, kx = _dhw(nd, case['k'])
    uz, uy, ux = _dhw(nd, case['up'])
    sd, ld, dyd, kd = _dev(skip), _dev(lo), _dev(dy), _dev(k)
    need = int(lib.sdb_conv_wgrad_workspace(n * d * h * w, kz * ky * kx, cin, cout))
    work = torch.empty(need, dtype=torch.float32, device='cuda')
    dw, db = _nan(k.shape), _nan((cout,))
    L.check(lib.sdb_conv_wgrad_any_nd(L.ptr(sd), L.ptr(ld), n, d, h, w, c_skip, c_lo, uz, uy, ux, kz, ky, kx, L.ptr(dyd), cout, cout,
                                      L.ptr(work), need, L.ptr(dw), L.ptr(db), st))
    assert np.array_equal(dw.cpu().numpy().astype(np.float64), kt.grad.numpy())
    assert np.array_equal(db.cpu().numpy().astype(np.float64), bt.grad.numpy())
    taps = kz * ky * kx
    wf = _nan((taps, cout, cin))
    L.check(lib.sdb_conv_flip_weights(L.ptr(kd), taps, cin, cout, L.ptr(wf), st))
    dx = _nan((n,) + case['shape'] + (cin,))
    L.check(lib.sdb_conv_dgrad_any_nd(L.ptr(dyd), n, d, h, w, cout, L.ptr(wf), cin, kz, ky, kx, L.ptr(dx), st))
    if lo is None:
        assert np.array_equal(dx.cpu().numpy().astype(np.float64), xs.grad.numpy())
        return
    dlo, dsk = _nan(lo.shape), _nan(skip.shape)
    L.check(lib.sdb_decoder_split(L.ptr(dx), n, d, h, w, c_lo, c_skip, uz, uy, ux, L.ptr(dlo), L.ptr(dsk), st))
    assert np.array_equal(dlo.cpu().numpy().astype(np.float64), xl.grad.numpy())
    assert np.array_equal(dsk.cpu().numpy().astype(np.float64), xs.grad.numpy())


# ------------------------------------------------------------------------------------------------ activations
@pytest.mark.parametrize("act", AO.ACTS)
def test_act_backward_vs_float64(act):
    """g = 1 gives act'(z): relu / linear exactly, the others within act_grad_bound (8 float32 ulps of the summed terms'
    magnitude plus one rounding of z) over a sweep with the elu / selu and softplus branch points; a random g gives the
    float32 product g * act'(z) exactly"""
    from stardist_b200.models.unet_device import act_id
    L, lib = _lib()
    z = C.act_points()
    zd = _dev(z)
    ones = torch.ones(z.size, dtype=torch.float32, device='cuda')
    L.check(lib.sdb_act_backward(L.ptr(ones), L.ptr(zd), z.size, act_id(act), L.stream_ptr()))
    a = ones.cpu().numpy()
    if act in ('relu', 'linear'):
        assert np.array_equal(a, C.act_grad_np(act, z))
    else:
        want, bound = C.act_grad_bound(act, z)
        err = np.abs(a.astype(np.float64) - want)
        i = int(np.argmax(err / bound))
        assert np.all(err <= bound), "%s: z=%r got %r want %r (bound %g)" % (act, z[i], a[i], want[i], bound[i])
    g = np.random.default_rng(3).standard_normal(z.size).astype(np.float32)
    gd = _dev(g)
    L.check(lib.sdb_act_backward(L.ptr(gd), L.ptr(zd), z.size, act_id(act), L.stream_ptr()))
    want = np.where(z > 0, g, np.float32(0)) if act == 'relu' else g * a
    assert np.array_equal(gd.cpu().numpy(), want)


@pytest.mark.parametrize("act", AO.ACTS)
def test_linear_convolution_then_activation_equals_fused(act):
    """the training forward of an activation other than ReLU / linear (sdb_conv_any_nd linear, then sdb_act_any) gives the
    fused convolution's output bit for bit"""
    from stardist_b200.models.unet_device import act_id
    L, lib = _lib()
    rng = np.random.default_rng(7)
    x = rng.standard_normal((2, 19, 37, 5)).astype(np.float32)
    k = (0.4 * rng.standard_normal((5, 5, 5, 24))).astype(np.float32)
    b = rng.standard_normal(24).astype(np.float32)
    xd, kd, bd = _dev(x), _dev(k), _dev(b)
    outs = {}
    for a in (act, 'linear'):
        outs[a] = _nan((2, 19, 37, 24))
        L.check(lib.sdb_conv_any_nd(L.ptr(xd), None, 2, 1, 19, 37, 5, 0, 1, 1, 1, L.ptr(kd), L.ptr(bd), 24, 1, 5, 5, 1, 1, 1, act_id(a),
                                    L.ptr(outs[a]), L.stream_ptr()))
    y = _nan((2, 19, 37, 24))
    L.check(lib.sdb_act_any(L.ptr(outs['linear']), y.numel(), act_id(act), L.ptr(y), L.stream_ptr()))
    assert np.array_equal(y.cpu().numpy().view(np.int32), outs[act].cpu().numpy().view(np.int32))


# ------------------------------------------------------------------------------------------------ whole network
def _small_data(nd, n=4, seed=0, channels=1):
    from oracle import synth
    if nd == 2:
        Y = [synth.ellipse_labels((96, 96), seed=seed + i, rmin=5, rmax=9) for i in range(n)]
        X = [synth.image_from_labels(y, seed=seed + i) for i, y in enumerate(Y)]
        if channels > 1:
            X = [np.stack([x * (1 + 0.1 * c) for c in range(channels)], axis=-1) for x in X]
    else:
        Y = [synth.ellipsoid_labels((24, 48, 48), seed=seed + i, fill=0.1, rmin=4, rmax=7) for i in range(n)]
        X = [synth.volume_from_labels(y, seed=seed + i) for i, y in enumerate(Y)]
    return X, Y


def _config(case):
    from stardist_b200 import Config2D, Config3D
    c2 = dict(n_rays=16, unet_n_depth=2, grid=(1, 1), train_patch_size=(64, 64), train_batch_size=2)
    if case == '2d_k55_elu':
        return Config2D(unet_kernel_size=(5, 5), unet_activation='elu', **c2)
    if case == '2d_k22_swish':
        return Config2D(unet_kernel_size=(2, 2), unet_activation='swish', unet_last_activation='softplus', **c2)
    if case == '2d_base16_gelu_cin3':
        return Config2D(unet_n_filter_base=16, unet_activation='gelu', n_channel_in=3, **c2)
    if case == '2d_classes_k55_selu':
        return Config2D(unet_kernel_size=(5, 5), unet_activation='selu', unet_last_activation='tanh', n_classes=3,
                        train_class_weights=(0.5, 1, 2, 1.5), train_loss_weights=(1, 0.2, 0.7), **c2)
    from stardist_b200.rays3d import Rays_GoldenSpiral
    return Config3D(rays=Rays_GoldenSpiral(24), unet_n_depth=2, unet_n_filter_base=16, unet_kernel_size=(1, 3, 3), unet_pool=(1, 2, 2),
                    grid=(1, 2, 2), train_patch_size=(6, 16, 16), train_batch_size=1, train_background_reg=1e-4)


CASES = ['2d_k55_elu', '2d_k22_swish', '2d_base16_gelu_cin3', '3d_k133_pool122', '2d_classes_k55_selu']


def _batches(config, seed=0, length=4):
    from stardist_b200.models import StarDistData2D, StarDistData3D
    X, Y = _small_data(config.n_dim, seed=seed, channels=config.n_channel_in)
    kw = dict(patch_size=config.train_patch_size, grid=config.grid, foreground_prob=config.train_foreground_only)
    if config.n_classes is not None:
        kw.update(n_classes=config.n_classes, classes=[{int(l): 1 + int(l) % config.n_classes for l in np.unique(y) if l > 0} for y in Y])
    np.random.seed(seed)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        if config.n_dim == 2:
            g = StarDistData2D(X, Y, batch_size=config.train_batch_size, n_rays=config.n_rays, length=length, **kw)
        else:
            from stardist_b200.rays3d import rays_from_json
            g = StarDistData3D(X, Y, batch_size=config.train_batch_size, rays=rays_from_json(config.rays_json), length=length, **kw)
        return [g.batch_device(i) for i in range(length)]


def _act64(name, t):
    """any_config_oracle.act64, with TensorFlow's ReLU gradient (0 at 0; clamp_min passes 1 there)"""
    return F.relu(t) if name == 'relu' else AO.act64(name, t)


def _forward64(config, W, x):
    """(prob, dist, prob_class or None), channels last, differentiable in W (Keras-layout float64 leaves)"""
    from stardist_b200.models.weights import unet_layers
    skips, lo, up, base = {}, None, None, None
    for l in unet_layers(config):
        if l['kind'] == 'conv':
            if l['name'] == 'features':
                base = x
            inp = x if lo is None else torch.cat([AO.upsample(lo, up), x], dim=-1)
            x = _act64(l['act'], AO.conv_same(inp, *W[l['name']]))
            lo = None
        elif l['kind'] == 'pool':
            if 'save_skip' in l:
                skips[l['save_skip']] = x
            x = AO.maxpool(x, l['pool'])
        elif l['kind'] == 'up':
            lo, up = x, tuple(l['pool'])
            x = skips.pop(l['skip'])
    base = x if base is None else base
    prob, dist = AO._heads(W, x, None)
    pc = None
    if config.n_classes is not None:
        c = base
        if 'features_class' in W:
            c = _act64(config.unet_activation, AO.conv_same(base, *W['features_class']))
        wc, bc = W['prob_class']
        pc = torch.softmax(c @ wc.reshape(c.shape[-1], -1) + bc, dim=-1)
    return prob, dist, pc


@pytest.mark.parametrize("case", CASES)
def test_network_gradient_against_float64_autograd(case):
    """every parameter tensor's gradient within relative L2 error 1e-4 of float64 autograd on a real batch"""
    from stardist_b200.models.train import UNetTrainer
    from stardist_b200.models.weights import glorot_uniform_weights
    config = _config(case)
    weights = glorot_uniform_weights(config, seed=1)
    tr = UNetTrainer(config, weights)
    batch = _batches(config)[0]
    (x,), targets = batch
    got = tr.gradients(x, *targets)
    W = {n: tuple(torch.from_numpy(np.asarray(a, np.float64)).requires_grad_(True) for a in weights[n]) for n in tr.names}
    prob, dist, pc = _forward64(config, W, x.cpu().double())
    w = tuple(float(v) for v in config.train_loss_weights)
    tot, _, _ = O.loss64(prob, dist, targets[0].cpu().double(), targets[1].cpu().double(), dist_loss=config.train_dist_loss,
                         lam=float(config.train_background_reg), weights=w[:2])
    if pc is not None:
        tot = tot + w[2] * OC.class_loss64(pc, targets[2].cpu().double(), config.train_class_weights)
    tot.backward()
    worst = 0.0
    for n in tr.names:
        for a, b in zip(got[n], W[n]):
            b = b.grad.numpy()
            rel = np.linalg.norm(a.astype(np.float64) - b) / max(np.linalg.norm(b), 1e-30)
            worst = max(worst, rel)
            assert rel <= 1e-4, (n, rel)
    print("%s: worst relative L2 gradient error %.3g" % (case, worst))


def test_forward_with_kept_preactivations_equals_prediction_forward():
    """keep=True (convolutions linear, then sdb_act_any) leaves prob, dist and prob_class bit for bit as in prediction"""
    from stardist_b200.models.unet_device import UNetDeviceND
    from stardist_b200.models.weights import glorot_uniform_weights
    config = _config('2d_classes_k55_selu')
    net = UNetDeviceND(config, glorot_uniform_weights(config, seed=3))
    x = torch.from_numpy(np.random.default_rng(0).uniform(0, 1, (2, 64, 64, 1)).astype(np.float32)).cuda()
    p1, d1 = net.forward(x)
    c1 = net.prob_class.clone()
    p2, d2 = net.forward(x, keep=True)
    for a, b in ((p1, p2), (d1, d2), (c1, net.prob_class)):
        assert np.array_equal(a.cpu().numpy().view(np.int32), b.cpu().numpy().view(np.int32))
    kept = [s for s in net.saved if s is not None and 'y' in s]
    assert kept and all(s['z'] is not None for s in kept) and net.saved_class_z is not None


def test_training_is_deterministic():
    from stardist_b200.models.train import UNetTrainer
    from stardist_b200.models.weights import glorot_uniform_weights
    config = _config('2d_k55_elu')
    runs = []
    for _ in range(2):
        tr = UNetTrainer(config, glorot_uniform_weights(config, seed=4))
        losses = [tr.step(x, p, d).cpu().numpy().copy() for (x,), (p, d) in _batches(config, seed=5, length=3)]
        runs.append((tr.params.cpu().numpy(), np.stack(losses)))
    assert np.array_equal(runs[0][0], runs[1][0])
    assert np.array_equal(runs[0][1], runs[1][1])


def test_adam_bit_identical_to_numpy():
    from stardist_b200.models.train import UNetTrainer
    from stardist_b200.models.weights import glorot_uniform_weights
    config = _config('2d_k22_swish')
    tr = UNetTrainer(config, glorot_uniform_weights(config, seed=2))
    w = tr.params.cpu().numpy(); m = np.zeros_like(w); v = np.zeros_like(w)
    for t, ((x,), (p, d)) in enumerate(_batches(config, seed=3, length=3), start=1):
        tr.gradients(x, p, d)
        g = tr.grad.cpu().numpy()
        tr.step(x, p, d)
        w, m, v = O.adam_np(w, g, m, v, tr.lr, tr.coef.cpu().numpy()[t - 1])
        assert np.array_equal(tr.params.cpu().numpy(), w), t
        assert np.array_equal(tr.m.cpu().numpy(), m) and np.array_equal(tr.v.cpu().numpy(), v)


# ------------------------------------------------------------------------------------------------ train()
def test_train_end_to_end_k55_elu(tmp_path):
    from stardist_b200 import Config2D, StarDist2D
    X, Y = _small_data(2, n=6, seed=10)
    config = Config2D(n_rays=16, unet_n_depth=2, unet_kernel_size=(5, 5), unet_activation='elu', grid=(1, 1), train_patch_size=(64, 64),
                      train_batch_size=4, train_epochs=6, train_steps_per_epoch=50, train_learning_rate=1e-3)
    model = StarDist2D(config, name='m', basedir=str(tmp_path))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        hist = model.train(X[:4], Y[:4], validation_data=(X[4:], Y[4:]), seed=0)
    h = hist.history
    print("val_loss per epoch:", ["%.4f" % v for v in h['val_loss']])
    assert all(len(v) == 6 for v in h.values())
    assert h['val_loss'][-1] < 0.5 * h['val_loss'][0]
    for f in ('config.json', 'weights.npz', 'weights_last.npz'):
        assert (tmp_path / 'm' / f).exists(), f
    again = StarDist2D(None, name='m', basedir=str(tmp_path))
    assert tuple(again.config.unet_kernel_size) == (5, 5) and again.config.unet_activation == 'elu'
    for n, (k, b) in model.weights.items():
        assert np.array_equal(again.weights[n][0], k) and np.array_equal(again.weights[n][1], b), n
    img = X[5]
    l1, r1 = model.predict_instances(img)
    l2, r2 = again.predict_instances(img)
    assert np.array_equal(l1, l2) and np.array_equal(r1['points'], r2['points'])
