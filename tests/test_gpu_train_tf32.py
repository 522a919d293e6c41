"""The TF32 backward pass on the device (csrc/unet_train_tf32.cu behind stardist_b200.enable_tensor_float_32_execution,
DESIGN.md 4.2): layer-exact weight and input gradients on TF32-exact integers and on 12-bit operands whose rounding is
pinned, whole-network gradients against float64 autograd with the same roundings, determinism, and train() end to end."""
import os, sys, warnings
from contextlib import contextmanager
from unittest import mock
import numpy as np
import pytest
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import train_oracle as O
import train_oracle_classes as OC
import train_tf32_cases as C

pytestmark = pytest.mark.gpu


def _lib():
    from stardist_b200 import _lib as L
    return L, L.require_cuda()


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


@contextmanager
def tf32(on):
    import stardist_b200 as s
    before = s.tensor_float_32_execution_enabled()
    s.enable_tensor_float_32_execution(on)
    try:
        yield
    finally:
        s.enable_tensor_float_32_execution(before)


def _same_bits(a, b):
    return np.array_equal(np.asarray(a, np.float32).view(np.uint32), np.asarray(b, np.float32).view(np.uint32))


# ------------------------------------------------------------------------------------------------ layers
def _run_wgrad(case, x, lo, skip, dy_rows):
    """sdb_conv_wgrad_tf32_nd on the case's layout: (dw, db) numpy"""
    L, lib = _lib()
    nd, n, shape, cout = case['nd'], case['n'], case['shape'], case['cout']
    d, h, w = ((1,) + shape) if nd == 2 else shape
    k = case.get('k', (3,) * nd)
    kz, kyx = (1, k[-1]) if nd == 2 else (k[0], k[-1])
    up = case.get('up', (1,) * nd)
    uz, uy, ux = ((1,) + tuple(up)) if nd == 2 else tuple(up)
    c_lo = 0 if lo is None else lo.shape[-1]
    ldy, off = dy_rows.shape[-1], case.get('off', 0)
    taps = int(np.prod(k))
    need = int(lib.sdb_conv_wgrad_workspace(n * d * h * w, taps, skip.shape[-1] + c_lo, cout))
    work = torch.empty(need, dtype=torch.float32, device='cuda')
    dw = torch.empty(tuple(k) + (skip.shape[-1] + c_lo, cout), dtype=torch.float32, device='cuda')
    db = torch.empty(cout, dtype=torch.float32, device='cuda')
    xs, xl, dyd = _dev(skip), None if lo is None else _dev(lo), _dev(dy_rows)
    L.check(lib.sdb_conv_wgrad_tf32_nd(L.ptr(xs), L.ptr(xl), n, d, h, w, skip.shape[-1], c_lo, uz, uy, ux, kz, kyx,
                                       L.ptr(dyd.view(-1)[off:]), ldy, cout, L.ptr(work), need, L.ptr(dw), L.ptr(db), L.stream_ptr()))
    return dw.cpu().numpy(), db.cpu().numpy()


def _run_dgrad(case, dy, k):
    L, lib = _lib()
    nd, n, shape, cin, cout = case['nd'], case['n'], case['shape'], case['cin'], case['cout']
    d, h, w = ((1,) + shape) if nd == 2 else shape
    taps = 3 ** nd
    kd, dyd = _dev(k), _dev(dy)
    wf = torch.empty((taps, cout, cin), dtype=torch.float32, device='cuda')
    L.check(lib.sdb_conv_flip_weights(L.ptr(kd), taps, cin, cout, L.ptr(wf), L.stream_ptr()))
    gin = torch.empty((n,) + shape + (cin,), dtype=torch.float32, device='cuda')
    L.check(lib.sdb_conv_dgrad_tf32_nd(L.ptr(dyd), n, d, h, w, cout, L.ptr(wf), cin, 1 if nd == 2 else 3, 3, L.ptr(gin), L.stream_ptr()))
    return gin.cpu().numpy()


@pytest.mark.parametrize("case", C.TF32_WGRAD + C.TF32_DECODER, ids=lambda c: c['id'])
def test_wgrad_tf32_exact_on_integers(case):
    """dW and db bit-equal to float64 autograd on TF32-exact integers"""
    x, lo, skip, dy_rows = C.int_wgrad_data(case)
    off = case.get('off', 0)
    dy = dy_rows[..., off:off + case['cout']]
    want_dw, want_db, _ = C.conv_grads64(x, dy, None, case['nd'], case.get('k', (3,) * case['nd']))
    dw, db = _run_wgrad(case, x, lo, skip, dy_rows)
    assert np.array_equal(dw.astype(np.float64), want_dw)
    assert np.array_equal(db.astype(np.float64), want_db)


@pytest.mark.parametrize("case", C.TF32_DGRAD, ids=lambda c: c['id'])
def test_dgrad_tf32_exact_on_integers(case):
    dy, k = C.int_dgrad_data(case)
    x0 = np.zeros(dy.shape[:-1] + (case['cin'],))
    _, _, want = C.conv_grads64(x0, dy, k, case['nd'])
    assert np.array_equal(_run_dgrad(case, dy, k).astype(np.float64), want)


@pytest.mark.parametrize("case", C.ROUNDING_WGRAD, ids=lambda c: c['id'])
def test_wgrad_tf32_rounding_is_rna(case):
    """12-bit operands (ties at 11 bits): dW bit-equal to float64 of rna(x) rna(dy); db bit-equal to float64 of the unrounded dy"""
    x, dy_rows = C.rounding_wgrad_data(case)
    off = case.get('off', 0)
    dy = dy_rows[..., off:off + case['cout']]
    k = case['k']
    want_dw = C.conv_grads64(C.rna(x), C.rna(dy), None, case['nd'], k)[0]
    want_db = C.conv_grads64(x, dy, None, case['nd'], k)[1]
    dw, db = _run_wgrad(case, x, None, x, dy_rows)
    assert np.array_equal(dw.astype(np.float64), want_dw)
    assert np.array_equal(db.astype(np.float64), want_db)


@pytest.mark.parametrize("case", C.ROUNDING_DGRAD, ids=lambda c: c['id'])
def test_dgrad_tf32_rounding_is_rna(case):
    dy, k = C.rounding_dgrad_data(case)
    x0 = np.zeros(dy.shape[:-1] + (case['cin'],))
    want = C.conv_grads64(x0, C.rna(dy), C.rna(k), case['nd'])[2]
    assert np.array_equal(_run_dgrad(case, dy, k).astype(np.float64), want)


def test_dgrad_tf32_refuses_shapes_outside_conv_dgrad3_accepts():
    L, lib = _lib()
    buf = torch.zeros(4096, device='cuda')
    for cout, cin, kz, kyx, d in ((16, 48, 1, 3, 1), (5, 32, 1, 3, 1), (4, 96, 1, 3, 1), (32, 32, 1, 1, 1), (32, 32, 1, 3, 2)):
        assert lib.sdb_conv_dgrad_tf32_nd(L.ptr(buf), 1, d, 4, 4, cout, L.ptr(buf), cin, kz, kyx, L.ptr(buf), L.stream_ptr()) != 0


# ------------------------------------------------------------------------------------------------ whole network
def _rna64(t):
    return torch.from_numpy(C.rna(t.detach().numpy().astype(np.float32)).astype(np.float64))


class _TF32Conv(torch.autograd.Function):
    """float64 convolution whose backward is the TF32 trainer's: dW from rna(x) and rna(dy), db from dy, and dx from rna(dy)
    and rna(W) where conv_dgrad3_accepts routes the layer to the TF32 kernel (exact otherwise)"""

    @staticmethod
    def forward(ctx, x, w, b, conv, round_dx):
        ctx.save_for_backward(x, w)
        ctx.conv, ctx.round_dx = conv, round_dx
        return conv(x, w, b, padding='same')

    @staticmethod
    def backward(ctx, gy):
        x, w = ctx.saved_tensors
        conv = ctx.conv
        with torch.enable_grad():
            xr = _rna64(x).requires_grad_(True)
            wr = w.detach().clone().requires_grad_(True)
            dw, = torch.autograd.grad(conv(xr, wr, None, padding='same'), wr, _rna64(gy))
            dx = None
            if ctx.needs_input_grad[0]:
                x2 = x.detach().clone().requires_grad_(True)
                if ctx.round_dx:
                    dx, = torch.autograd.grad(conv(x2, _rna64(w), None, padding='same'), x2, _rna64(gy))
                else:
                    dx, = torch.autograd.grad(conv(x2, w.detach(), None, padding='same'), x2, gy)
        db = gy.sum(dim=[0] + list(range(2, gy.dim())))
        return dx, dw, db, None, None


@contextmanager
def _tf32_oracle(nd):
    """the oracles' convolutions with the TF32 trainer's backward (weights in torch layout (Cout, Cin, k...))"""
    from stardist_b200.models.unet_device import conv_dgrad3_accepts
    name = 'conv2d' if nd == 2 else 'conv3d'
    orig = getattr(F, name)

    def conv(x, w, b=None, padding=0, **kw):
        k = tuple(w.shape[2:])
        round_dx = conv_dgrad3_accepts(nd, k, w.shape[1], w.shape[0])
        return _TF32Conv.apply(x, w, b, orig, round_dx)
    with mock.patch.object(F, name, conv):
        yield


def _net_config(case):
    from stardist_b200 import Config2D, Config3D
    from stardist_b200.rays3d import Rays_GoldenSpiral
    if case == '2d':
        return Config2D(n_rays=16, unet_n_depth=2, unet_n_filter_base=32, grid=(1, 1), train_patch_size=(64, 64), train_batch_size=2)
    if case == '2d_classes':
        return Config2D(n_rays=16, unet_n_depth=2, unet_n_filter_base=32, grid=(1, 1), train_patch_size=(64, 64), train_batch_size=2,
                        n_classes=3, train_class_weights=(0.5, 1, 2, 1.5), train_loss_weights=(1, 0.2, 0.7))
    return Config3D(rays=Rays_GoldenSpiral(24), unet_n_depth=2, unet_n_filter_base=32, unet_pool=(1, 2, 2), grid=(1, 2, 2),
                    train_patch_size=(6, 16, 16), train_batch_size=1, train_background_reg=1e-4)


def _small_data(nd, n=4, seed=0):
    from oracle import synth
    if nd == 2:
        Y = [synth.ellipse_labels((96, 96), seed=seed + i, rmin=5, rmax=9) for i in range(n)]
        X = [synth.image_from_labels(y, seed=seed + i) for i, y in enumerate(Y)]
    else:
        Y = [synth.ellipsoid_labels((24, 48, 48), seed=seed + i, fill=0.1, rmin=4, rmax=7) for i in range(n)]
        X = [synth.volume_from_labels(y, seed=seed + i) for i, y in enumerate(Y)]
    return X, Y


def _batches(config, seed=0, length=4):
    from stardist_b200.models import StarDistData2D, StarDistData3D
    X, Y = _small_data(config.n_dim, seed=seed)
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


def _oracle_grads(config, weights, names, x, targets, rounded):
    P = O.params64(weights, names)
    w = tuple(float(v) for v in config.train_loss_weights)
    p, d = targets[0], targets[1]

    def run():
        if config.n_classes is None:
            prob, dist = O.forward64(config, P, x.cpu().double())
        else:
            prob, dist, pc = OC.forward64_classes(config, P, x.cpu().double())
        tot = O.loss64(prob, dist, p.cpu().double(), d.cpu().double(), dist_loss=config.train_dist_loss,
                       lam=float(config.train_background_reg), weights=w[:2])[0]
        if config.n_classes is not None:
            tot = tot + w[2] * OC.class_loss64(pc, targets[2].cpu().double(), config.train_class_weights)
        tot.backward()
    if rounded:
        with _tf32_oracle(config.n_dim):
            run()
    else:
        run()
    return O.grads_keras(P)


# Per case (bound against the rna-rounded float64 oracle, bound against plain float64): the worst relative L2 errors measured
# on an H100 80GB HBM3 at 700 W were (4.4e-5, 6.0e-4) for 2d, (4.4e-4, 1.5e-3) for 3d_pool122 and (6.8e-5, 4.5e-4) for
# 2d_classes; the bounds allow about 3x.  Against the oracle the kernels differ by fp32 summation order and by operands that
# round to a different TF32 value because the fp32 activations and gradients differ from the float64 ones in the last bits;
# the differences grow along the backward chain and are largest on the 3-D case's small batch.  Against plain float64 the
# TF32 rounding itself dominates.
BOUNDS = {'2d': (1.5e-4, 2e-3), '3d_pool122': (1.5e-3, 5e-3), '2d_classes': (2e-4, 1.5e-3)}


@pytest.mark.parametrize("case", ['2d', '3d_pool122', '2d_classes'])
def test_network_gradient_tf32(case):
    """switch on: forward loss bit-equal to the switch-off run; every gradient tensor within BOUNDS[case] (relative L2) of
    float64 autograd with the TF32 roundings and of plain float64 autograd"""
    from stardist_b200.models.train import UNetTrainer
    from stardist_b200.models.weights import glorot_uniform_weights
    config = _net_config(case)
    weights = glorot_uniform_weights(config, seed=1)
    with tf32(False):
        tr_off = UNetTrainer(config, weights)
    with tf32(True):
        tr_on = UNetTrainer(config, weights)
    assert tr_on.tf32 and not tr_off.tf32
    (x,), targets = _batches(config)[0]
    loss_off = tr_off.evaluate(x, *targets).cpu().numpy()
    loss_on = tr_on.evaluate(x, *targets).cpu().numpy()
    assert _same_bits(loss_on, loss_off)
    got = tr_on.gradients(x, *targets)
    want_rna = _oracle_grads(config, weights, tr_on.names, x, targets, True)
    want_64 = _oracle_grads(config, weights, tr_on.names, x, targets, False)
    err = {}
    for n in tr_on.names:
        for i, (a, b_rna, b_64) in enumerate(zip(got[n], want_rna[n], want_64[n])):
            a = a.astype(np.float64)
            err[(n, i)] = (np.linalg.norm(a - b_rna) / max(np.linalg.norm(b_rna), 1e-30),
                           np.linalg.norm(a - b_64) / max(np.linalg.norm(b_64), 1e-30))
    worst_rna, worst_64 = (max(e[j] for e in err.values()) for j in (0, 1))
    print("%s: worst relative L2 gradient error %.3g against the TF32 oracle, %.3g against plain float64"
          % (case, worst_rna, worst_64))
    b_rna, b_64 = BOUNDS[case]
    assert worst_rna <= b_rna, {k: e[0] for k, e in err.items() if e[0] > b_rna}
    assert worst_64 <= b_64, {k: e[1] for k, e in err.items() if e[1] > b_64}


def test_trainer_reads_the_switch_at_construction():
    from stardist_b200.models.train import UNetTrainer
    from stardist_b200.models.weights import glorot_uniform_weights
    config = _net_config('2d')
    weights = glorot_uniform_weights(config, seed=2)
    (x,), (p, d) = _batches(config)[0]
    with tf32(True):
        a = UNetTrainer(config, weights)
    with tf32(False):
        g_on = a.gradients(x, p, d)
        g_off = UNetTrainer(config, weights).gradients(x, p, d)
    assert a.tf32
    assert any(not np.array_equal(g_on[n][0], g_off[n][0]) for n in a.names)


def test_tf32_training_is_deterministic():
    from stardist_b200.models.train import UNetTrainer
    from stardist_b200.models.weights import glorot_uniform_weights
    config = _net_config('3d_pool122')
    batches = _batches(config, seed=5, length=3)
    runs = []
    with tf32(True):
        for _ in range(2):
            tr = UNetTrainer(config, glorot_uniform_weights(config, seed=4))
            losses = [tr.step(x, p, d).cpu().numpy().copy() for (x,), (p, d) in batches]
            runs.append((tr.params.cpu().numpy(), np.stack(losses)))
        (x,), (p, d) = batches[0]
        g1, g2 = tr.gradients(x, p, d), tr.gradients(x, p, d)
    assert _same_bits(runs[0][0], runs[1][0]) and _same_bits(runs[0][1], runs[1][1])
    for n in tr.names:
        assert _same_bits(g1[n][0], g2[n][0]) and _same_bits(g1[n][1], g2[n][1]), n


# ------------------------------------------------------------------------------------------------ train()
# |val_loss(on) - val_loss(off)| / val_loss(off) after 6 epochs: 0.023 measured on an H100 80GB HBM3 at 700 W (0.4126 against
# 0.4033); the bound allows about 3x
VAL_LOSS_REL = 0.07


def test_train_end_to_end_tf32(tmp_path):
    from stardist_b200 import Config2D, StarDist2D
    X, Y = _small_data(2, n=6, seed=10)
    config = Config2D(n_rays=16, unet_n_depth=2, grid=(1, 1), train_patch_size=(64, 64), train_batch_size=4, train_epochs=6,
                      train_steps_per_epoch=50, train_learning_rate=1e-3)
    hists, models = {}, {}
    for on in (False, True):
        model = StarDist2D(config, name='m%d' % on, basedir=str(tmp_path))
        with tf32(on), warnings.catch_warnings():
            warnings.simplefilter("ignore")
            hists[on] = model.train(X[:4], Y[:4], validation_data=(X[4:], Y[4:]), seed=0).history
        models[on] = model
    h = hists[True]
    print("val_loss per epoch, TF32:", ["%.4f" % v for v in h['val_loss']], "fp32:", ["%.4f" % v for v in hists[False]['val_loss']])
    assert h['loss'][-1] < h['loss'][0] and h['val_loss'][-1] < h['val_loss'][0]
    rel = abs(h['val_loss'][-1] - hists[False]['val_loss'][-1]) / hists[False]['val_loss'][-1]
    print("relative val_loss difference %.3g" % rel)
    assert rel <= VAL_LOSS_REL
    # prediction ignores the switch
    img = X[5]
    l_off, r_off = models[True].predict_instances(img)
    with tf32(True):
        l_on, r_on = models[True].predict_instances(img)
        prob_on = models[True].predict(img)
    prob_off = models[True].predict(img)
    assert np.array_equal(l_on, l_off) and np.array_equal(r_on['points'], r_off['points'])
    for a, b in zip(prob_on, prob_off):
        assert _same_bits(a, b)
