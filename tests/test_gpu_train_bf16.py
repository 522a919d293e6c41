"""The mixed_bfloat16 trainer on the device (csrc/unet_train_bf16.cu behind stardist_b200.mixed_precision, DESIGN.md 4.2):
layer-exact forward, input-gradient and weight-gradient kernels on bf16-exact integers and on 12-bit operands whose rounding
is pinned, whole-network gradients against float64 autograd with the same rounding points, the bf16 saved activations,
determinism, the policy read at construction, and train() end to end."""
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
import train_bf16_cases as C
from test_gpu_train_tf32 import _net_config, _batches, _small_data, _same_bits

pytestmark = pytest.mark.gpu


def _lib():
    from stardist_b200 import _lib as L
    return L, L.require_cuda()


def _bf(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda().to(torch.bfloat16)


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


def _host(t):
    return t.float().cpu().numpy()


@contextmanager
def policy(name):
    from stardist_b200 import mixed_precision as mp
    before = mp.global_policy()
    mp.set_global_policy(name)
    try:
        yield
    finally:
        mp.set_global_policy(before)


# ------------------------------------------------------------------------------------------------ layers
def _dims(case):
    nd, shape = case['nd'], case['shape']
    d, h, w = ((1,) + shape) if nd == 2 else shape
    kz, ky, kx = ((1,) + tuple(case['k'])) if nd == 2 else tuple(case['k'])
    up = case.get('up', (1,) * nd)
    uz, uy, ux = ((1,) + tuple(up)) if nd == 2 else tuple(up)
    return d, h, w, kz, ky, kx, uz, uy, ux


def _weights_bf16(k, flip):
    """the kernel's bf16 copy in sdb_conv_bf16_nd's layout (flip = 1: the input gradient's)"""
    L, lib = _lib()
    taps, cin, cout = int(np.prod(k.shape[:-2])), k.shape[-2], k.shape[-1]
    wb = torch.empty(taps * cin * cout, dtype=torch.bfloat16, device='cuda')
    kd = _dev(k)
    L.check(lib.sdb_weights_bf16(L.ptr(kd), taps, cin, cout, flip, cout if flip else cin, L.ptr(wb), L.stream_ptr()))
    return wb


def _run_forward(case, lo, skip, k, b, relu):
    L, lib = _lib()
    d, h, w, kz, ky, kx, uz, uy, ux = _dims(case)
    c_lo = 0 if lo is None else lo.shape[-1]
    y = torch.empty(skip.shape[:-1] + (case['cout'],), dtype=torch.bfloat16, device='cuda')
    xs, xl, wb, bd = _bf(skip), None if lo is None else _bf(lo), _weights_bf16(k, 0), _dev(b)     # alive until the call returns
    L.check(lib.sdb_conv_bf16_nd(L.ptr(xs), L.ptr(xl), case['n'], d, h, w, skip.shape[-1], c_lo, uz, uy, ux, kz, ky, kx, L.ptr(wb),
                                 L.ptr(bd), case['cout'], relu, 0, L.ptr(y), L.stream_ptr()))
    return _host(y)


def _run_dgrad(case, dy, k):
    L, lib = _lib()
    d, h, w, kz, ky, kx, _, _, _ = _dims(case)
    cin, cout = k.shape[-2], k.shape[-1]
    gin = torch.empty(dy.shape[:-1] + (cin,), dtype=torch.bfloat16, device='cuda')
    dyd, wfb = _bf(dy), _weights_bf16(k, 1)
    L.check(lib.sdb_conv_bf16_nd(L.ptr(dyd), None, case['n'], d, h, w, cout, 0, 1, 1, 1, kz, ky, kx, L.ptr(wfb), None, cin, 0, 0,
                                 L.ptr(gin), L.stream_ptr()))
    return _host(gin)


def _run_wgrad(case, lo, skip, dy, dy_bf16=True):
    L, lib = _lib()
    d, h, w, kz, ky, kx, uz, uy, ux = _dims(case)
    c_lo = 0 if lo is None else lo.shape[-1]
    cin, cout, n = skip.shape[-1] + c_lo, dy.shape[-1], case['n']
    need = int(lib.sdb_conv_wgrad_workspace(n * d * h * w, kz * ky * kx, cin, cout))
    work = torch.empty(need, dtype=torch.float32, device='cuda')
    dw = torch.empty(tuple(case['k']) + (cin, cout), dtype=torch.float32, device='cuda')
    db = torch.empty(cout, dtype=torch.float32, device='cuda')
    dyd = _bf(dy) if dy_bf16 else _dev(dy)
    xs, xl = _bf(skip), None if lo is None else _bf(lo)
    L.check(lib.sdb_conv_wgrad_bf16_nd(L.ptr(xs), L.ptr(xl), n, d, h, w, skip.shape[-1], c_lo,
                                       uz, uy, ux, kz, ky, L.ptr(dyd), 1 if dy_bf16 else 0, cout, cout, L.ptr(work), need, L.ptr(dw),
                                       L.ptr(db), L.stream_ptr()))
    return dw.cpu().numpy(), db.cpu().numpy()


@pytest.mark.parametrize("case", C.CONV + C.DECODER, ids=lambda c: c['id'])
def test_conv_bf16_exact_on_integers(case):
    """forward (with bias and ReLU), input gradient and weight gradient equal float64 element by element; the bf16 outputs are
    rne of the float64 result (integer sums above 256 are ties)"""
    x, lo, skip, k, b, dy = C.int_data(case)
    y64, dw64, db64, dx64 = C.conv64(x, k, b, dy, case['nd'])
    y = _run_forward(case, lo, skip, k, b, 1)
    assert np.array_equal(y, C.rne(np.maximum(y64, 0).astype(np.float32)))
    assert np.array_equal(_run_forward(case, lo, skip, k, b, 0), C.rne(y64.astype(np.float32)))
    dw, db = _run_wgrad(case, lo, skip, dy)
    assert np.array_equal(dw.astype(np.float64), dw64) and np.array_equal(db.astype(np.float64), db64)
    if 'up' not in case and case['cin'] > 4:
        assert np.array_equal(_run_dgrad(case, dy, k), C.rne(dx64.astype(np.float32)))


@pytest.mark.parametrize("case", C.ROUNDING, ids=lambda c: c['id'])
def test_conv_bf16_rounding_is_rne(case):
    """12-bit operands: every result equals float64 of the rne-rounded operands (then rne for bf16 stores); the truncation
    mutant does not match; with an fp32 dy (the heads) the operand is rounded on load and db sums it unrounded"""
    x, k, dy = C.rounding_data(case)
    b = np.zeros(case['cout'], np.float32)
    r, t = C.rne, C.round_truncate
    y64, dw64, db64, dx64 = C.conv64(r(x), r(k), b, r(dy), case['nd'])
    y = _run_forward(case, None, r(x), k, b, 0)                           # the input is stored bf16; the kernel rounded on copy
    assert np.array_equal(y, r(y64.astype(np.float32)))
    assert not np.array_equal(y, r(C.conv64(t(x), t(k), b, dy, case['nd'])[0].astype(np.float32)))
    dw, db = _run_wgrad(case, None, r(x), dy, dy_bf16=False)
    assert np.array_equal(dw.astype(np.float64), dw64)
    assert np.array_equal(db.astype(np.float64), C.conv64(x, k, b, dy, case['nd'])[2])
    assert not np.array_equal(dw.astype(np.float64), C.conv64(t(x), t(k), b, t(dy), case['nd'])[1])
    if case['cin'] > 4:
        gin = _run_dgrad(case, r(dy), k)
        assert np.array_equal(gin, r(dx64.astype(np.float32)))


# ------------------------------------------------------------------------------------------------ whole network
def _rne64(t):
    return torch.from_numpy(C.rne(t.detach().numpy().astype(np.float32)).astype(np.float64))


class _Bf16Conv(torch.autograd.Function):
    """float64 convolution at the mixed_bfloat16 trainer's rounding points: rne operands; a hidden layer's output and input
    gradient stored as rne; its stored output gradient is rne (the sum of its consumers' gradients, masked by ReLU); a head's
    output fp32-exact, its upstream gradient rounded as a GEMM operand while its bias gradient sums it unrounded"""

    @staticmethod
    def forward(ctx, x, w, b, conv, head):
        xr, wr = _rne64(x), _rne64(w)
        ctx.save_for_backward(xr, wr)
        ctx.conv, ctx.head = conv, head
        y = conv(xr, wr, b, padding='same')
        return y if head else _rne64(y)

    @staticmethod
    def backward(ctx, gy):
        xr, wr = ctx.saved_tensors
        conv = ctx.conv
        gr = _rne64(gy)
        with torch.enable_grad():
            x2, w2 = xr.clone().requires_grad_(True), wr.clone().requires_grad_(True)
            dx, dw = torch.autograd.grad(conv(x2, w2, None, padding='same'), (x2, w2), gr)
        db = (gy if ctx.head else gr).sum(dim=[0] + list(range(2, gy.dim())))
        return _rne64(dx), dw, db, None, None


@contextmanager
def _bf16_oracle(nd, P):
    name = 'conv2d' if nd == 2 else 'conv3d'
    orig = getattr(F, name)
    heads = {id(P[n][0]) for n in ('prob', 'dist', 'prob_class') if n in P}

    def conv(x, w, b=None, padding=0, **kw):
        return _Bf16Conv.apply(x, w, b, orig, id(w) in heads)
    with mock.patch.object(F, name, conv):
        yield


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
        return float(tot.detach())
    if rounded:
        with _bf16_oracle(config.n_dim, P):
            loss = run()
    else:
        loss = run()
    return O.grads_keras(P), loss


# Per case (bound against the rounded float64 oracle, bound against plain float64): the worst relative L2 errors measured on an
# H100 80GB HBM3 at 700 W were (1.4e-3, 1.6e-2) for 2d, (5.8e-2, 1.3e-1) for 3d_pool122 and (1.9e-3, 2.0e-2) for 2d_classes;
# the bounds allow about 3x.  Against the oracle the kernels differ where an fp32 value lands on the other side of a bf16
# rounding boundary than the float64 one, and those differences grow along the backward chain; they are largest on the 3-D
# case's single 6x16x16 patch, whose deep layers sum few pixels.  Against plain float64 the bf16 rounding itself dominates.
BOUNDS = {'2d': (5e-3, 5e-2), '3d_pool122': (0.18, 0.4), '2d_classes': (6e-3, 6e-2)}


@pytest.mark.parametrize("case", ['2d', '3d_pool122', '2d_classes'])
def test_network_gradient_bf16(case):
    from stardist_b200.models.train import UNetTrainer
    from stardist_b200.models.weights import glorot_uniform_weights
    config = _net_config(case)
    weights = glorot_uniform_weights(config, seed=1)
    with policy('mixed_bfloat16'):
        tr = UNetTrainer(config, weights)
    assert tr.bf16
    (x,), targets = _batches(config)[0]
    got = tr.gradients(x, *targets)
    loss = float(tr.evaluate(x, *targets).cpu().numpy()[0])
    want_r, loss_r = _oracle_grads(config, weights, tr.names, x, targets, True)
    want_64, loss_64 = _oracle_grads(config, weights, tr.names, x, targets, False)
    err = {}
    for n in tr.names:
        for i, (a, b_r, b_64) in enumerate(zip(got[n], want_r[n], want_64[n])):
            a = a.astype(np.float64)
            err[(n, i)] = (np.linalg.norm(a - b_r) / max(np.linalg.norm(b_r), 1e-30),
                           np.linalg.norm(a - b_64) / max(np.linalg.norm(b_64), 1e-30))
    worst_r, worst_64 = (max(e[j] for e in err.values()) for j in (0, 1))
    print("%s: loss %.6g (rounded oracle %.6g, float64 %.6g); worst relative L2 gradient error %.3g against the rounded "
          "oracle, %.3g against plain float64" % (case, loss, loss_r, loss_64, worst_r, worst_64))
    assert abs(loss - loss_r) <= 1e-2 * abs(loss_r)
    b_r, b_64 = BOUNDS[case]
    assert worst_r <= b_r, {k: e[0] for k, e in err.items() if e[0] > b_r}
    assert worst_64 <= b_64, {k: e[1] for k, e in err.items() if e[1] > b_64}


@pytest.mark.parametrize("case", ['2d', '3d_pool122', '2d_classes'])
def test_saved_activations_are_half_the_bytes(case):
    from stardist_b200.models.train import UNetTrainer
    from stardist_b200.models.weights import glorot_uniform_weights
    config = _net_config(case)
    weights = glorot_uniform_weights(config, seed=1)
    (x,), targets = _batches(config)[0]
    nbytes = {}
    for name in ('float32', 'mixed_bfloat16'):
        with policy(name):
            tr = UNetTrainer(config, weights)
        tr.gradients(x, *targets)
        saved = tr.saved_activations()
        want = torch.bfloat16 if name == 'mixed_bfloat16' else torch.float32
        assert all(t.dtype == want for t in saved), [t.dtype for t in saved]
        nbytes[name] = sum(t.numel() * t.element_size() for t in saved)
    print("%s: saved activations %d bytes (float32), %d bytes (mixed_bfloat16)" % (case, nbytes['float32'], nbytes['mixed_bfloat16']))
    assert 2 * nbytes['mixed_bfloat16'] == nbytes['float32']


def test_bf16_training_is_deterministic():
    from stardist_b200.models.train import UNetTrainer
    from stardist_b200.models.weights import glorot_uniform_weights
    config = _net_config('3d_pool122')
    batches = _batches(config, seed=5, length=3)
    runs = []
    with policy('mixed_bfloat16'):
        for _ in range(2):
            tr = UNetTrainer(config, glorot_uniform_weights(config, seed=4))
            losses = [tr.step(x, p, d).cpu().numpy().copy() for (x,), (p, d) in batches]
            runs.append((tr.params.cpu().numpy(), np.stack(losses)))
    assert _same_bits(runs[0][0], runs[1][0]) and _same_bits(runs[0][1], runs[1][1])


def test_trainer_reads_the_policy_at_construction():
    from stardist_b200.models.train import UNetTrainer
    from stardist_b200.models.weights import glorot_uniform_weights
    config = _net_config('2d')
    weights = glorot_uniform_weights(config, seed=2)
    (x,), (p, d) = _batches(config)[0]
    with policy('mixed_bfloat16'):
        a = UNetTrainer(config, weights)
        b = UNetTrainer(config, weights)
    g_b = b.gradients(x, p, d)
    with policy('float32'):
        g_a = a.gradients(x, p, d)
        g_off = UNetTrainer(config, weights).gradients(x, p, d)
    assert a.bf16 and a.policy.name == 'mixed_bfloat16'
    for n in a.names:
        assert _same_bits(g_a[n][0], g_b[n][0]), n
    assert any(not np.array_equal(g_a[n][0], g_off[n][0]) for n in a.names)


def test_tf32_switch_has_no_effect_under_bf16():
    import stardist_b200 as s
    from stardist_b200.models.train import UNetTrainer
    from stardist_b200.models.weights import glorot_uniform_weights
    config = _net_config('2d')
    weights = glorot_uniform_weights(config, seed=3)
    (x,), (p, d) = _batches(config)[0]
    grads = []
    for on in (False, True):
        before = s.tensor_float_32_execution_enabled()
        s.enable_tensor_float_32_execution(on)
        try:
            with policy('mixed_bfloat16'):
                tr = UNetTrainer(config, weights)
        finally:
            s.enable_tensor_float_32_execution(before)
        assert not tr.tf32
        grads.append(tr.gradients(x, p, d))
    for n in grads[0]:
        assert _same_bits(grads[0][n][0], grads[1][n][0]) and _same_bits(grads[0][n][1], grads[1][n][1]), n


# ------------------------------------------------------------------------------------------------ train()
def test_train_end_to_end_bf16(tmp_path):
    from stardist_b200 import Config2D, StarDist2D
    X, Y = _small_data(2, n=6, seed=10)
    config = Config2D(n_rays=16, unet_n_depth=2, grid=(1, 1), train_patch_size=(64, 64), train_batch_size=4, train_epochs=6,
                      train_steps_per_epoch=50, train_learning_rate=1e-3)
    model = StarDist2D(config, name='bf16', basedir=str(tmp_path))
    with policy('mixed_bfloat16'), warnings.catch_warnings():
        warnings.simplefilter("ignore")
        h = model.train(X[:4], Y[:4], validation_data=(X[4:], Y[4:]), seed=0).history
    print("val_loss per epoch, mixed_bfloat16:", ["%.4f" % v for v in h['val_loss']])
    assert h['val_loss'][-1] < 0.5 * h['val_loss'][0]
    for f in ('weights.npz', 'weights_last.npz'):
        with np.load(str(tmp_path / 'bf16' / f)) as z:
            assert all(z[k].dtype == np.float32 for k in z.files)
    img = X[5]
    labels, res = model.predict_instances(img)
    reloaded = StarDist2D(None, name='bf16', basedir=str(tmp_path))
    l2, r2 = reloaded.predict_instances(img)
    assert np.array_equal(labels, l2) and np.array_equal(res['points'], r2['points'])
