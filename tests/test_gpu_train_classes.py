"""Multi-class training on the device (csrc/unet_train.cu sdb_stardist_class_loss / sdb_class_head_backward,
models/train.py): the class loss kernel against float64, the class head's input gradient bit-equal on exactly representable
data, whole-network gradients of multi-class U-Nets against float64 autograd on real StarDistData batches with classes,
determinism, Adam over the enlarged parameter buffer, an end-to-end train() with two classes, and lazy data."""
import os, sys, warnings
import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import train_oracle as O
import train_oracle_classes as OC
import train_class_cases as CC

pytestmark = pytest.mark.gpu


def _lib():
    from stardist_b200 import _lib as L
    return L, L.require_cuda()


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


# ------------------------------------------------------------------------------------------------ loss kernel
@pytest.mark.parametrize("C", [3, 5])
def test_class_loss_kernel_against_float64(C):
    """L_class and the total within 4e-6 relative; per-pixel dL/dz within 4e-6 |ref| + 1e-6 max|ref|"""
    L, lib = _lib()
    rng = np.random.default_rng(C)
    npix, w2 = 3000, 0.7
    cw = np.array([0.5, 1.0, 2.0, 1.5, 0.25][:C])
    z = rng.normal(0, 3, (npix, C))
    z[:40, 0] += 60.0                                   # saturated softmax rows: the other channels underflow / clip
    z[40:80, C - 1] += 25.0
    s = torch.softmax(torch.from_numpy(z), dim=-1).numpy().astype(np.float32)
    t = np.eye(C, dtype=np.float32)[rng.integers(0, C, npix)]
    t[100:130] = rng.dirichlet(np.ones(C), 30)          # soft targets
    t[rng.uniform(0, 1, npix) < 0.2] = -1               # ignored pixels
    s64 = torch.from_numpy(s.astype(np.float64)).requires_grad_(True)
    lc = OC.class_loss64(s64, torch.from_numpy(t.astype(np.float64)), cw)
    (w2 * lc).backward()
    want_dz = OC.softmax_backward64(s64.detach(), s64.grad).numpy()
    total0 = np.float32(1.25)                           # what sdb_stardist_loss would have written
    out = torch.tensor([total0, 0, 0, 0, -1], dtype=torch.float32, device='cuda')
    work = torch.empty(int(lib.sdb_stardist_class_loss_workspace(npix)) // 4, dtype=torch.float32, device='cuda')
    dz = torch.empty((npix, C), dtype=torch.float32, device='cuda')
    sd, td, cwd = _dev(s), _dev(t), _dev(cw)
    L.check(lib.sdb_stardist_class_loss(L.ptr(sd), L.ptr(td), npix, C, L.ptr(cwd), w2, L.ptr(work), L.ptr(dz), L.ptr(out[0:1]),
                                        L.ptr(out[4:5]), L.stream_ptr()))
    o = out.cpu().numpy().astype(np.float64)
    ref = lc.item()
    assert abs(o[4] - ref) <= 4e-6 * abs(ref), (o[4], ref)
    assert abs(o[0] - (float(total0) + w2 * ref)) <= 4e-6 * (float(total0) + w2 * ref)
    assert o[1] == 0 and o[2] == 0 and o[3] == 0
    err = np.abs(dz.cpu().numpy().astype(np.float64) - want_dz)
    assert np.all(err <= 4e-6 * np.abs(want_dz) + 1e-6 * np.abs(want_dz).max()), err.max()
    # without a gradient buffer (validation) the loss is the same
    out2 = torch.zeros(5, dtype=torch.float32, device='cuda')
    L.check(lib.sdb_stardist_class_loss(L.ptr(sd), L.ptr(td), npix, C, L.ptr(cwd), w2, L.ptr(work), None, L.ptr(out2[0:1]),
                                        L.ptr(out2[4:5]), L.stream_ptr()))
    assert out2[4].item() == out[4].item()


@pytest.mark.parametrize("relu", [0, 1])
@pytest.mark.parametrize("accumulate", [0, 1])
@pytest.mark.parametrize("case", CC.EXACT_CLASS_HEAD, ids=lambda c: c['id'])
def test_class_head_backward_exact(case, relu, accumulate):
    L, lib = _lib()
    feat, dz, W, d0 = CC.int_data(case)
    want = dz.astype(np.float64) @ W.astype(np.float64).T
    if relu:
        want = want * (feat > 0)
    if accumulate:
        want = want + d0
    out = _dev(d0)
    fd, dzd, wd = _dev(feat), _dev(dz), _dev(W)
    L.check(lib.sdb_class_head_backward(L.ptr(fd), L.ptr(dzd), case['npix'], case['cf'], L.ptr(wd), case['C'], relu, accumulate,
                                        L.ptr(out), L.stream_ptr()))
    assert np.array_equal(out.cpu().numpy().astype(np.float64), want)


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


def _class_dicts(Y, n_classes):
    """label -> class: 1 + label % n_classes for every label of every image"""
    return [{int(l): 1 + int(l) % n_classes for l in np.unique(y) if l > 0} for y in Y]


def _config(case):
    from stardist_b200 import Config2D, Config3D
    if case == '2d_classes':
        return Config2D(n_rays=16, unet_n_depth=2, unet_n_filter_base=32, grid=(1, 1), train_patch_size=(64, 64), train_batch_size=2,
                        n_classes=3, train_class_weights=(0.5, 1, 2, 1.5), train_loss_weights=(1, 0.2, 0.7))
    if case == '2d_grid_no_features':
        # the heads read the 128-channel backbone output; 8 input channels keep the first convolution off the few-channel
        # stem kernel, which has 32 or 64 outputs
        return Config2D(n_rays=16, n_channel_in=8, unet_n_depth=1, unet_n_filter_base=128, grid=(2, 2), net_conv_after_unet=0,
                        train_patch_size=(64, 64), train_batch_size=2, n_classes=3, train_class_weights=(1, 2, 0.5, 1))
    from stardist_b200.rays3d import Rays_GoldenSpiral
    return Config3D(rays=Rays_GoldenSpiral(24), unet_n_depth=2, unet_n_filter_base=32, unet_pool=(1, 2, 2), grid=(1, 2, 2),
                    train_patch_size=(6, 16, 16), train_batch_size=1, train_background_reg=1e-4, n_classes=2)


def _batches(config, seed=0, length=4):
    from stardist_b200.models import StarDistData2D, StarDistData3D
    X, Y = _small_data(config.n_dim, seed=seed, channels=config.n_channel_in)
    kw = dict(patch_size=config.train_patch_size, grid=config.grid, foreground_prob=config.train_foreground_only,
              n_classes=config.n_classes, classes=_class_dicts(Y, config.n_classes))
    np.random.seed(seed)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        if config.n_dim == 2:
            g = StarDistData2D(X, Y, batch_size=config.train_batch_size, n_rays=config.n_rays, length=length, **kw)
        else:
            from stardist_b200.rays3d import rays_from_json
            g = StarDistData3D(X, Y, batch_size=config.train_batch_size, rays=rays_from_json(config.rays_json), length=length, **kw)
        return [g.batch_device(i) for i in range(length)]


@pytest.mark.parametrize("case", ['2d_classes', '2d_grid_no_features', '3d_pool122_classes'])
def test_multiclass_network_gradient_against_float64_autograd(case):
    """every parameter tensor's gradient, features_class and prob_class included, within relative L2 1e-4 of float64 autograd"""
    from stardist_b200.models.train import UNetTrainer
    from stardist_b200.models.weights import glorot_uniform_weights
    config = _config(case)
    weights = glorot_uniform_weights(config, seed=1)
    tr = UNetTrainer(config, weights)
    assert 'prob_class' in tr.names and ('features_class' in tr.names) == (config.net_conv_after_unet > 0)
    (x,), (p, d, pc) = _batches(config)[0]
    assert (pc.cpu().numpy()[..., 1:].max(axis=-1) > 0).any()          # some pixels carry a foreground class
    got = tr.gradients(x, p, d, pc)
    P = O.params64(weights, tr.names)
    prob, dist, prob_class = OC.forward64_classes(config, P, x.cpu().double())
    w = tuple(float(v) for v in config.train_loss_weights)
    tot, _, _ = O.loss64(prob, dist, p.cpu().double(), d.cpu().double(), dist_loss=config.train_dist_loss,
                         lam=float(config.train_background_reg), weights=w[:2])
    tot = tot + w[2] * OC.class_loss64(prob_class, pc.cpu().double(), config.train_class_weights)
    tot.backward()
    want = O.grads_keras(P)
    worst = 0.0
    for n in tr.names:
        for a, b in zip(got[n], want[n]):
            rel = np.linalg.norm(a.astype(np.float64) - b) / max(np.linalg.norm(b), 1e-30)
            worst = max(worst, rel)
            assert rel <= 1e-4, (n, rel)
    print("%s: worst relative L2 gradient error %.3g" % (case, worst))


def test_multiclass_training_is_deterministic():
    from stardist_b200.models.train import UNetTrainer
    from stardist_b200.models.weights import glorot_uniform_weights
    config = _config('2d_classes')
    runs = []
    for _ in range(2):
        tr = UNetTrainer(config, glorot_uniform_weights(config, seed=4))
        losses = [tr.step(x, p, d, pc).cpu().numpy().copy() for (x,), (p, d, pc) in _batches(config, seed=5, length=5)]
        runs.append((tr.params.cpu().numpy(), np.stack(losses)))
    assert runs[0][1].shape == (5, 5) and np.all(runs[0][1][:, 4] > 0) and np.all(runs[0][1][:, 3] == 0)
    assert np.array_equal(runs[0][0], runs[1][0])
    assert np.array_equal(runs[0][1], runs[1][1])


def test_multiclass_adam_bit_identical_to_numpy():
    from stardist_b200.models.train import UNetTrainer
    from stardist_b200.models.weights import glorot_uniform_weights
    config = _config('2d_classes')
    tr = UNetTrainer(config, glorot_uniform_weights(config, seed=2))
    w = tr.params.cpu().numpy(); m = np.zeros_like(w); v = np.zeros_like(w)
    for t, ((x,), (p, d, pc)) in enumerate(_batches(config, seed=3), start=1):
        tr.gradients(x, p, d, pc)
        g = tr.grad.cpu().numpy()
        tr.step(x, p, d, pc)
        coef = tr.coef.cpu().numpy()
        w, m, v = O.adam_np(w, g, m, v, tr.lr, coef[t - 1])
        assert np.array_equal(tr.params.cpu().numpy(), w), t
        assert np.array_equal(tr.m.cpu().numpy(), m) and np.array_equal(tr.v.cpu().numpy(), v)


# ------------------------------------------------------------------------------------------------ train()
def _by_radius(Y):
    """class 1 for objects smaller than the median area of all objects, class 2 for the others"""
    areas = [np.bincount(y.ravel())[1:] for y in Y]
    thr = np.median(np.concatenate([a[a > 0] for a in areas]))
    return [{int(l): (1 if a[l - 1] < thr else 2) for l in np.unique(y) if l > 0} for y, a in zip(Y, areas)]


def test_train_multiclass_end_to_end(tmp_path):
    from stardist_b200 import Config2D, StarDist2D
    from stardist_b200.models.base import load_weights_npz
    from oracle import synth
    Y = [synth.ellipse_labels((96, 96), seed=20 + i, rmin=5, rmax=9) for i in range(15)]
    X = [synth.image_from_labels(y, seed=20 + i) for i, y in enumerate(Y)]
    cls = _by_radius(Y)
    config = Config2D(n_rays=16, unet_n_depth=2, grid=(1, 1), train_patch_size=(64, 64), train_batch_size=4, train_epochs=10,
                      train_steps_per_epoch=50, train_learning_rate=1e-3, n_classes=2)
    model = StarDist2D(config, name='m', basedir=str(tmp_path))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        hist = model.train(X[:12], Y[:12], classes=cls[:12], validation_data=(X[12:], Y[12:], cls[12:]), seed=0)
    h = hist.history
    assert list(h) == ['loss', 'prob_loss', 'dist_loss', 'prob_class_loss', 'val_loss', 'val_prob_loss', 'val_dist_loss',
                       'val_prob_class_loss', 'lr']
    assert all(len(v) == 10 for v in h.values())
    print("val_loss per epoch:", ["%.4f" % v for v in h['val_loss']])
    print("val_prob_class_loss per epoch:", ["%.4f" % v for v in h['val_prob_class_loss']])
    # the best epoch is the checkpoint the model folder keeps
    assert min(h['val_loss']) < 0.5 * h['val_loss'][0]
    assert min(h['val_prob_class_loss']) < 0.5 * h['val_prob_class_loss'][0]
    saved = load_weights_npz(tmp_path / 'm' / 'weights.npz')
    assert {'features_class', 'prob_class'} <= set(saved)
    again = StarDist2D(None, name='m', basedir=str(tmp_path))
    for n, (k, b) in model.weights.items():
        assert np.array_equal(again.weights[n][0], k) and np.array_equal(again.weights[n][1], b), n
    img, y = X[14], Y[14]
    l1, r1 = model.predict_instances(img)
    l2, r2 = again.predict_instances(img)
    assert np.array_equal(l1, l2) and np.array_equal(r1['class_id'], r2['class_id'])
    # class accuracy on matched objects (reported, not asserted): each predicted object against the true label at its centre
    hit = n = 0
    for i, (py, px) in enumerate(np.round(r1['points']).astype(int)):
        gt = int(y[py, px])
        if gt > 0:
            n += 1
            hit += int(r1['class_id'][i] == cls[14][gt])
    print("class accuracy on %d matched objects: %.3f" % (n, hit / max(n, 1)))


class _Lazy:
    def __init__(self, items):
        self.items = items

    def __len__(self):
        return len(self.items)

    def __getitem__(self, k):
        return self.items[k]


def test_multiclass_train_on_lazy_data_equals_lists():
    from stardist_b200 import Config2D, StarDist2D
    from oracle import synth
    Y = [synth.ellipse_labels((96, 96), seed=10 + i, rmin=5, rmax=9) for i in range(6)]
    X = [synth.image_from_labels(y, seed=10 + i) for i, y in enumerate(Y)]
    cls = _class_dicts(Y, 2)
    config = Config2D(n_rays=16, unet_n_depth=2, grid=(2, 2), train_patch_size=(64, 64), train_batch_size=2, train_epochs=2,
                      train_steps_per_epoch=6, train_n_val_patches=3, train_foreground_only=0.5, n_classes=2)
    runs = []
    for lazy in (False, True):
        wrap = _Lazy if lazy else list
        model = StarDist2D(config, name=None, basedir=None)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            hist = model.train(wrap(X[:4]), wrap(Y[:4]), classes=cls[:4], validation_data=(wrap(X[4:]), wrap(Y[4:]), cls[4:]), seed=3)
        runs.append((model.weights, hist.history))
    (w0, h0), (w1, h1) = runs
    assert 'val_prob_class_loss' in h0 and h0 == h1
    assert w0.keys() == w1.keys() and 'prob_class' in w0
    for n in w0:
        assert all(a.tobytes() == b.tobytes() for a, b in zip(w0[n], w1[n])), n
