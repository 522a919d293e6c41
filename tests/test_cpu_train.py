"""Host side of training: the float64 loss restatement against hand-computed values and finite differences, the Adam
restatement against its formula, ReduceLROnPlateau and the best-checkpoint rule on scripted val_loss sequences, the
NotImplementedError scope of train(), and the bounds that make the exact GPU cases exact."""
import os, sys
import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import train_oracle as O
import train_cpu_cases as C


def _t(a):
    return torch.tensor(np.asarray(a, np.float64))


# ------------------------------------------------------------------------------------------------ loss restatement
def _hand_loss(prob, dist, prob_t, dam, mae, lam, w=(1.0, 0.2)):
    eps = O.EPS
    bce = []
    for y, t in zip(prob, prob_t):
        if t < 0:
            continue
        c = min(max(y, eps), O.ONE_M_EPS)
        bce.append(-(t * np.log(c + eps) + (1 - t) * np.log(1 - c + eps)))
    lp = sum(bce) / len(bce)
    R = dist.shape[1]
    M = dam[:, R].mean()
    pen = np.abs if mae else np.square
    per = []
    for i in range(len(prob)):
        m = dam[i, R]
        v = sum(m * pen(dam[i, r] - dist[i, r]) for r in range(R)) / R / (M + eps)
        if lam > 0:
            v += lam * sum((1 - m) * pen(dist[i, r]) for r in range(R)) / R
        per.append(v)
    ld = sum(per) / len(per)
    return w[0] * lp + w[1] * ld, lp, ld


@pytest.mark.parametrize("mae", [True, False])
@pytest.mark.parametrize("lam", [0.0, 0.1])
def test_loss_restatement_matches_hand_computation(mae, lam):
    prob = np.array([0.3, 1.0, 0.0, 0.9, 0.5])          # 1.0 and 0.0 lie in the clip region
    prob_t = np.array([1.0, 0.0, 0.7, -1.0, 0.2])       # pixel 3 is ignored
    dist = np.array([[1.0, 2.0], [0.5, -1.0], [3.0, 0.0], [2.0, 2.0], [0.0, 1.5]])
    dam = np.array([[1.5, 2.5, 1.0], [0.5, 0.5, 0.0], [2.0, 1.0, 1.0], [9.0, 9.0, 1.0], [0.0, 0.0, 0.0]])
    got = O.loss64(_t(prob), _t(dist), _t(prob_t), _t(dam), dist_loss='mae' if mae else 'mse', lam=lam)
    want = _hand_loss(prob, dist, prob_t, dam, mae, lam)
    for g, w in zip(got, want):
        assert abs(g.item() - w) <= 1e-12 * max(1.0, abs(w))
    # an ignored pixel changes nothing, whatever its prediction
    prob2 = prob.copy(); prob2[3] = 0.01
    assert O.loss64(_t(prob2), _t(dist), _t(prob_t), _t(dam), dist_loss='mae' if mae else 'mse', lam=lam)[1].item() == got[1].item()


@pytest.mark.parametrize("mae", [True, False])
def test_loss_gradient_against_finite_differences(mae):
    rng = np.random.default_rng(0)
    n, R = 12, 3
    z = rng.normal(0, 1.5, n)
    prob_t = rng.uniform(0, 1, n); prob_t[[2, 7]] = -1
    dist = rng.normal(2, 1, (n, R))
    dam = np.concatenate([rng.uniform(0, 4, (n, R)), (rng.uniform(0, 1, (n, 1)) < 0.5)], axis=1)
    zt, dt = _t(z).requires_grad_(True), _t(dist).requires_grad_(True)

    def f(zz, dd):
        return O.loss64(torch.sigmoid(zz), dd, _t(prob_t), _t(dam), dist_loss='mae' if mae else 'mse', lam=0.05)[0]

    f(zt, dt).backward()
    h = 1e-6
    for i in range(n):
        e = torch.zeros(n, dtype=torch.float64); e[i] = h
        fd = (f(_t(z) + e, _t(dist)) - f(_t(z) - e, _t(dist))).item() / (2 * h)
        assert abs(fd - zt.grad[i].item()) <= 1e-6 * max(1.0, abs(fd))
    for i in range(n):
        for r in range(R):
            e = torch.zeros((n, R), dtype=torch.float64); e[i, r] = h
            fd = (f(_t(z), _t(dist) + e) - f(_t(z), _t(dist) - e)).item() / (2 * h)
            assert abs(fd - dt.grad[i, r].item()) <= 1e-6 * max(1.0, abs(fd))


def test_adam_restatement_matches_formula():
    from stardist_b200.models.train import adam_coef
    rng = np.random.default_rng(1)
    w = rng.normal(0, 1, 50).astype(np.float32)
    m = np.zeros_like(w); v = np.zeros_like(w)
    wd, md, vd = w.astype(np.float64), np.zeros(50), np.zeros(50)
    lr = 1e-3
    coef = adam_coef(5)
    for t in range(1, 6):
        g = rng.normal(0, 1, 50).astype(np.float32)
        w, m, v = O.adam_np(w, g, m, v, lr, coef[t - 1])
        md = 0.9 * md + 0.1 * g; vd = 0.999 * vd + 0.001 * g.astype(np.float64) ** 2
        alpha = lr * np.sqrt(1 - 0.999 ** t) / (1 - 0.9 ** t)
        wd = wd - alpha * md / (np.sqrt(vd) + 1e-7)
        # float32 1 - beta2^t cancels: a relative error of order 1e-7 / (1 - beta2^t), as in TF's float32 computation
        assert abs(coef[t - 1] - np.sqrt(1 - 0.999 ** t) / (1 - 0.9 ** t)) <= 1e-4 * coef[t - 1]
        np.testing.assert_allclose(w, wd, rtol=0, atol=1e-6)
        np.testing.assert_allclose(m, md, rtol=1e-5, atol=1e-7)


# ------------------------------------------------------------------------------------------------ callbacks
def _run_rlr(vals, lr=1.0, **kw):
    from stardist_b200.models.train import ReduceLROnPlateau
    cb = ReduceLROnPlateau(**kw)
    lrs = []
    for v in vals:
        lrs.append(float(lr))
        lr = cb.on_epoch_end(v, lr)
    return lrs, float(lr)


def test_reduce_lr_on_plateau_patience_and_history():
    lrs, last = _run_rlr([1.0, 0.9, 0.95, 0.95, 0.8, 0.85, 0.85], factor=0.5, patience=2, min_delta=0)
    # epochs 3 and 4 do not improve on 0.9 -> reduced after epoch 4; 0.8 improves; 0.85 x2 -> reduced again
    assert lrs == [1.0, 1.0, 1.0, 1.0, 0.5, 0.5, 0.5]
    assert last == 0.25


def test_reduce_lr_equal_value_and_min_delta():
    # an equal value is no improvement
    lrs, last = _run_rlr([1.0, 1.0], factor=0.5, patience=1, min_delta=0)
    assert lrs == [1.0, 1.0] and last == 0.5
    # an improvement smaller than min_delta is none either
    lrs, last = _run_rlr([1.0, 0.95, 0.9], factor=0.5, patience=2, min_delta=0.1)
    assert lrs == [1.0, 1.0, 1.0] and last == 0.5
    # ... and a larger one resets the wait
    _, last = _run_rlr([1.0, 0.85, 0.84], factor=0.5, patience=2, min_delta=0.1)
    assert last == 1.0


def test_best_checkpoint_is_strict():
    from stardist_b200.models.train import BestCheckpoint
    cb = BestCheckpoint()
    assert [cb.improved(v) for v in [3.0, 2.0, 2.0, 2.5, 1.0, 1.0]] == [True, True, False, False, True, False]


# ------------------------------------------------------------------------------------------------ scope
def _model2d(**kw):
    from stardist_b200 import Config2D, StarDist2D
    return StarDist2D(Config2D(n_rays=8, **kw), name=None, basedir=None)


@pytest.mark.parametrize("setup,word", [
    (lambda: _model2d(n_classes=2), 'n_classes'),
    (lambda: _model2d(train_dist_loss='iou'), 'iou'),
    (lambda: _model2d(train_shape_completion=True), 'train_shape_completion'),
    (lambda: _model2d(unet_batch_norm=True), 'unet_batch_norm'),
])
def test_unsupported_settings_raise_before_the_device(setup, word, monkeypatch):
    from stardist_b200 import _lib
    monkeypatch.setattr(_lib, 'require_cuda', lambda: pytest.fail("device touched"))
    model = setup()
    X = [np.zeros((64, 64), np.float32)]; Y = [np.zeros((64, 64), np.int32)]
    with pytest.raises(NotImplementedError, match=word):
        model.train(X, Y, validation_data=(X, Y), epochs=1, steps_per_epoch=1)


def test_resnet_3d_and_optimizer_raise(monkeypatch):
    from stardist_b200 import _lib, Config3D, StarDist3D
    monkeypatch.setattr(_lib, 'require_cuda', lambda: pytest.fail("device touched"))
    model = StarDist3D(Config3D(backbone='resnet'), name=None, basedir=None)
    X = [np.zeros((16, 32, 32), np.float32)]; Y = [np.zeros((16, 32, 32), np.int32)]
    with pytest.raises(NotImplementedError, match='resnet'):
        model.train(X, Y, validation_data=(X, Y), epochs=1, steps_per_epoch=1)
    with pytest.raises(NotImplementedError, match='optimizer'):
        _model2d().prepare_for_training(optimizer='sgd')


# ------------------------------------------------------------------------------------------------ exactness bounds
@pytest.mark.parametrize("case", C.EXACT_WGRAD + C.EXACT_DECODER, ids=lambda c: c['id'])
def test_exact_cases_stay_below_2_24(case):
    assert C.max_partial(case) < 2 ** 24


def test_exactness_bound_rejects_mutants():
    big = dict(C.EXACT_WGRAD[2], shape=(2048, 2048))
    assert C.max_partial(big) >= 2 ** 24
    assert C.max_partial(C.EXACT_WGRAD[2], vmax=2 ** 11) >= 2 ** 24
