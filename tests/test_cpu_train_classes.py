"""Host side of multi-class training: the float64 class-loss restatement against a hand computation and its gradient
through the softmax against finite differences and against the closed form the device kernel evaluates, _parse_classes_arg
against the reference's own method, the settings train() rejects before the device, and the bound that makes the exact
class-head cases exact."""
import math, os, sys
import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import train_oracle as O
import train_oracle_classes as OC
import train_class_cases as CC


def _t(a):
    return torch.tensor(np.asarray(a, np.float64))


# ------------------------------------------------------------------------------------------------ loss restatement
def _hand_class_loss(s, t, w):
    eps = O.EPS
    total = 0.0
    for sp, tp in zip(s, t):
        S = sum(v + eps for v in sp)
        l = 0.0
        for k in range(len(sp)):
            c = min(max(sp[k] / S, eps), O.ONE_M_EPS)
            if tp[k] >= 0:
                l -= w[k] * tp[k] * math.log(c)
        total += l
    return total / len(s)


def test_class_loss_restatement_matches_hand_computation():
    w = (0.5, 1.0, 2.0)
    s = np.array([[0.2, 0.5, 0.3],
                  [1e-9, 0.4, 0.6],            # q_0 below eps: clipped at the lower end
                  [5.0, 0.0, 0.0],             # q_0 = 5 / (5 + 3 eps) > 1 - eps: clipped at the upper end, q_1,2 at the lower
                  [0.1, 0.1, 0.8],             # ignored pixel: counts in N, adds nothing
                  [0.3, 0.3, 0.4]])
    t = np.array([[0, 1, 0], [1, 0, 0], [1, 0, 0], [-1, -1, -1], [0.2, 0.3, 0.5]], np.float64)
    got = OC.class_loss64(_t(s), _t(t), w).item()
    want = _hand_class_loss(s, t, w)
    assert abs(got - want) <= 1e-12 * max(1.0, abs(want))
    q = s / (s + O.EPS).sum(axis=1, keepdims=True)
    assert q[1, 0] < O.EPS and q[2, 0] > O.ONE_M_EPS            # both clip ends are exercised
    s2 = s.copy(); s2[3] = (0.7, 0.2, 0.1)
    assert OC.class_loss64(_t(s2), _t(t), w).item() == got


def _closed_form_dz(s, t, w, w2):
    """the gradient sdb_stardist_class_loss evaluates (DESIGN.md 4.2), in float64"""
    eps = O.EPS
    N = s.shape[0]
    S = (s + eps).sum(axis=1, keepdims=True)
    q = s / S
    wt = np.where(t >= 0, np.asarray(w)[None] * t, 0.0)
    a = np.where((q >= eps) & (q <= O.ONE_M_EPS), -wt / q, 0.0)
    b = a / S - (a * s).sum(axis=1, keepdims=True) / S ** 2
    return (w2 / N) * s * (b - (s * b).sum(axis=1, keepdims=True))


@pytest.mark.parametrize("C", [2, 4])
def test_class_loss_gradient_against_finite_differences(C):
    rng = np.random.default_rng(C)
    n = 10
    w = rng.uniform(0.5, 2.0, C)
    z = rng.normal(0, 1.5, (n, C))
    t = np.eye(C)[rng.integers(0, C, n)]
    t[3] = -1
    t[5] = rng.dirichlet(np.ones(C))            # a soft target
    zt = _t(z).requires_grad_(True)

    def f(zz):
        return 0.7 * OC.class_loss64(torch.softmax(zz, dim=-1), _t(t), w)

    f(zt).backward()
    h = 1e-6
    for i in range(n):
        for k in range(C):
            e = torch.zeros((n, C), dtype=torch.float64); e[i, k] = h
            fd = (f(_t(z) + e) - f(_t(z) - e)).item() / (2 * h)
            assert abs(fd - zt.grad[i, k].item()) <= 1e-6 * max(1.0, abs(fd))
    # the softmax backward of the loss's gradient in s equals autograd through the softmax, and equals the closed form
    s = torch.softmax(_t(z), dim=-1).detach().requires_grad_(True)
    (0.7 * OC.class_loss64(s, _t(t), w)).backward()
    dz = OC.softmax_backward64(s.detach(), s.grad).numpy()
    np.testing.assert_allclose(dz, zt.grad.numpy(), rtol=1e-10, atol=1e-14)
    np.testing.assert_allclose(_closed_form_dz(s.detach().numpy(), t, w, 0.7), dz, rtol=1e-10, atol=1e-14)


# ------------------------------------------------------------------------------------------------ classes argument
class _Stub:
    def __init__(self, n_classes):
        self.config = type("C", (), {})()
        self.config.n_classes = n_classes


def _outcome(fn, *args):
    try:
        r = fn(*args)
        return ("ok", None if r is None else (type(r).__name__, [dict(v) if isinstance(v, dict) else v for v in r]))
    except Exception as e:
        return ("raise", type(e).__name__ if not isinstance(e, ValueError) else "ValueError", str(e))


@pytest.mark.parametrize("n_classes", [None, 1, 2])
@pytest.mark.parametrize("classes,length", [
    ('auto', 3), ('auto', 1), ('other', 2), ('', 2), ([1, 2, 1], 3), ((2, 1), 2), (np.array([1, 1]), 2), ([{1: 1, 2: 2}], 1),
    ([1, 2], 3), ((1,), 2), (np.array([1, 2, 1]), 2), (1, 2), (None, 2), (1.5, 1),
], ids=lambda v: repr(v)[:20])
def test_parse_classes_arg_equals_the_reference(n_classes, classes, length):
    if not os.path.exists("/root/reference/stardist/models/base.py"):
        pytest.skip("no reference checkout")
    sys.path.insert(0, os.path.join(HERE, "golden"))
    import _refpkg
    ref2d, _ = _refpkg.load_models()
    from stardist_b200.models.base import StarDistBase
    want = _outcome(ref2d.StarDist2D._parse_classes_arg, _Stub(n_classes), classes, length)
    got = _outcome(StarDistBase._parse_classes_arg, _Stub(n_classes), classes, length)
    if want[0] == "ok" and want[1] is not None and isinstance(classes, np.ndarray):
        assert got[0] == "ok" and np.array_equal(got[1][1], want[1][1])
    else:
        assert got == want


def test_auto_classes_for_several_classes_is_both_errors():
    from stardist_b200.models.base import StarDistBase
    with pytest.raises(ValueError, match="n_classes > 1"):
        StarDistBase._parse_classes_arg(_Stub(3), 'auto', 2)
    with pytest.raises(NotImplementedError, match="n_classes"):
        StarDistBase._parse_classes_arg(_Stub(3), 'auto', 2)


# ------------------------------------------------------------------------------------------------ scope
def _train_no_device(monkeypatch, config_kw, classes='auto', validation=None):
    from stardist_b200 import _lib, Config2D, StarDist2D
    monkeypatch.setattr(_lib, 'require_cuda', lambda: pytest.fail("device touched"))
    model = StarDist2D(Config2D(n_rays=8, **config_kw), name=None, basedir=None)
    X = [np.zeros((64, 64), np.float32)]; Y = [np.zeros((64, 64), np.int32)]
    vd = (X, Y) if validation is None else validation(X, Y)
    model.train(X, Y, validation_data=vd, classes=classes, epochs=1, steps_per_epoch=1)


@pytest.mark.parametrize("config_kw,word", [
    (dict(n_classes=32), 'n_classes'),                                        # n_classes + 1 = 33 > 32
    (dict(n_classes=2, unet_n_filter_base=16), 'features_class'),             # its input width is not a multiple of 32
])
def test_unsupported_class_settings_raise_before_the_device(config_kw, word, monkeypatch):
    with pytest.raises(NotImplementedError, match=word):
        _train_no_device(monkeypatch, config_kw, classes=[1])


@pytest.mark.parametrize("classes,validation,match", [
    ('auto', None, "n_classes > 1"),
    ('other', None, "only 'auto'"),
    ([1, 2], None, "len\\(classes\\)"),
    (1, None, "either be 'auto'"),
    ([1], lambda X, Y: (X, Y, [1], [1]), "should be 3"),
    ([1], lambda X, Y: (X,), "should be 3"),
    ([1], lambda X, Y: (X, Y, [1, 2]), "len\\(classes\\)"),
    ([1], lambda X, Y: (X, Y), "n_classes > 1"),                             # a pair takes 'auto' for its classes
])
def test_bad_classes_raise_before_the_device(classes, validation, match, monkeypatch):
    with pytest.raises(ValueError, match=match):
        _train_no_device(monkeypatch, dict(n_classes=2), classes=classes, validation=validation)


def test_n_classes_1_accepts_auto_up_to_the_device(monkeypatch):
    """with n_classes = 1, 'auto' means class 1 for every image; the first device call is the only thing that stops it"""
    with pytest.raises(pytest.fail.Exception, match="device touched"):
        _train_no_device(monkeypatch, dict(n_classes=1))


# ------------------------------------------------------------------------------------------------ exactness bound
@pytest.mark.parametrize("case", CC.EXACT_CLASS_HEAD, ids=lambda c: c['id'])
def test_exact_class_head_cases_stay_below_2_24(case):
    assert CC.max_partial(case) < 2 ** 24
    assert case['C'] <= 32 and CC.max_partial(case, vmax=2 ** 12) >= 2 ** 24
