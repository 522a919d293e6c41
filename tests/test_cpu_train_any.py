"""Training outside the default architecture family, without a device: the scope of check_trainable (new configurations
accepted, the others still refused before any device call), the exactness bound of the integer layer cases of
test_gpu_train_any.py, the float32 restatement of the activation derivatives against float64, and the per-layer routing of
the backward pass, which keeps the default configurations on the kernels they trained on before."""
import os, sys
import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import train_any_cases as C


def _no_device(monkeypatch):
    from stardist_b200 import _lib
    monkeypatch.setattr(_lib, 'require_cuda', lambda: pytest.fail("device touched"))


def _new_configs():
    from stardist_b200 import Config2D, Config3D, Rays_GoldenSpiral
    r = dict(rays=Rays_GoldenSpiral(16))
    return {
        '2d_k55_elu': Config2D(n_rays=8, unet_kernel_size=(5, 5), unet_activation='elu'),
        '2d_k22_swish': Config2D(n_rays=8, unet_kernel_size=(2, 2), unet_activation='swish', unet_last_activation='softplus'),
        '2d_k77': Config2D(n_rays=8, unet_kernel_size=(7, 7)),
        '2d_k14': Config2D(n_rays=8, unet_kernel_size=(1, 4), unet_activation='tanh'),
        '2d_base16_gelu_cin3': Config2D(n_rays=8, unet_n_filter_base=16, unet_activation='gelu', n_channel_in=3),
        '2d_classes_k55_selu': Config2D(n_rays=8, n_classes=3, unet_kernel_size=(5, 5), unet_activation='selu'),
        '2d_last_sigmoid': Config2D(n_rays=8, unet_last_activation='sigmoid'),
        '3d_k133': Config3D(unet_kernel_size=(1, 3, 3), unet_pool=(1, 2, 2), grid=(1, 2, 2), **r),
        '3d_k315_exponential': Config3D(unet_kernel_size=(3, 1, 5), unet_n_filter_base=16, unet_activation='exponential', **r),
        '3d_softsign': Config3D(unet_activation='softsign', unet_last_activation='linear', **r),
    }


@pytest.mark.parametrize("name", list(_new_configs()))
def test_new_configurations_are_trainable(name, monkeypatch):
    """check_trainable accepts them, and train() gets as far as its first device call"""
    from stardist_b200 import StarDist2D, StarDist3D
    from stardist_b200.models.train import check_trainable
    _no_device(monkeypatch)
    config = _new_configs()[name]
    check_trainable(config)
    model = (StarDist2D if config.n_dim == 2 else StarDist3D)(config, name=None, basedir=None)
    model.prepare_for_training()
    shape = (64, 64) if config.n_dim == 2 else (16, 64, 64)
    X = [np.zeros(shape + ((config.n_channel_in,) if config.n_channel_in > 1 else ()), np.float32)]
    Y = [np.zeros(shape, np.int32)]
    multi = config.n_classes is not None
    with pytest.raises(pytest.fail.Exception, match="device touched"):
        model.train(X, Y, validation_data=(X, Y, [1]) if multi else (X, Y), classes=[1] if multi else 'auto', epochs=1,
                    steps_per_epoch=1)


@pytest.mark.parametrize("kw,word", [
    (dict(unet_activation='hard_sigmoid'), 'hard_sigmoid'),
    (dict(unet_last_activation='leaky_relu'), 'leaky_relu'),
    (dict(unet_activation='softmax'), 'softmax'),
    (dict(unet_kernel_size=(9, 9)), 'unet_kernel_size'),
    (dict(unet_kernel_size=(3, 8)), 'unet_kernel_size'),
    (dict(train_dist_loss='iou'), 'iou'),
    (dict(unet_batch_norm=True, unet_kernel_size=(5, 5)), 'unet_batch_norm'),
    (dict(train_shape_completion=True, unet_activation='elu'), 'train_shape_completion'),
    (dict(n_classes=32, unet_kernel_size=(5, 5)), 'n_classes'),
    (dict(n_classes=2, unet_n_filter_base=16, unet_activation='elu'), 'features_class'),
])
def test_still_refused_before_the_device(kw, word, monkeypatch):
    from stardist_b200 import Config2D, StarDist2D
    _no_device(monkeypatch)
    model = StarDist2D(Config2D(n_rays=8, **kw), name=None, basedir=None)
    X = [np.zeros((64, 64), np.float32)]; Y = [np.zeros((64, 64), np.int32)]
    multi = kw.get('n_classes') is not None
    with pytest.raises(NotImplementedError, match=word):
        model.train(X, Y, validation_data=(X, Y, [1]) if multi else (X, Y), classes=[1] if multi else 'auto', epochs=1,
                    steps_per_epoch=1)


def test_resnet_and_optimizer_still_refused(monkeypatch):
    from stardist_b200 import Config3D, StarDist3D, Rays_GoldenSpiral
    _no_device(monkeypatch)
    model = StarDist3D(Config3D(rays=Rays_GoldenSpiral(16), backbone='resnet', resnet_activation='elu', resnet_kernel_size=(5, 5, 5)),
                       name=None, basedir=None)
    with pytest.raises(NotImplementedError, match='resnet'):
        model.prepare_for_training()
    model = StarDist3D(Config3D(rays=Rays_GoldenSpiral(16), unet_kernel_size=(1, 3, 3)), name=None, basedir=None)
    with pytest.raises(NotImplementedError, match='optimizer'):
        model.prepare_for_training(optimizer='sgd')


# ------------------------------------------------------------------------------------------------ exactness bound
@pytest.mark.parametrize("case", C.EXACT_ANY, ids=lambda c: c['id'])
def test_exact_cases_stay_below_2_24(case):
    assert C.max_partial(case) < 2 ** 24


def test_exact_cases_cover_the_grid():
    ks = {c['k'] for c in C.EXACT_ANY}
    assert {(e, e) for e in (1, 2, 4, 5, 7)} <= ks and {(1, 3, 3), (3, 1, 5)} <= ks
    assert {1, 3, 16, 48} <= {c['c_skip'] for c in C.EXACT_ANY if not c['c_lo']}
    assert {c['up'] for c in C.EXACT_ANY if c['c_lo']} == {(2, 2), (1, 2, 2)}


@pytest.mark.parametrize("mutant", [
    lambda c: dict(c, n=2 ** 14),                                           # the weight gradient's sum over the batch
    lambda c: dict(c, cout=2 ** 20),                                        # the input gradient's sum over taps x cout
    lambda c: dict(c, up=(64,) * c['nd'], cout=2 ** 14),                    # the up-sampling block sum
])
def test_exactness_bound_rejects_mutants(mutant):
    """each of the three sums can exceed 2^24 on a case made larger, and so can every case with larger operands"""
    assert any(C.max_partial(mutant(c)) >= 2 ** 24 for c in C.EXACT_ANY)
    assert all(C.max_partial(c, vmax=2 ** 12) >= 2 ** 24 for c in C.EXACT_ANY)


# ------------------------------------------------------------------------------------------------ activation derivatives
@pytest.mark.parametrize("act", C.ACTS_SMOOTH)
def test_exact_derivatives_match_float64_autograd(act):
    """the float64 closed forms the kernels are held to equal autograd of any_config_oracle.act64, except where autograd's
    own formula has cancelled (below 2^-50 in absolute value)"""
    z = C.act_points().astype(np.float64)
    want = C.act_grad_exact64(act, z)
    got = C.act_grad64(act, z)
    assert np.all(np.abs(got - want) <= 1e-12 * np.abs(want) + 2.0 ** -50)


@pytest.mark.parametrize("act", C.ACTS_SMOOTH)
def test_float32_derivatives_within_bound(act):
    z = C.act_points()
    got = C.act_grad_np(act, z).astype(np.float64)
    want, bound = C.act_grad_bound(act, z)
    err = np.abs(got - want)
    i = int(np.argmax(err / bound))
    assert np.all(err <= bound), "%s: z=%r got %r want %r bound %g" % (act, z[i], got[i], want[i], bound[i])


def test_relu_and_linear_derivatives():
    z = C.act_points()
    assert np.array_equal(C.act_grad_np('relu', z), (z > 0).astype(np.float32))        # 0 at z = 0 (TensorFlow's ReluGrad)
    assert np.array_equal(C.act_grad_np('linear', z), np.ones_like(z))


@pytest.mark.parametrize("name,formula", [
    ('tanh', lambda z: np.float32(1) - np.tanh(z) ** 2),                    # cancels once tanh rounds to +-1
    ('elu', lambda z: np.where(z > 0, np.float32(1), np.expm1(z) + np.float32(1))),
    ('sigmoid', lambda z: (lambda s: s * (np.float32(1) - s))(np.float32(1) / (np.float32(1) + np.exp(-z)))),
])
def test_bound_rejects_unstable_forms(name, formula):
    """the textbook forms lose the tails, and the bound notices"""
    z = C.act_points()
    with np.errstate(over='ignore'):
        got = formula(z).astype(np.float64)
    want, bound = C.act_grad_bound(name, z)
    assert not np.all(np.abs(got - want) <= bound)


# ------------------------------------------------------------------------------------------------ routing
def _backward_routes(config):
    """per convolution: (weight-gradient kernel, input-gradient kernel or None for the first layer, activation backward)"""
    from stardist_b200.models import unet_device as U
    from stardist_b200.models.weights import unet_layers
    nd, out, first = config.n_dim, {}, True
    for l in unet_layers(config):
        if l['kind'] not in ('conv', 'conv_class'):
            continue
        wg = 'sdb_conv_wgrad_nd' if U.conv_wgrad_accepts(nd, l['k']) else 'sdb_conv_wgrad_any_nd'
        dg = None if first else ('sdb_conv3_nd' if U.conv_dgrad3_accepts(nd, l['k'], l['cin'], l['cout']) else 'sdb_conv_dgrad_any_nd')
        ab = {'relu': 'sdb_relu_backward', 'linear': None}.get(l['act'], 'sdb_act_backward')
        out[l['name']] = (wg, dg, ab, U.keeps_preactivation(l['act']))
        first = False
    return out


def test_default_configurations_keep_their_backward_kernels():
    from stardist_b200 import Config2D, Config3D, Rays_GoldenSpiral
    for config in (Config2D(), Config2D(n_rays=64, grid=(2, 2)), Config2D(n_classes=3), Config3D(rays=Rays_GoldenSpiral(96)),
                   Config3D(rays=Rays_GoldenSpiral(96), unet_pool=(1, 2, 2), grid=(1, 2, 2), n_classes=2)):
        r = _backward_routes(config)
        assert r, config
        for name, (wg, dg, ab, keep) in r.items():
            assert wg == 'sdb_conv_wgrad_nd' and dg in (None, 'sdb_conv3_nd') and ab in ('sdb_relu_backward', None) and not keep, (name, r[name])


def test_new_configurations_leave_the_default_backward_kernels():
    cfg = _new_configs()
    r = _backward_routes(cfg['2d_k55_elu'])
    assert {v[0] for v in r.values()} == {'sdb_conv_wgrad_any_nd'}
    assert {v[1] for v in r.values()} == {None, 'sdb_conv_dgrad_any_nd'}
    assert {v[2] for v in r.values()} == {'sdb_act_backward', 'sdb_relu_backward'}     # unet_last_activation is relu
    # a 3-D (1, 3, 3) kernel is one sdb_conv_wgrad_nd always took; its input gradient needs the any-extent kernel
    r = _backward_routes(cfg['3d_k133'])
    assert {v[0] for v in r.values()} == {'sdb_conv_wgrad_nd'} and {v[1] for v in r.values()} == {None, 'sdb_conv_dgrad_any_nd'}
    # 16 channels: 3^d kernels whose transposed shape sdb_conv3_nd does not take
    r = _backward_routes(cfg['2d_base16_gelu_cin3'])
    assert 'sdb_conv_dgrad_any_nd' in {v[1] for v in r.values()}
