"""Models outside the default architecture family (any kernel extent, channel width, feature width and Keras activation),
without a device: layer lists and weight shapes, which layers leave the unet_simt.cu kernels, the settings refused before
the device is touched, the float64 restatement of tests/any_config_oracle.py, and the exactness bound of the integer
layer cases of tests/test_gpu_any_config.py."""
import itertools

import numpy as np
import pytest

import any_config_oracle as O


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


CONFIGS = list(_configs())


def _routes(config):
    """per layer of the network: the kernel family the CUDA-core executor picks ('simt' = unet_simt.cu, 'any' = unet_any.cu)"""
    from stardist_b200.models import unet_device as U
    from stardist_b200.models.weights import net_layers
    nd, out = config.n_dim, {}
    resnet = getattr(config, 'backbone', 'unet') == 'resnet'
    for l in net_layers(config):
        if l['kind'] in ('conv', 'conv_class'):
            stride = l.get('stride', (1,) * nd)
            if resnet and not (tuple(l['k']) == (3, 3, 3) and tuple(stride) == (1, 1, 1) and l['cin'] > 4):
                ok = U.conv_generic_accepts(l['act'])
            else:
                c_lo = l.get('cin_lo', 0)
                ok = U.conv3_accepts(nd, l['k'], stride, l['cin'] - c_lo, c_lo, l['cout'], l['act'])
            out[l['name']] = 'simt' if ok else 'any'
        elif l['kind'] == 'head' and l['name'] == 'prob':
            out['heads'] = 'simt' if U.heads_accept(l['cin'], config.n_rays) else 'any'
        elif l['kind'] == 'block_end':
            out.setdefault('add_act', set()).add('simt' if U.add_act_accepts(l['act']) else 'any')
    return out


@pytest.mark.parametrize("name", CONFIGS)
def test_layer_lists_and_weight_shapes(name):
    from stardist_b200.models.base import StarDistBase
    from stardist_b200.models.weights import net_layers, glorot_uniform_weights
    config = _configs()[name]
    layers = net_layers(config)
    W = glorot_uniform_weights(config)
    StarDistBase._check_weights(config, W)
    for l in layers:
        if l['kind'] in ('conv', 'head', 'conv_class', 'head_class'):
            assert W[l['name']][0].shape == tuple(l['k']) + (l['cin'], l['cout'])
    convs = [l for l in layers if l['kind'] == 'conv']
    heads = {l['name']: l for l in layers if l['kind'] == 'head'}
    if getattr(config, 'backbone', 'unet') == 'unet':
        assert all(tuple(l['k']) == tuple(config.unet_kernel_size) for l in convs)
        assert convs[0]['cin'] == config.n_channel_in
        n_after = config.net_conv_after_unet
        assert ('features' in W) == (n_after > 0)
        assert heads['prob']['cin'] == (n_after if n_after > 0 else config.unet_n_filter_base)
    else:
        assert any(tuple(l['stride']) != (1, 1, 1) for l in convs)
        assert heads['prob']['cin'] == config.net_conv_after_resnet
    assert W['dist'][0].shape[-1] == config.n_rays
    if config.n_classes is not None:
        assert W['prob_class'][0].shape[-2:] == (config.net_conv_after_unet, config.n_classes + 1)
    # a wrong kernel extent is refused when weights are loaded
    bad = dict(W)
    k, b = W[convs[1]['name']]
    bad[convs[1]['name']] = (np.zeros(k.shape[:-3] + (k.shape[-3] + 1,) + k.shape[-2:], np.float32), b)
    with pytest.raises(ValueError, match='kernel shape'):
        StarDistBase._check_weights(config, bad)


@pytest.mark.parametrize("name", CONFIGS)
def test_new_configurations_leave_the_default_kernels(name):
    """each configuration has a layer none of the unet_simt.cu kernels accepts (so it could not predict before)"""
    r = _routes(_configs()[name])
    assert 'any' in set(itertools.chain.from_iterable(v if isinstance(v, set) else [v] for v in r.values())), r


def test_default_configurations_stay_on_the_default_kernels():
    from stardist_b200 import Config2D, Config3D, Rays_GoldenSpiral
    for config in (Config2D(), Config2D(n_rays=64, grid=(2, 2)), Config2D(n_classes=3), Config3D(rays=Rays_GoldenSpiral(96)),
                   Config3D(backbone='resnet', rays=Rays_GoldenSpiral(32))):
        r = _routes(config)
        assert set(itertools.chain.from_iterable(v if isinstance(v, set) else [v] for v in r.values())) == {'simt'}, r


# ------------------------------------------------------------------------------------------------ refused before the device
def _no_device(monkeypatch):
    from stardist_b200 import _lib
    monkeypatch.setattr(_lib, 'require_cuda', lambda: pytest.fail("device touched"))


@pytest.mark.parametrize("act", ['hard_sigmoid', 'leaky_relu', 'softmax'])
@pytest.mark.parametrize("where", ['unet_activation', 'unet_last_activation'])
def test_unsupported_activation_raises_before_the_device(act, where, monkeypatch):
    from stardist_b200 import Config2D, StarDist2D
    _no_device(monkeypatch)
    model = StarDist2D(Config2D(n_rays=8, **{where: act}), name=None, basedir=None)
    with pytest.raises(NotImplementedError, match=act):
        model.net


def test_unsupported_activation_raises_before_the_device_3d_and_resnet(monkeypatch):
    from stardist_b200 import Config3D, StarDist3D, Rays_GoldenSpiral
    _no_device(monkeypatch)
    r = Rays_GoldenSpiral(16)
    with pytest.raises(NotImplementedError, match='hard_sigmoid'):
        StarDist3D(Config3D(rays=r, unet_activation='hard_sigmoid'), name=None, basedir=None).net
    with pytest.raises(NotImplementedError, match='hard_sigmoid'):
        StarDist3D(Config3D(rays=r, backbone='resnet', resnet_activation='hard_sigmoid'), name=None, basedir=None).net


def test_batch_norm_raises_before_the_device(monkeypatch):
    from stardist_b200 import Config2D, StarDist2D, Config3D, StarDist3D, Rays_GoldenSpiral
    from stardist_b200.models.unet_device import UNetDeviceND
    from stardist_b200.models.weights import glorot_uniform_weights
    _no_device(monkeypatch)
    for config in (Config2D(n_rays=8, unet_batch_norm=True, unet_kernel_size=(5, 5)),
                   Config3D(rays=Rays_GoldenSpiral(16), unet_batch_norm=True, unet_n_filter_base=16)):
        with pytest.raises(NotImplementedError, match='batch_norm'):
            UNetDeviceND(config, glorot_uniform_weights(config))
    with pytest.raises(NotImplementedError, match='batch_norm'):
        StarDist3D(Config3D(rays=Rays_GoldenSpiral(16), backbone='resnet', resnet_batch_norm=True), name=None, basedir=None).net


# ------------------------------------------------------------------------------------------------ the float64 restatement
def _conv_loops(x, k, b, stride):
    """direct-loop 'same' convolution (TensorFlow padding) of channels-last float64 x [N, *sp, Cin]"""
    nd = x.ndim - 2
    ks = k.shape[:nd]
    pads = [O.tf_same_pad(x.shape[1 + a], ks[a], stride[a])[0] for a in range(nd)]
    osp = [-(-x.shape[1 + a] // stride[a]) for a in range(nd)]
    out = np.zeros((x.shape[0],) + tuple(osp) + (k.shape[-1],))
    for o in itertools.product(*[range(s) for s in osp]):
        acc = np.array(b, np.float64).copy()
        for t in itertools.product(*[range(s) for s in ks]):
            i = [o[a] * stride[a] - pads[a] + t[a] for a in range(nd)]
            if all(0 <= i[a] < x.shape[1 + a] for a in range(nd)):
                acc = acc + x[(slice(None),) + tuple(i)] @ k[t]
        out[(slice(None),) + o] = acc
    return out


@pytest.mark.parametrize("k,s,shape", [((4, 1), (2, 2), (7, 6)), ((2, 2), (1, 1), (5, 4)), ((5, 5), (2, 1), (6, 9)),
                                       ((2, 3, 1), (2, 2, 1), (5, 4, 3))])
def test_conv_same_matches_direct_loops(k, s, shape):
    import torch
    rng = np.random.default_rng(1)
    x = rng.standard_normal((2,) + shape + (3,)); w = rng.standard_normal(k + (3, 4)); b = rng.standard_normal(4)
    got = O.conv_same(torch.from_numpy(x), torch.from_numpy(w), torch.from_numpy(b), stride=s).numpy()
    np.testing.assert_allclose(got, _conv_loops(x, w, b, s), rtol=1e-12, atol=1e-12)


def test_activation_table():
    import math, torch
    xs = [-20.0, -3.0, -0.5, 0.0, 0.25, 2.0, 15.0]
    x = torch.tensor(xs, dtype=torch.float64)
    want = {
        'linear': xs, 'relu': [max(v, 0) for v in xs], 'elu': [v if v > 0 else math.expm1(v) for v in xs],
        'selu': [O.SELU_SCALE * (v if v > 0 else O.SELU_ALPHA * math.expm1(v)) for v in xs],
        'tanh': [math.tanh(v) for v in xs], 'sigmoid': [1 / (1 + math.exp(-v)) for v in xs],
        'softplus': [math.log1p(math.exp(v)) for v in xs], 'softsign': [v / (1 + abs(v)) for v in xs],
        'exponential': [math.exp(v) for v in xs], 'swish': [v / (1 + math.exp(-v)) for v in xs],
        'gelu': [0.5 * v * (1 + math.erf(v / math.sqrt(2))) for v in xs],
    }
    assert set(want) == set(O.ACTS)
    for name in O.ACTS:
        np.testing.assert_allclose(O.act64(name, x).numpy(), want[name], rtol=1e-12, atol=1e-300 if name != 'gelu' else 1e-15,
                                   err_msg=name)
    from stardist_b200.models.unet_device import ACTIVATIONS
    assert list(ACTIVATIONS) == list(O.ACTS)


# ------------------------------------------------------------------------------------------------ exactness bound
@pytest.mark.parametrize("case", O.CONV_CASES, ids=lambda c: c['id'])
def test_exact_cases_stay_below_2_24(case):
    assert O.max_partial(case) < 2 ** 24


def test_conv_cases_cover_the_grid():
    C = O.CONV_CASES
    assert {c['k'] for c in C} == {(1, 3, 3), (5, 5), (2, 2), (7, 7, 7), (4, 1)}
    assert {c['s'][0] for c in C} == {1, 2}
    assert {c['c_skip'] for c in C if not c['c_lo']} == {1, 3, 5, 16, 40}
    assert {c['cout'] for c in C} == {1, 16, 48, 96}
    assert {len(c['up']) for c in C if c['c_lo']} == {2, 3}
