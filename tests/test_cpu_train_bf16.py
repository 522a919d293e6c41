"""Host side of the mixed_bfloat16 trainer (DESIGN.md 4.2): the Keras policy API, the numpy restatement of cvt.rn.bf16.f32 on
hand cases and against torch, the rounding mutants the GPU cases reject, the exactness bounds of those cases, and the
trainer's routing of every layer under each policy, with out-of-family models refused before the device is touched."""
import os, subprocess, sys
import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
import train_bf16_cases as C


def _f(bits):
    return np.array([bits], np.uint32).view(np.float32)[0]


def _bits_of(v):
    return int(np.array([v], np.float32).view(np.uint32)[0])


@pytest.fixture
def policy():
    from stardist_b200 import mixed_precision as mp
    before = mp.global_policy()
    yield mp
    mp.set_global_policy(before)


# ------------------------------------------------------------------------------------------------ policy API
def test_policy_defaults_to_float32_in_a_fresh_process():
    out = subprocess.run([sys.executable, "-c", "from stardist_b200 import mixed_precision as m; p = m.global_policy(); "
                          "print(p.name, p.compute_dtype, p.variable_dtype)"], cwd=ROOT, capture_output=True, text=True, check=True)
    assert out.stdout.split() == ['float32', 'float32', 'float32']


def test_policy_round_trips(policy):
    policy.set_global_policy('mixed_bfloat16')
    p = policy.global_policy()
    assert (p.name, p.compute_dtype, p.variable_dtype) == ('mixed_bfloat16', 'bfloat16', 'float32')
    policy.set_global_policy(policy.Policy('float32'))
    assert policy.global_policy().name == 'float32' and policy.global_policy() == policy.Policy('float32')
    import stardist_b200
    assert stardist_b200.mixed_precision is policy


def test_policy_errors(policy):
    with pytest.raises(NotImplementedError, match='loss scaling'):
        policy.set_global_policy('mixed_float16')
    with pytest.raises(NotImplementedError, match='loss scaling'):
        policy.Policy('mixed_float16')
    for bad in ('float16', 'bfloat16', 'mixed_bf16', '', None, 3):
        with pytest.raises(ValueError):
            policy.set_global_policy(bad)
    assert policy.global_policy().name == 'float32'


# ------------------------------------------------------------------------------------------------ rne
@pytest.mark.parametrize("v,want", [
    (1.0, 1.0), (-3.0, -3.0), (0.0, 0.0), (1.0 + 2 ** -7, 1.0 + 2 ** -7),                  # already 8 significant bits
    (1.0 + 2 ** -8, 1.0), (1.0 + 3 * 2 ** -8, 1.0 + 2 ** -6),                               # ties to even
    (-(1.0 + 2 ** -8), -1.0), (-(1.0 + 3 * 2 ** -8), -(1.0 + 2 ** -6)),
    (1.0 + 2 ** -8 + 2 ** -23, 1.0 + 2 ** -7), (1.0 + 2 ** -8 - 2 ** -23, 1.0),             # just above / below the tie
    (2.0 - 2 ** -9, 2.0), (257.0, 256.0), (259.0, 260.0), (-261.0, -260.0), (263.0, 264.0),  # carry; integer ties
])
def test_rne_hand_cases(v, want):
    got = C.rne(np.float32(v))
    assert _bits_of(got) == _bits_of(want), (v, float(got), want)


@pytest.mark.parametrize("bits,want", [
    (0x00000001, 0x00000000), (0x00008000, 0x00000000), (0x00018000, 0x00020000),         # subnormals: ties to even
    (0x00008001, 0x00010000), (0x80018000, 0x80020000), (0x007FFFFF, 0x00800000),         # largest subnormal -> FLT_MIN
    (0x7F7FFFFF, 0x7F800000), (0xFF7F8000, 0xFF800000), (0x7F7F7FFF, 0x7F7F0000),         # overflow to inf; just below
    (0x7F800000, 0x7F800000), (0xFF800000, 0xFF800000),                                    # +-inf
])
def test_rne_bit_cases(bits, want):
    got = _bits_of(C.rne(_f(bits)))
    assert got == want, (hex(bits), hex(got), hex(want))


def test_rne_nan_stays_nan():
    for bits in (0x7FC00000, 0x7F800001, 0xFFFFFFFF, 0x7FFF8000):
        assert np.isnan(C.rne(_f(bits)))


def test_rne_equals_torch_bfloat16():
    import torch
    rng = np.random.default_rng(0)
    bits = rng.integers(0, 2 ** 32, 400000, dtype=np.uint64).astype(np.uint32)
    ties = (rng.integers(0, 2 ** 16, 20000, dtype=np.uint64).astype(np.uint32) << np.uint32(16)) | np.uint32(0x8000)
    edge = np.array([0, 0x80000000, 0x00008000, 0x00018000, 0x7F7FFFFF, 0x7F7F8000, 0xFF7F8000, 0x7F800000, 0xFF800000],
                    np.uint32)
    v = np.concatenate([bits, ties, edge]).view(np.float32)
    v = v[~np.isnan(v)]
    want = torch.from_numpy(v).to(torch.bfloat16).float().numpy()
    assert np.array_equal(C.rne(v).view(np.uint32), want.view(np.uint32))


def test_mutant_roundings_differ_from_rne_on_ties():
    ties = np.array([1.0 + 2 ** -8, 257.0, -(1.0 + 2 ** -8), 1.0 + 3 * 2 ** -8 + 2 ** -20], np.float32)
    assert not np.array_equal(C.round_truncate(ties), C.rne(ties))
    assert not np.array_equal(C.round_half_away(ties), C.rne(ties))
    nt = np.array([1.0, 3.0, 2.0 ** -100], np.float32)                          # exact values: every rounding agrees
    assert np.array_equal(C.round_truncate(nt), C.rne(nt)) and np.array_equal(C.round_half_away(nt), C.rne(nt))


# ------------------------------------------------------------------------------------------------ exactness bounds
@pytest.mark.parametrize("case", C.CONV + C.DECODER, ids=lambda c: c['id'])
def test_integer_cases_stay_below_2_24(case):
    assert C.max_partial(case) < 2 ** 24


def test_integer_cases_produce_bf16_ties():
    """integer outputs above 256 are not all bf16 values, so the stores round"""
    assert sum(C.max_partial(c) > 512 for c in C.CONV + C.DECODER) >= len(C.CONV + C.DECODER) - 2


@pytest.mark.parametrize("case", C.ROUNDING, ids=lambda c: c['id'])
def test_rounding_cases_are_exact_in_fp32(case):
    """rne operands of exponent 0 are multiples of 2^-7 below 2, products multiples of 2^-14 below 4: fewer than 256 terms keep
    every partial sum below 2^10 = 2^24 quanta; and the data does contain ties and values rne changes"""
    assert C.max_terms(case) < 256
    x, k, dy = C.rounding_data(case)
    for a in (x, k, dy):
        assert np.all(np.mod(C.rne(a).astype(np.float64), 2.0 ** -7) == 0) and np.any(C.rne(a) != a)
    assert any(np.any(C.rne(a) != C.round_half_away(a)) for a in (x, k, dy))


def test_exactness_bound_rejects_a_mutated_case():
    case = dict(C.ROUNDING[1], cin=32, cout=32)
    assert C.max_terms(case) >= 256
    case = dict(C.CONV[2], shape=(2048, 2048))
    assert C.max_partial(case) >= 2 ** 24


# ------------------------------------------------------------------------------------------------ routing
class _RecordingLib:
    """stands in for the CUDA library: records every entry point called; with forbid_bf16, any *bf16* name fails the test"""

    def __init__(self, forbid_bf16):
        self.calls, self.forbid_bf16 = [], forbid_bf16

    def __getattr__(self, name):
        if self.forbid_bf16 and 'bf16' in name:
            pytest.fail("%s reached under the float32 policy" % name)

        def call(*args):
            self.calls.append(name)
            return 16 if name.endswith('_workspace') else 0
        return call


def _configs():
    from stardist_b200 import Config2D, Config3D, Rays_GoldenSpiral
    return dict(
        c2d=Config2D(), c2d_classes=Config2D(n_classes=3, grid=(2, 2)), c2d_classes_128=Config2D(n_classes=4, net_conv_after_unet=128),
        c3d=Config3D(rays=Rays_GoldenSpiral(96)),
        c3d_nb=Config3D(rays=Rays_GoldenSpiral(96), unet_pool=(1, 2, 2), grid=(1, 2, 2)),
        c3d_k133=Config3D(rays=Rays_GoldenSpiral(24), unet_kernel_size=(1, 3, 3)),
        c2d_k5=Config2D(unet_kernel_size=(5, 5)),
        c2d_base16=Config2D(unet_n_filter_base=16),
        c2d_elu=Config2D(unet_activation='elu'))


def _routes(config, bf16, monkeypatch):
    """(layer, entry points of its forward, weight gradient, input gradient and ReLU backward) with a recording library"""
    import torch
    from types import SimpleNamespace
    from stardist_b200 import _lib as L
    from stardist_b200.models.train import UNetTrainer
    from stardist_b200.models.weights import unet_layers
    lib = _RecordingLib(forbid_bf16=not bf16)
    monkeypatch.setattr(L, 'load', lambda: lib)
    monkeypatch.setattr(L, 'stream_ptr', lambda stream=None: None)
    tr = UNetTrainer.__new__(UNetTrainer)
    tr.nd, tr.tf32, tr.bf16, tr._bufs, tr.net = config.n_dim, False, bf16, {}, SimpleNamespace(device='cpu')
    dt = torch.bfloat16 if bf16 else torch.float32
    sp = (4,) * config.n_dim
    out, first = [], True
    for l in unet_layers(config):
        if l['kind'] not in ('conv', 'conv_class', 'head', 'head_class'):
            continue
        k, cin, cout = tuple(l['k']), l['cin'], l['cout']
        x = torch.zeros((1,) + sp + (cin,), dtype=dt)
        g = torch.zeros((1,) + sp + (cout,), dtype=dt)
        tr.pview = {l['name']: (torch.zeros(k + (cin, cout)), torch.zeros(cout))}
        routes = {}
        if bf16 and l['kind'] in ('conv', 'conv_class'):
            lib.calls.clear()
            tr._conv_bf16(x, None, (1,) * config.n_dim, l)
            routes['fwd'] = lib.calls[:]
        lib.calls.clear()
        tr._wgrad(x, None, (1,) * config.n_dim, k, g, cout, cout, torch.zeros(k + (cin, cout)), torch.zeros(cout))
        routes['wgrad'] = [c for c in lib.calls if not c.endswith('_workspace')]
        if l['kind'] in ('conv', 'conv_class') and not first:
            lib.calls.clear()
            tr._dgrad(0, l['name'], g, x.shape, cin, cout, k)
            routes['dgrad'] = lib.calls[:]
        if l.get('act') == 'relu':
            lib.calls.clear()
            tr._act_backward(g, 'relu', g, None)
            routes['act'] = lib.calls[:]
        first = first and l['kind'] != 'conv'
        out.append((l['name'], routes))
    return out


@pytest.mark.parametrize("name", ['c2d', 'c2d_classes', 'c3d_nb', 'c3d_k133', 'c2d_k5', 'c2d_base16'])
def test_float32_never_reaches_a_bf16_entry_point(name, monkeypatch, policy):
    from stardist_b200.models.train import check_trainable
    config = _configs()[name]
    policy.set_global_policy('float32')
    check_trainable(config)
    for layer, r in _routes(config, False, monkeypatch):
        assert not any('bf16' in c for v in r.values() for c in v), (layer, r)


@pytest.mark.parametrize("name", ['c2d', 'c2d_classes', 'c2d_classes_128', 'c3d', 'c3d_nb', 'c3d_k133'])
def test_bf16_routes_every_layer_to_the_bf16_kernels(name, monkeypatch, policy):
    from stardist_b200.models.train import check_trainable
    config = _configs()[name]
    policy.set_global_policy('mixed_bfloat16')
    check_trainable(config)
    routes = _routes(config, True, monkeypatch)
    assert routes
    for layer, r in routes:
        assert r['wgrad'] == ['sdb_conv_wgrad_bf16_nd'], (layer, r)
        if 'fwd' in r:
            assert r['fwd'] == ['sdb_weights_bf16', 'sdb_conv_bf16_nd'], (layer, r)
        if 'dgrad' in r:
            assert r['dgrad'] == ['sdb_weights_bf16', 'sdb_conv_bf16_nd'], (layer, r)
        if 'act' in r:
            assert r['act'] == ['sdb_relu_backward_bf16'], (layer, r)


@pytest.mark.parametrize("name,layer", [('c2d_k5', 'down_level_0_no_0'), ('c2d_base16', 'down_level_0_no_0'),
                                        ('c2d_elu', 'down_level_0_no_0')])
def test_out_of_family_models_are_refused_before_the_device(name, layer, monkeypatch, policy):
    from stardist_b200 import _lib as L
    from stardist_b200.models import train as T
    from stardist_b200.models.weights import glorot_uniform_weights
    config = _configs()[name]

    def no_device(*a, **k):
        raise AssertionError("the device was touched")
    monkeypatch.setattr(L, 'require_cuda', no_device)
    monkeypatch.setattr(L, 'load', no_device)
    policy.set_global_policy('mixed_bfloat16')
    with pytest.raises(NotImplementedError, match="layer %s " % layer):
        T.UNetTrainer(config, glorot_uniform_weights(config, seed=0))
    with pytest.raises(NotImplementedError, match="layer %s " % layer):
        T.check_trainable(config)
    policy.set_global_policy('float32')
    T.check_trainable(config)                                   # trains as before under float32


def test_family_predicate():
    from stardist_b200.models.unet_device import conv_bf16_accepts as acc
    assert acc(2, (3, 3), 1, 0, 32, 'relu') and acc(2, (3, 3), 3, 0, 64, 'relu') and acc(3, (3, 3, 3), 4, 0, 32, 'linear')
    assert acc(2, (3, 3), 32, 64, 32, 'relu') and acc(3, (1, 3, 3), 64, 64, 128, 'relu') and acc(2, (1, 1), 128, 0, 32, 'linear')
    assert not acc(2, (5, 5), 32, 0, 32, 'relu') and not acc(2, (3, 3), 32, 0, 16, 'relu') and not acc(2, (3, 3), 32, 0, 32, 'elu')
    assert not acc(2, (3, 3), 12, 0, 32, 'relu') and not acc(2, (3, 3), 2, 2, 32, 'relu') and not acc(3, (3, 1, 1), 32, 0, 32, 'relu')
