"""Host side of the TF32 backward pass (DESIGN.md 4.2): the numpy restatement of cvt.rna.tf32.f32 on hand cases, the
exactness bounds of the layer cases the GPU tests run, the rounding mutants those cases reject, the public switch, and the
trainer's routing of each convolution gradient with the switch off and on."""
import os, subprocess, sys
import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
import train_tf32_cases as C


def _f(bits):
    return np.array([bits], np.uint32).view(np.float32)[0]


def _bits_of(v):
    return int(np.array([v], np.float32).view(np.uint32)[0])


# ------------------------------------------------------------------------------------------------ rna
@pytest.mark.parametrize("v,want", [
    (1.0, 1.0), (-3.0, -3.0), (0.0, 0.0), (1.0 + 2 ** -10, 1.0 + 2 ** -10),                # already 11 significant bits
    (1.0 + 2 ** -11, 1.0 + 2 ** -10), (-(1.0 + 2 ** -11), -(1.0 + 2 ** -10)),            # ties round away from zero
    (1.0 + 3 * 2 ** -11, 1.0 + 2 ** -9), (-(1.0 + 3 * 2 ** -11), -(1.0 + 2 ** -9)),
    (1.0 + 2 ** -11 - 2 ** -23, 1.0), (1.0 + 2 ** -11 + 2 ** -23, 1.0 + 2 ** -10),         # just below / above the tie
    (2.0 - 2 ** -23, 2.0), (-(2.0 - 2 ** -12), -2.0),                                      # carry into the exponent
    (4095.0, 4096.0), (4093.0, 4094.0), (2049.0, 2050.0), (-2051.0, -2052.0),              # 12-bit integers: ties
])
def test_rna_hand_cases(v, want):
    got = C.rna(np.float32(v))
    assert _bits_of(got) == _bits_of(want), (v, float(got), want)


@pytest.mark.parametrize("bits,want", [
    (0x00000001, 0x00000000), (0x00000FFF, 0x00000000), (0x00001000, 0x00002000),         # subnormals: below, at the tie
    (0x00005000, 0x00006000), (0x80005000, 0x80006000), (0x00003FFF, 0x00004000),
    (0x007FF000, 0x00800000),                                                              # largest subnormals -> FLT_MIN
    (0x7F7FFFFF, 0x7F800000), (0xFF7FF000, 0xFF800000),                                    # rounding past FLT_MAX -> inf
    (0x7F800000, 0x7F800000), (0xFF800000, 0xFF800000),                                    # +-inf
])
def test_rna_bit_cases(bits, want):
    got = _bits_of(C.rna(_f(bits)))
    assert got == want, (hex(bits), hex(got), hex(want))


def test_rna_nan_stays_nan():
    for bits in (0x7FC00000, 0x7F800001, 0xFFFFFFFF, 0x7FBFF000):
        assert np.isnan(C.rna(_f(bits)))


def test_rna_equals_an_independent_restatement():
    """nearest 11-significant-bit value, ties away from zero, computed in float64 from frexp, on normal float32 values"""
    rng = np.random.default_rng(0)
    v = (rng.standard_normal(200000) * 2.0 ** rng.integers(-60, 60, 200000)).astype(np.float32)
    v[:1000] = (rng.integers(2 ** 11, 2 ** 12, 1000) * 2.0 ** rng.integers(-30, 30, 1000)).astype(np.float32)   # ties
    m, e = np.frexp(v.astype(np.float64))
    s = np.abs(m) * 2.0 ** 11
    want = (np.sign(m) * np.floor(s + 0.5) / 2.0 ** 11 * 2.0 ** e).astype(np.float32)
    assert np.array_equal(C.rna(v).view(np.uint32), want.view(np.uint32))


def test_mutant_roundings_differ_from_rna_on_ties():
    ties = np.array([2049, 2051, 2053, -2049, -2051], np.float32)
    assert not np.array_equal(C.round_truncate(ties), C.rna(ties))
    assert not np.array_equal(C.round_half_even(ties), C.rna(ties))
    assert np.array_equal(C.round_half_even(np.float32([2051, 2049])), np.float32([2052, 2048]))


# ------------------------------------------------------------------------------------------------ exactness bounds
@pytest.mark.parametrize("case", C.TF32_WGRAD + C.TF32_DECODER + C.TF32_DGRAD, ids=lambda c: c['id'])
def test_integer_cases_stay_below_2_24(case):
    assert C.max_partial(case) < 2 ** 24


@pytest.mark.parametrize("case", C.ROUNDING_WGRAD, ids=lambda c: c['id'])
def test_rounding_wgrad_cases_are_exact(case):
    x, dy = C.rounding_wgrad_data(case)
    off = case.get('off', 0)
    bound, multiples = C.rounding_bound(x, dy[..., off:off + case['cout']], None, case['nd'], case['k'])
    assert multiples and bound < 2 ** 24, bound
    assert np.count_nonzero(dy) >= 3 * min(case['cout'], 3)          # the case does test something
    m = np.frexp(np.abs(x[x != 0]))[0] * 2 ** 12
    assert np.all(m == np.round(m)) and (np.mod(m, 2) == 1).mean() > 0.4     # 12 significant bits, ~half exact ties


@pytest.mark.parametrize("case", C.ROUNDING_DGRAD, ids=lambda c: c['id'])
def test_rounding_dgrad_cases_are_exact(case):
    dy, k = C.rounding_dgrad_data(case)
    bound, multiples = C.rounding_bound(None, dy, k, case['nd'])
    assert multiples and bound < 2 ** 24, bound


def test_exactness_bound_rejects_dense_twelve_bit_data():
    """the bound is what makes the rounding cases exact: dense 12-bit operands would overflow fp32's 24 bits"""
    rng = np.random.default_rng(1)
    x = C.twelve_bit(rng, (1, 8, 8, 32), 0)
    dy = C.twelve_bit(rng, (1, 8, 8, 32), 0)
    bound, _ = C.rounding_bound(x, dy, None, 2, (3, 3))
    assert bound >= 2 ** 24


# ------------------------------------------------------------------------------------------------ mutants
@pytest.mark.parametrize("case", C.ROUNDING_WGRAD, ids=lambda c: c['id'])
def test_wgrad_rounding_cases_reject_mutants(case):
    """the expected dW and db of a rounding case differ from what truncation, round-half-even or a rounded bias give"""
    x, dy = C.rounding_wgrad_data(case)
    off = case.get('off', 0)
    dy = dy[..., off:off + case['cout']]
    want_dw, rounded_db, _ = C.conv_grads64(C.rna(x), C.rna(dy), None, case['nd'], case['k'])
    want_db = C.conv_grads64(x, dy, None, case['nd'], case['k'])[1]
    for mutant in (C.round_truncate, C.round_half_even):
        dw, _, _ = C.conv_grads64(mutant(x), mutant(dy), None, case['nd'], case['k'])
        assert not np.array_equal(dw, want_dw), mutant.__name__
    assert not np.array_equal(rounded_db, want_db)


@pytest.mark.parametrize("case", C.ROUNDING_DGRAD, ids=lambda c: c['id'])
def test_dgrad_rounding_cases_reject_mutants(case):
    dy, k = C.rounding_dgrad_data(case)
    x0 = np.zeros(dy.shape[:-1] + (case['cin'],), np.float32)
    _, _, want = C.conv_grads64(x0, C.rna(dy), C.rna(k), case['nd'])
    for mutant in (C.round_truncate, C.round_half_even):
        _, _, got = C.conv_grads64(x0, mutant(dy), mutant(k), case['nd'])
        assert not np.array_equal(got, want), mutant.__name__


# ------------------------------------------------------------------------------------------------ the switch
def test_switch_defaults_to_off_in_a_fresh_process():
    code = "import stardist_b200 as s; print(s.tensor_float_32_execution_enabled())"
    r = subprocess.run([sys.executable, "-s", "-c", code], cwd=ROOT, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    assert r.stdout.strip().splitlines()[-1] == "False"


def test_switch_round_trips():
    import stardist_b200 as s
    before = s.tensor_float_32_execution_enabled()
    try:
        s.enable_tensor_float_32_execution(True)
        assert s.tensor_float_32_execution_enabled() is True
        s.enable_tensor_float_32_execution(False)
        assert s.tensor_float_32_execution_enabled() is False
        s.enable_tensor_float_32_execution(1)
        assert s.tensor_float_32_execution_enabled() is True
    finally:
        s.enable_tensor_float_32_execution(before)


# ------------------------------------------------------------------------------------------------ routing
class _RecordingLib:
    """stands in for the CUDA library: records every entry point called; with forbid_tf32, any *_tf32* name fails the test"""

    def __init__(self, forbid_tf32):
        self.calls, self.forbid_tf32 = [], forbid_tf32

    def __getattr__(self, name):
        if self.forbid_tf32 and '_tf32' in name:
            pytest.fail("%s reached with the switch off" % name)

        def call(*args):
            self.calls.append(name)
            return 16 if name.endswith('_workspace') else 0
        return call


def _configs():
    from stardist_b200 import Config2D, Config3D, Rays_GoldenSpiral
    return dict(
        c2d=Config2D(), c2d_classes=Config2D(n_classes=3, grid=(2, 2)),
        c3d=Config3D(rays=Rays_GoldenSpiral(96), unet_pool=(1, 2, 2), grid=(1, 2, 2)),
        c3d_k133=Config3D(rays=Rays_GoldenSpiral(24), unet_kernel_size=(1, 3, 3)),
        c2d_k5=Config2D(unet_kernel_size=(5, 5)),
        c2d_base16=Config2D(unet_n_filter_base=16))


def _routes(config, tf32, monkeypatch):
    """(layer, wgrad entry point, dgrad entry point) of every convolution gradient the trainer sends, with a recording library"""
    import torch
    from types import SimpleNamespace
    from stardist_b200 import _lib as L
    from stardist_b200.models.train import UNetTrainer
    from stardist_b200.models.weights import unet_layers
    lib = _RecordingLib(forbid_tf32=not tf32)
    monkeypatch.setattr(L, 'load', lambda: lib)
    monkeypatch.setattr(L, 'stream_ptr', lambda stream=None: None)
    tr = UNetTrainer.__new__(UNetTrainer)
    tr.nd, tr.tf32, tr._bufs, tr.net = config.n_dim, tf32, {}, SimpleNamespace(device='cpu')
    sp = (4,) * config.n_dim
    out, first = [], True
    for l in unet_layers(config):
        if l['kind'] not in ('conv', 'conv_class', 'head', 'head_class'):
            continue
        k, cin, cout = tuple(l['k']), l['cin'], l['cout']
        x = torch.zeros((1,) + sp + (cin,))
        g = torch.zeros((1,) + sp + (cout,))
        lib.calls.clear()
        tr._wgrad(x, None, (1,) * config.n_dim, k, g, cout, cout, torch.zeros(k + (cin, cout)), torch.zeros(cout))
        wg = [c for c in lib.calls if c.startswith('sdb_conv_wgrad') and not c.endswith('_workspace')]
        dg = None
        if l['kind'] in ('conv', 'conv_class') and not first:
            tr.pview = {l['name']: (torch.zeros(k + (cin, cout)),)}
            lib.calls.clear()
            tr._dgrad(0, l['name'], g, x.shape, cin, cout, k)
            dg = [c for c in lib.calls if c != 'sdb_conv_flip_weights']
        first = first and l['kind'] != 'conv'
        out.append((l['name'], wg, dg))
    return out


@pytest.mark.parametrize("name", ['c2d', 'c2d_classes', 'c3d', 'c3d_k133', 'c2d_k5', 'c2d_base16'])
def test_switch_off_never_reaches_a_tf32_entry_point(name, monkeypatch):
    from stardist_b200.models import unet_device as U
    config = _configs()[name]
    for layer, wg, dg in _routes(config, False, monkeypatch):
        assert wg in (['sdb_conv_wgrad_nd'], ['sdb_conv_wgrad_any_nd']), (layer, wg)
        assert dg in (None, ['sdb_conv3_nd'], ['sdb_conv_dgrad_any_nd']), (layer, dg)


@pytest.mark.parametrize("name", ['c2d', 'c2d_classes', 'c3d', 'c3d_k133', 'c2d_k5', 'c2d_base16'])
def test_switch_on_routes_exactly_the_accepted_layers(name, monkeypatch):
    """TF32 for every layer conv_wgrad_accepts / conv_dgrad3_accepts takes; the any-extent kernels for the rest"""
    from stardist_b200.models import unet_device as U
    from stardist_b200.models.weights import unet_layers
    config = _configs()[name]
    layers = {l['name']: l for l in unet_layers(config)}
    n_tf32 = 0
    for layer, wg, dg in _routes(config, True, monkeypatch):
        l = layers[layer]
        want_wg = 'sdb_conv_wgrad_tf32_nd' if U.conv_wgrad_accepts(config.n_dim, l['k']) else 'sdb_conv_wgrad_any_nd'
        assert wg == [want_wg], (layer, wg)
        if dg is not None:
            tf32 = U.conv_dgrad3_accepts(config.n_dim, l['k'], l['cin'], l['cout'])
            assert dg == ['sdb_conv_dgrad_tf32_nd' if tf32 else 'sdb_conv_dgrad_any_nd'], (layer, dg)
            n_tf32 += tf32
        n_tf32 += want_wg.endswith('tf32_nd')
    if name in ('c2d', 'c2d_classes', 'c3d'):
        assert n_tf32 > 0
