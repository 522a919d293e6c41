"""Test cases and float64 oracles of the mixed_bfloat16 trainer (csrc/unet_train_bf16.cu, DESIGN.md 4.2), shared by
test_cpu_train_bf16.py and test_gpu_train_bf16.py.

rne(v) is cvt.rn.bf16.f32: v rounded to 8 significant bits, to nearest, ties to even.  Two kinds of layer cases:
- integer cases: entries in [-VMAX, VMAX], which bf16 holds exactly; every partial sum is an integer below 2^24, so the fp32
  accumulators hold float64's result exactly, and a stored bf16 output is rne of it (integers above 256 give ties);
- rounding cases: operands with 12 significant bits on exponent 0 and few enough terms per sum (max_terms) that every sum of
  rne-rounded products is exact in fp32.  The kernels must then equal float64 of the rne-rounded operands; truncated
  operands would not."""
import numpy as np

VMAX = 2


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def rne(a):
    """float32 -> the nearest bf16 value (ties to even) as float32: (bits + 0x7FFF + lsb) & 0xFFFF0000 for finite values (a
    carry into the exponent is the correct rounding, up to inf); NaN stays NaN, inf stays inf"""
    a = np.asarray(a, np.float32)
    b = _bits(a).astype(np.uint64)
    r = ((b + 0x7FFF + ((b >> 16) & 1)) & 0xFFFF0000).astype(np.uint32)
    out = r.view(np.float32).reshape(a.shape)
    return np.where(np.isfinite(a), out, a).astype(np.float32)


def round_truncate(a):
    """mutant: drop the 16 low bits"""
    return (_bits(a) & np.uint32(0xFFFF0000)).view(np.float32).reshape(np.shape(a))


def round_half_away(a):
    """mutant: round to nearest, ties away from zero"""
    a = np.asarray(a, np.float32)
    b = _bits(a).astype(np.uint64)
    out = ((b + 0x8000) & 0xFFFF0000).astype(np.uint32).view(np.float32).reshape(a.shape)
    return np.where(np.isfinite(a), out, a).astype(np.float32)


# ------------------------------------------------------------------------------------------------ layer cases
# convolutions: x [n, *shape, cin] (cin = c_skip, or c_lo + c_skip with an up-sampled source), kernel k, cout outputs
CONV = [
    dict(id='2d_stem_cin1', nd=2, n=2, shape=(21, 13), k=(3, 3), cin=1, cout=32, seed=1),
    dict(id='2d_stem_cin3', nd=2, n=2, shape=(17, 19), k=(3, 3), cin=3, cout=64, seed=2),
    dict(id='2d_c32_c64_edge', nd=2, n=3, shape=(21, 37), k=(3, 3), cin=32, cout=64, seed=3),
    dict(id='2d_c64_c128', nd=2, n=1, shape=(9, 14), k=(3, 3), cin=64, cout=128, seed=5),
    dict(id='2d_k1_c128_c32', nd=2, n=1, shape=(12, 11), k=(1, 1), cin=128, cout=32, seed=8),
    dict(id='3d_stem_cin1', nd=3, n=1, shape=(5, 11, 9), k=(3, 3, 3), cin=1, cout=32, seed=9),
    dict(id='3d_c32_c32_edge', nd=3, n=2, shape=(5, 11, 9), k=(3, 3, 3), cin=32, cout=32, seed=10),
    dict(id='3d_k133_c32_c64', nd=3, n=1, shape=(4, 9, 10), k=(1, 3, 3), cin=32, cout=64, seed=11),
    dict(id='3d_k1_c64_c128', nd=3, n=1, shape=(3, 7, 9), k=(1, 1, 1), cin=64, cout=128, seed=12),
]

# decoder input [upsample(x_lo), skip], every up-sampling factor the trainers use
DECODER = [
    dict(id='2d_up22', nd=2, n=2, shape=(12, 20), k=(3, 3), up=(2, 2), c_lo=32, c_skip=32, cout=32, seed=13),
    dict(id='2d_up21', nd=2, n=1, shape=(10, 6), k=(3, 3), up=(2, 1), c_lo=64, c_skip=32, cout=32, seed=16),
    dict(id='3d_up122', nd=3, n=2, shape=(3, 8, 12), k=(3, 3, 3), up=(1, 2, 2), c_lo=32, c_skip=32, cout=32, seed=14),
    dict(id='3d_up222', nd=3, n=2, shape=(4, 8, 6), k=(3, 3, 3), up=(2, 2, 2), c_lo=64, c_skip=32, cout=64, seed=15),
    dict(id='3d_k133_up122', nd=3, n=1, shape=(2, 6, 10), k=(1, 3, 3), up=(1, 2, 2), c_lo=64, c_skip=64, cout=128, seed=17),
]

# rounding cases: 12-bit operands, at most 255 terms per sum
ROUNDING = [
    dict(id='2d_stem_cin1', nd=2, n=1, shape=(9, 7), k=(3, 3), cin=1, cout=24, seed=31),
    dict(id='2d_c24_c24', nd=2, n=1, shape=(7, 9), k=(3, 3), cin=24, cout=24, seed=32),
    dict(id='3d_k133_c16_c24', nd=3, n=1, shape=(2, 6, 5), k=(1, 3, 3), cin=16, cout=24, seed=33),
]


def npix(case):
    return case['n'] * int(np.prod(case['shape']))


def cin_of(case):
    return case['c_lo'] + case['c_skip'] if 'up' in case else case['cin']


def max_partial(case, vmax=VMAX):
    """largest |partial sum| of an integer case: forward and input gradient sum taps x channels (+ an integer bias), the
    weight gradient sums over every pixel of the batch"""
    taps = int(np.prod(case['k']))
    fwd = taps * max(cin_of(case), case['cout']) * vmax * vmax + vmax
    return max(fwd, npix(case) * vmax * vmax)


def max_terms(case):
    """largest number of products in one sum of a rounding case (forward, input gradient, weight gradient)"""
    taps = int(np.prod(case['k']))
    return max(taps * cin_of(case), taps * case['cout'], npix(case))


def upsample(lo, up):
    for ax, u in enumerate(up):
        lo = np.repeat(lo, u, axis=1 + ax)
    return lo


def int_data(case):
    """(x -- for decoder cases the concatenation [upsample(x_lo), skip] --, x_lo or None, skip or x, kernel, bias, dy) float32
    integers in [-VMAX, VMAX]"""
    rng = np.random.default_rng(case['seed'])
    n, shape, cout = case['n'], case['shape'], case['cout']
    r = lambda s: rng.integers(-VMAX, VMAX + 1, s).astype(np.float32)
    if 'up' in case:
        lo = r((n,) + tuple(s // u for s, u in zip(shape, case['up'])) + (case['c_lo'],))
        skip = r((n,) + shape + (case['c_skip'],))
        x = np.concatenate([upsample(lo, case['up']), skip], axis=-1)
    else:
        lo, skip = None, r((n,) + shape + (case['cin'],))
        x = skip
    k = r(tuple(case['k']) + (x.shape[-1], cout))
    return x, lo, skip, k, r((cout,)), r((n,) + shape + (cout,))


def twelve_bit(rng, shape):
    """+-M * 2^-11 with M in [2^11, 2^12): 12 significant bits on exponent 0; one in 16 is an exact bf16 tie"""
    m = rng.integers(2 ** 11, 2 ** 12, shape)
    s = rng.choice(np.array([-1.0, 1.0]), shape)
    return (s * m * 2.0 ** -11).astype(np.float32)


def rounding_data(case):
    """(x, kernel, dy) of a rounding case, 12-bit values on exponent 0"""
    rng = np.random.default_rng(100 + case['seed'])
    x = twelve_bit(rng, (case['n'],) + case['shape'] + (case['cin'],))
    k = twelve_bit(rng, tuple(case['k']) + (case['cin'], case['cout']))
    dy = twelve_bit(rng, (case['n'],) + case['shape'] + (case['cout'],))
    return x, k, dy


# ------------------------------------------------------------------------------------------------ float64 oracle
def conv64(x, k, b, dy, nd):
    """float64 autograd of y = conv(x, W, b, 'same') with upstream dy: (y, dW (k..., cin, cout), db, dx), channels last"""
    import torch
    import torch.nn.functional as F
    conv = F.conv2d if nd == 2 else F.conv3d
    cf = lambda a: torch.from_numpy(np.asarray(a, np.float64)).permute(0, nd + 1, *range(1, nd + 1))
    xt = cf(x).requires_grad_(True)
    kt = torch.from_numpy(np.asarray(k, np.float64)).permute(nd + 1, nd, *range(nd)).contiguous().requires_grad_(True)
    bt = torch.from_numpy(np.asarray(b, np.float64)).requires_grad_(True)
    y = conv(xt, kt, bt, padding='same')
    y.backward(cf(dy))
    back = lambda t: t.detach().permute(0, *range(2, nd + 2), 1).numpy()
    return back(y), kt.grad.permute(*range(2, nd + 2), 1, 0).numpy(), bt.grad.numpy(), back(xt.grad)
