"""Test cases and float64 oracles of the TF32 backward pass (sdb_conv_wgrad_tf32_nd / sdb_conv_dgrad_tf32_nd, DESIGN.md 4.2),
shared by test_cpu_train_tf32.py and test_gpu_train_tf32.py.

rna(v) is cvt.rna.tf32.f32: v rounded to 10 explicit mantissa bits, to nearest, ties away from zero.  Two kinds of layer cases:
- integer cases: entries in [-VMAX, VMAX], which TF32 holds exactly; every partial sum is an integer below 2^24, so the
  kernels must give float64 autograd bit for bit (the argument of train_cpu_cases.max_partial);
- rounding cases: operands with 12 significant bits (odd mantissas are exact ties at 11 bits) on one exponent per tensor,
  and a dy with at most three non-zero entries per output channel and per 3^d window, so that every product of rounded
  operands and every partial sum is exact in fp32 (rounding_bound).  The kernels must then equal float64 autograd on the
  rna-rounded operands bit for bit, with db the float64 sum of the unrounded dy; truncation or round-half-even would not."""
import numpy as np

VMAX = 2
MASK = np.uint32(0xFFFFE000)


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def rna(a):
    """cvt.rna.tf32.f32 on a float32 array: (bits + 0x1000) & 0xFFFFE000 for finite values (a carry into the exponent is the
    correct rounding, up to inf); inf and NaN unchanged"""
    a = np.asarray(a, np.float32)
    out = ((_bits(a) + np.uint32(0x1000)) & MASK).view(np.float32).reshape(a.shape)
    return np.where(np.isfinite(a), out, a).astype(np.float32)


def round_truncate(a):
    """mutant: drop the 13 low mantissa bits"""
    a = np.asarray(a, np.float32)
    return (_bits(a) & MASK).view(np.float32).reshape(a.shape)


def round_half_even(a):
    """mutant: round to nearest, ties to even (cvt.rn)"""
    a = np.asarray(a, np.float32)
    b = _bits(a)
    out = ((b + np.uint32(0xFFF) + ((b >> np.uint32(13)) & np.uint32(1))) & MASK).view(np.float32).reshape(a.shape)
    return np.where(np.isfinite(a), out, a).astype(np.float32)


# ------------------------------------------------------------------------------------------------ layer cases
# weight gradient: k the kernel extents, dy read as columns [off, off + cout) of rows of ldy floats (the heads' layout)
TF32_WGRAD = [
    dict(id='2d_stem_cin1', nd=2, n=2, shape=(21, 13), k=(3, 3), cin=1, cout=32, seed=1),
    dict(id='2d_stem_cin3', nd=2, n=2, shape=(17, 19), k=(3, 3), cin=3, cout=64, seed=2),
    dict(id='2d_c32_c64_edge', nd=2, n=3, shape=(21, 37), k=(3, 3), cin=32, cout=64, seed=3),
    dict(id='2d_c96_c32', nd=2, n=1, shape=(16, 16), k=(3, 3), cin=96, cout=32, seed=4),
    dict(id='2d_c64_c256', nd=2, n=1, shape=(9, 14), k=(3, 3), cin=64, cout=256, seed=5),
    dict(id='2d_head_prob_ldy17', nd=2, n=2, shape=(13, 16), k=(1, 1), cin=32, cout=1, ldy=17, off=0, seed=6),
    dict(id='2d_head_dist_ldy17', nd=2, n=2, shape=(13, 16), k=(1, 1), cin=32, cout=16, ldy=17, off=1, seed=7),
    dict(id='2d_k1_c128_c97', nd=2, n=1, shape=(12, 11), k=(1, 1), cin=128, cout=97, seed=8),
    dict(id='3d_stem_cin1', nd=3, n=1, shape=(5, 11, 9), k=(3, 3, 3), cin=1, cout=32, seed=9),
    dict(id='3d_c32_c32_edge', nd=3, n=2, shape=(5, 11, 9), k=(3, 3, 3), cin=32, cout=32, seed=10),
    dict(id='3d_k133_c32_c64', nd=3, n=1, shape=(4, 9, 10), k=(1, 3, 3), cin=32, cout=64, seed=11),
    dict(id='3d_head_dist_ldy97', nd=3, n=1, shape=(3, 8, 8), k=(1, 1, 1), cin=32, cout=96, ldy=97, off=1, seed=12),
]

# decoder input [upsample(x_lo), skip] (3^d kernels)
TF32_DECODER = [
    dict(id='2d_up22', nd=2, n=2, shape=(12, 20), up=(2, 2), c_lo=32, c_skip=32, cout=32, seed=13),
    dict(id='3d_up122', nd=3, n=2, shape=(3, 8, 12), up=(1, 2, 2), c_lo=32, c_skip=32, cout=32, seed=14),
    dict(id='3d_up222', nd=3, n=2, shape=(4, 8, 6), up=(2, 2, 2), c_lo=64, c_skip=32, cout=64, seed=15),
]

# input gradient on the flipped 3^d kernel: cout = dy's channels, cin = the layer input's (conv_dgrad3_accepts)
TF32_DGRAD = [
    dict(id='2d_c32_c32', nd=2, n=2, shape=(17, 23), cin=32, cout=32, seed=21),
    dict(id='2d_c96_c64', nd=2, n=1, shape=(16, 16), cin=96, cout=64, seed=22),
    dict(id='2d_c64_c8', nd=2, n=2, shape=(9, 35), cin=64, cout=8, seed=23),
    dict(id='2d_stem_c32_c3', nd=2, n=2, shape=(11, 12), cin=32, cout=3, seed=24),
    dict(id='2d_c256_c128', nd=2, n=1, shape=(8, 8), cin=256, cout=128, seed=25),
    dict(id='3d_c64_c32', nd=3, n=2, shape=(5, 7, 9), cin=64, cout=32, seed=26),
    dict(id='3d_stem_c64_c4', nd=3, n=1, shape=(4, 6, 10), cin=64, cout=4, seed=27),
    dict(id='3d_c32_c16', nd=3, n=1, shape=(6, 5, 13), cin=32, cout=16, seed=28),
]

ROUNDING_WGRAD = [c for c in TF32_WGRAD if c['id'] in ('2d_stem_cin1', '2d_c32_c64_edge', '2d_head_dist_ldy17', '3d_c32_c32_edge',
                                                       '3d_k133_c32_c64')]
ROUNDING_DGRAD = [c for c in TF32_DGRAD if c['id'] in ('2d_c32_c32', '2d_stem_c32_c3', '3d_c64_c32')]


def _npix(case):
    return case['n'] * int(np.prod(case['shape']))


def max_partial(case, vmax=VMAX):
    """largest |partial sum| of an integer case: the weight and bias gradients sum over every pixel of the batch, the input
    gradient over taps x cout"""
    if 'k' in case or 'up' in case:
        return _npix(case) * vmax * vmax
    return 3 ** case['nd'] * case['cout'] * vmax * vmax


def upsample(lo, up):
    """nearest up-sampling of a channels-last batch by integer factors"""
    for ax, u in enumerate(up):
        lo = np.repeat(lo, u, axis=1 + ax)
    return lo


def int_wgrad_data(case):
    """(x [n, *shape, cin] -- for decoder cases the concatenation [upsample(x_lo), skip] -- , x_lo or None, skip or x,
    dy rows [n, *shape, ldy]) float32 integers in [-VMAX, VMAX]"""
    rng = np.random.default_rng(case['seed'])
    n, shape = case['n'], case['shape']
    ldy = case.get('ldy', case['cout'])
    dy = rng.integers(-VMAX, VMAX + 1, (n,) + shape + (ldy,)).astype(np.float32)
    if 'up' in case:
        lo_shape = tuple(s // u for s, u in zip(shape, case['up']))
        lo = rng.integers(-VMAX, VMAX + 1, (n,) + lo_shape + (case['c_lo'],)).astype(np.float32)
        skip = rng.integers(-VMAX, VMAX + 1, (n,) + shape + (case['c_skip'],)).astype(np.float32)
        return np.concatenate([upsample(lo, case['up']), skip], axis=-1), lo, skip, dy
    x = rng.integers(-VMAX, VMAX + 1, (n,) + shape + (case['cin'],)).astype(np.float32)
    return x, None, x, dy


def int_dgrad_data(case):
    """(dy [n, *shape, cout], kernel (3^d, cin, cout)) float32 integers in [-VMAX, VMAX]"""
    rng = np.random.default_rng(case['seed'])
    dy = rng.integers(-VMAX, VMAX + 1, (case['n'],) + case['shape'] + (case['cout'],)).astype(np.float32)
    k = rng.integers(-VMAX, VMAX + 1, (3,) * case['nd'] + (case['cin'], case['cout'])).astype(np.float32)
    return dy, k


def twelve_bit(rng, shape, e):
    """+-M * 2^(e - 11) with M in [2^11, 2^12): 12 significant bits, half of them (odd M) exact ties at 11 bits"""
    m = rng.integers(2 ** 11, 2 ** 12, shape)
    s = rng.choice(np.array([-1.0, 1.0]), shape)
    return (s * m * 2.0 ** (e - 11)).astype(np.float32)


def sparse_dy(rng, n, shape, ldy, cols, e):
    """dy rows [n, *shape, ldy] that are zero except on a lattice of pixels 3 apart along every axis (one per 3^d window),
    each holding 3 of the columns `cols`, each column used at most 3 times"""
    dy = np.zeros((n,) + shape + (ldy,), np.float32)
    lattice = [(b,) + p for b in range(n) for p in np.ndindex(*[(s + 2) // 3 for s in shape])]
    rng.shuffle(lattice)
    use = {c: 0 for c in cols}
    for b, *p in lattice:
        free = [c for c in cols if use[c] < 3]
        if len(free) < 3:
            break
        for c in rng.choice(free, 3, replace=False):
            dy[(b,) + tuple(3 * q for q in p) + (int(c),)] = twelve_bit(rng, (), e)
            use[c] += 1
    return dy


def rounding_wgrad_data(case):
    """(x, dy rows) of a rounding case: 12-bit x on exponent 0, sparse 12-bit dy on exponent -3"""
    rng = np.random.default_rng(100 + case['seed'])
    ldy, off = case.get('ldy', case['cout']), case.get('off', 0)
    x = twelve_bit(rng, (case['n'],) + case['shape'] + (case['cin'],), 0)
    dy = sparse_dy(rng, case['n'], case['shape'], ldy, list(range(off, off + case['cout'])), -3)
    return x, dy


def rounding_dgrad_data(case):
    """(dy, kernel) of a rounding case: sparse 12-bit dy on exponent 1, 12-bit weights on exponent -2"""
    rng = np.random.default_rng(100 + case['seed'])
    dy = sparse_dy(rng, case['n'], case['shape'], case['cout'], list(range(case['cout'])), 1)
    k = twelve_bit(rng, (3,) * case['nd'] + (case['cin'], case['cout']), -2)
    return dy, k


# ------------------------------------------------------------------------------------------------ float64 oracles
def conv_grads64(x, dy, k, nd, kernel=None):
    """float64 autograd of y = conv(x, W, b, 'same') with upstream dy: (dW (k..., cin, cout), db, dx (like x)).  x, dy channels
    last; W the Keras kernel k, or zeros of extents `kernel` when only dW / db are wanted"""
    import torch
    import torch.nn.functional as F
    conv = F.conv2d if nd == 2 else F.conv3d
    cf = lambda a: torch.from_numpy(np.asarray(a, np.float64)).permute(0, nd + 1, *range(1, nd + 1))
    if k is None:
        k = np.zeros(tuple(kernel) + (x.shape[-1], dy.shape[-1]))
    xt = cf(x).requires_grad_(True)
    kt = torch.from_numpy(np.asarray(k, np.float64)).permute(nd + 1, nd, *range(nd)).contiguous().requires_grad_(True)
    bt = torch.zeros(dy.shape[-1], dtype=torch.float64, requires_grad=True)
    conv(xt, kt, bt, padding='same').backward(cf(dy))
    return (kt.grad.permute(*range(2, nd + 2), 1, 0).numpy(), bt.grad.numpy(), xt.grad.permute(0, *range(2, nd + 2), 1).numpy())


def rounding_bound(x, dy, k, nd, kernel=None):
    """largest partial sum of |rna(x)| |rna(dy)| (weight gradient) and |rna(dy)| |rna(W)| (input gradient) in units of the
    quantum of the smallest product, and whether every rounded operand is a multiple of its tensor's quantum -- both sums are
    exact in fp32 when the bound is below 2^24"""
    def quantum(a):
        nz = np.abs(a[a != 0]).astype(np.float64)
        if nz.size == 0:
            return 1.0, True
        m, e = np.frexp(nz)
        q = 2.0 ** (e.min() - 11)                       # an ulp of 11 significant bits at the smallest exponent
        return q, bool(np.all(np.mod(nz, q) == 0))
    xr, dyr = np.abs(rna(x)), np.abs(rna(dy))
    qx, okx = quantum(xr); qd, okd = quantum(dyr)
    if k is None:
        dw, _, _ = conv_grads64(xr / qx, dyr / qd, None, nd, kernel)
        return float(dw.max()), okx and okd
    kr = np.abs(rna(k))
    qk, okk = quantum(kr)
    _, _, dx = conv_grads64(np.zeros(dyr.shape[:-1] + (k.shape[-2],)), dyr / qd, kr / qk, nd)
    return float(dx.max()), okd and okk
