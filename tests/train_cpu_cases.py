"""Exactly representable test cases of the training kernels (shared by test_gpu_train.py and the bounds checks of
test_cpu_train.py): small integer activations, gradients and weights, so that every partial sum is an integer below 2^24
and any summation order gives the float64 result bit for bit."""
import numpy as np

VMAX = 2                     # |x|, |dy|, |w| <= VMAX

EXACT_WGRAD = [
    dict(id='2d_stem_cin1', nd=2, n=2, shape=(21, 13), cin=1, cout=32, seed=1),
    dict(id='2d_stem_cin3', nd=2, n=2, shape=(17, 19), cin=3, cout=64, seed=2),
    dict(id='2d_c32_c64_edge', nd=2, n=3, shape=(21, 37), cin=32, cout=64, seed=3),
    dict(id='2d_c64_c32', nd=2, n=1, shape=(16, 16), cin=64, cout=32, seed=4),
    dict(id='3d_stem_cin1', nd=3, n=1, shape=(5, 11, 9), cin=1, cout=32, seed=5),
    dict(id='3d_c32_c32_edge', nd=3, n=2, shape=(5, 11, 9), cin=32, cout=32, seed=6),
]

EXACT_DECODER = [
    dict(id='2d_up22', nd=2, shape=(12, 20), up=(2, 2), c_lo=32, c_skip=32, cout=32, seed=7),
    dict(id='3d_up122', nd=3, shape=(3, 8, 12), up=(1, 2, 2), c_lo=32, c_skip=32, cout=32, seed=8),
    dict(id='3d_up222', nd=3, shape=(4, 8, 6), up=(2, 2, 2), c_lo=32, c_skip=32, cout=64, seed=9),
]


def int_data(case):
    """(x [n, *shape, cin], dy [n, *shape, cout], kernel (3^d, cin, cout)) float32 integers in [-VMAX, VMAX]"""
    rng = np.random.default_rng(case['seed'])
    n, nd = case['n'], case['nd']
    x = rng.integers(-VMAX, VMAX + 1, (n,) + case['shape'] + (case['cin'],)).astype(np.float32)
    dy = rng.integers(-VMAX, VMAX + 1, (n,) + case['shape'] + (case['cout'],)).astype(np.float32)
    k = rng.integers(-VMAX, VMAX + 1, (3,) * nd + (case['cin'], case['cout'])).astype(np.float32)
    return x, dy, k


def max_partial(case, vmax=VMAX):
    """largest |partial sum| any kernel can form on the case: the weight gradient sums over every pixel of the batch, the
    input gradient over taps x Cout, the up-sampling backward over one block, the bias gradient over every pixel"""
    nd = case['nd']
    npix = case.get('n', 2) * int(np.prod(case['shape']))
    cout = case['cout']
    cin = case.get('cin', case.get('c_lo', 0) + case.get('c_skip', 0))
    up = int(np.prod(case.get('up', (1,))))
    wgrad = npix * vmax * vmax
    dgrad = 3 ** nd * cout * vmax * vmax
    upsum = up * dgrad + vmax          # a block sum of input gradients, plus the max-pool contribution
    return max(wgrad, dgrad, upsum, cin)
