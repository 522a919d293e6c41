"""Exactly representable cases of sdb_class_head_backward (shared by test_gpu_train_classes.py and the bound check of
test_cpu_train_classes.py): small integer features, logit gradients and weights, so every partial sum is an integer below 2^24."""
import numpy as np

VMAX = 2

EXACT_CLASS_HEAD = [
    dict(id='c3_f128', npix=1000, cf=128, C=3, seed=11),
    dict(id='c5_f32_tail', npix=77, cf=32, C=5, seed=12),
    dict(id='c32_f128', npix=300, cf=128, C=32, seed=13),
]


def int_data(case):
    """(feat [npix, cf], dz [npix, C], W [cf, C], dfeat0 [npix, cf]: what an accumulating call adds to) float32 integers"""
    rng = np.random.default_rng(case['seed'])
    n, cf, C = case['npix'], case['cf'], case['C']
    f = lambda *s: rng.integers(-VMAX, VMAX + 1, s).astype(np.float32)
    return f(n, cf), f(n, C), f(cf, C), f(n, cf)


def max_partial(case, vmax=VMAX):
    """largest |partial sum|: C products of two values, plus the accumulated term"""
    return case['C'] * vmax * vmax + vmax
