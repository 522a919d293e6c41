"""Training cases outside the default architecture family (shared by test_gpu_train_any.py and the checks of
test_cpu_train_any.py): exactly representable layer cases of sdb_conv_wgrad_any_nd / sdb_conv_dgrad_any_nd, and a float32
numpy restatement of the activation derivatives of sdb_act_backward with the error bound the device kernel is held to."""
import numpy as np

VMAX = 2                     # |x|, |dy|, |w| <= VMAX


def _case(id, k, shape, c_skip, cout, c_lo=0, up=None, n=2, seed=0):
    nd = len(k)
    return dict(id=id, nd=nd, k=tuple(k), n=n, shape=tuple(shape), c_skip=c_skip, c_lo=c_lo, up=tuple(up or (1,) * nd), cout=cout,
                seed=seed)


# kernel extents 1, 2, 4, 5, 7 in 2-D and (1,3,3), (3,1,5) in 3-D; input widths 1, 3, 16, 48; decoder inputs
# [upsample(x_lo), skip] with up-sampling (2,2) and (1,2,2).  Sizes are not multiples of the 16 x 16 output tile.
EXACT_ANY = [
    _case('2d_k11_ci3_co16', (1, 1), (13, 17), 3, 16, seed=1),
    _case('2d_k22_ci1_co32', (2, 2), (15, 18), 1, 32, seed=2),
    _case('2d_k44_ci16_co16', (4, 4), (14, 19), 16, 16, seed=3),
    _case('2d_k55_ci48_co8', (5, 5), (12, 21), 48, 8, seed=4),
    _case('2d_k77_ci3_co40', (7, 7), (17, 23), 3, 40, seed=5),
    _case('2d_k55_ci1_co3', (5, 5), (9, 11), 1, 3, n=3, seed=6),
    _case('3d_k133_ci16_co24', (1, 3, 3), (5, 9, 11), 16, 24, seed=7),
    _case('3d_k315_ci48_co16', (3, 1, 5), (4, 10, 9), 48, 16, seed=8),
    _case('2d_k55_up22_lo16_sk16_co16', (5, 5), (12, 20), 16, 16, c_lo=16, up=(2, 2), seed=9),
    _case('2d_k22_up22_lo3_sk1_co48', (2, 2), (10, 14), 1, 48, c_lo=3, up=(2, 2), seed=10),
    _case('3d_k133_up122_lo16_sk16_co16', (1, 3, 3), (3, 8, 12), 16, 16, c_lo=16, up=(1, 2, 2), seed=11),
    _case('3d_k315_up122_lo48_sk3_co8', (3, 1, 5), (4, 6, 10), 3, 8, c_lo=48, up=(1, 2, 2), seed=12),
]


def int_data(case):
    """(skip [n, *shape, c_skip], lo [n, *shape / up, c_lo] or None, dy [n, *shape, cout], kernel (*k, cin, cout)) float32
    integers in [-VMAX, VMAX]"""
    rng = np.random.default_rng(case['seed'])
    r = lambda *s: rng.integers(-VMAX, VMAX + 1, s).astype(np.float32)
    n, shape = case['n'], case['shape']
    skip = r(n, *shape, case['c_skip'])
    lo = r(n, *(s // u for s, u in zip(shape, case['up'])), case['c_lo']) if case['c_lo'] else None
    dy = r(n, *shape, case['cout'])
    k = r(*case['k'], case['c_lo'] + case['c_skip'], case['cout'])
    return skip, lo, dy, k


def max_partial(case, vmax=VMAX):
    """largest |partial sum| a kernel forms on the case: the weight gradient sums x * dy over every pixel of the batch (the
    bias row sums dy), the input gradient sums over taps x cout, the up-sampling backward over one block of those"""
    npix = case['n'] * int(np.prod(case['shape']))
    wgrad = npix * vmax * vmax
    dgrad = int(np.prod(case['k'])) * case['cout'] * vmax * vmax
    upsum = int(np.prod(case['up'])) * dgrad
    return max(wgrad, dgrad, upsum)


# ------------------------------------------------------------------------------------------------ activation derivatives
ACTS_SMOOTH = ('elu', 'selu', 'tanh', 'sigmoid', 'softplus', 'softsign', 'exponential', 'swish', 'gelu')


def act_grad_np(name, z):
    """act'(z) in float32 with the formulas of act_grad (csrc/unet_any.cu)"""
    f = np.float32
    z = np.asarray(z, np.float32)
    with np.errstate(over='ignore', under='ignore'):
        if name == 'linear':
            return np.ones_like(z)
        if name == 'relu':
            return (z > 0).astype(np.float32)
        if name == 'elu':
            return np.where(z > 0, f(1), np.exp(z)).astype(np.float32)
        if name == 'selu':
            return np.where(z > 0, f(1.05070098735548049342), f(1.75809934084737685994) * np.exp(z)).astype(np.float32)
        if name == 'tanh':
            u = np.exp(f(-2) * np.abs(z)); q = f(1) + u
            return f(4) * u / (q * q)
        if name == 'sigmoid':
            u = np.exp(-np.abs(z)); q = f(1) + u
            return u / (q * q)
        if name == 'softplus':
            u = np.exp(-np.abs(z))
            return np.where(z >= 0, f(1), u) / (f(1) + u)
        if name == 'softsign':
            q = f(1) + np.abs(z)
            return f(1) / (q * q)
        if name == 'exponential':
            return np.exp(z)
        if name == 'swish':
            u = np.exp(-np.abs(z)); r = f(1) / (f(1) + u)
            s = np.where(z >= 0, r, u * r); sc = np.where(z >= 0, u * r, r)
            return s * (f(1) + z * sc)
        if name == 'gelu':
            from scipy.special import erfc
            return (f(0.5) * erfc(z * f(-0.707106781186547524)).astype(np.float32)
                    + z * f(0.398942280401432678) * np.exp(f(-0.5) * z * z)).astype(np.float32)
    raise KeyError(name)


def act_grad64(name, z):
    """float64 autograd of tests/any_config_oracle.act64 at the points z"""
    import torch
    from any_config_oracle import act64
    t = torch.from_numpy(np.asarray(z, np.float64)).requires_grad_(True)
    act64(name, t).sum().backward()
    return t.grad.numpy()


def act_grad_exact64(name, z):
    """act'(z) in float64 closed forms that keep their relative accuracy in both tails.  Autograd of act64 does not there:
    torch differentiates tanh as 1 - y^2 and expm1 as y + 1, which cancel to 0 once y rounds to +-1 (|z| > 19 for tanh,
    z < -37 for elu / selu); test_cpu_train_any.py checks that the two agree wherever those have not cancelled."""
    from scipy.special import erfc, expit
    from any_config_oracle import SELU_ALPHA, SELU_SCALE
    z = np.asarray(z, np.float64)
    with np.errstate(over='ignore', under='ignore'):
        if name == 'linear':
            return np.ones_like(z)
        if name == 'relu':
            return (z > 0).astype(np.float64)
        if name == 'elu':
            return np.where(z > 0, 1.0, np.exp(np.minimum(z, 0)))
        if name == 'selu':
            return SELU_SCALE * np.where(z > 0, 1.0, SELU_ALPHA * np.exp(np.minimum(z, 0)))
        if name == 'tanh':
            return 1.0 / np.cosh(z) ** 2
        if name in ('sigmoid', 'softplus', 'swish'):
            s, sc = expit(z), expit(-z)
            return {'sigmoid': s * sc, 'softplus': s, 'swish': s + z * s * sc}[name]
        if name == 'softsign':
            return 1.0 / (1.0 + np.abs(z)) ** 2
        if name == 'exponential':
            return np.exp(z)
        if name == 'gelu':
            return 0.5 * erfc(-z / np.sqrt(2)) + z * np.exp(-0.5 * z * z) / np.sqrt(2 * np.pi)
    raise KeyError(name)


def _magnitude64(name, z):
    """sum of the magnitudes of the terms the float32 formula adds: |act'| except for swish s + |z s (1 - s)| and gelu
    Phi(z) + |z phi(z)|, whose two terms cancel near the derivative's zero"""
    from scipy.special import erfc, expit
    z = np.asarray(z, np.float64)
    with np.errstate(over='ignore', under='ignore'):
        if name == 'swish':
            return expit(z) + np.abs(z * expit(z) * expit(-z))
        if name == 'gelu':
            return 0.5 * erfc(-z / np.sqrt(2)) + np.abs(z) * np.exp(-0.5 * z * z) / np.sqrt(2 * np.pi)
        return np.abs(act_grad_exact64(name, z))


def act_grad_bound(name, z):
    """(act'(z) in float64, the bound on |float32 act'(z) - act'(z)|): 8 * 2^-23 * (magnitude of the summed terms) + the
    change of act' under one relative rounding (2^-23) of z + 2^-146 (below float32's normal range)"""
    z64 = np.asarray(z, np.float32).astype(np.float64)
    want = act_grad_exact64(name, z64)
    sens = np.maximum(np.abs(act_grad_exact64(name, z64 * (1 + 2.0 ** -23)) - want),
                      np.abs(act_grad_exact64(name, z64 * (1 - 2.0 ** -23)) - want))
    return want, 8 * 2.0 ** -23 * _magnitude64(name, z64) + sens + 2.0 ** -146


def act_points():
    """a sweep of [-30, 30], the branch points of elu / selu (0) and softplus (+-13.9423847, log(FLT_EPSILON) + 2), tiny
    magnitudes and the zeros of the swish and gelu derivatives"""
    x = np.linspace(-30, 30, 6001, dtype=np.float64)
    special = [-1e-6, -1e-30, 0.0, 1e-30, 1e-6, -13.9423847, 13.9423847, -14.5, 14.5, -1.2784645, -0.7517916, 60.0, -60.0]
    ex = np.array([np.nextafter(np.float32(v), np.float32(s)) for v in (-13.9423847, 13.9423847, 0.0) for s in (-np.inf, np.inf)])
    return np.concatenate([x.astype(np.float32), np.asarray(special, np.float32), ex.astype(np.float32)])
