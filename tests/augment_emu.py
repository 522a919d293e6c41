"""numpy restatement of the device augmenter (stardist_b200.models.Augmenter, csrc/augment.cu), written from its description:

- normal_emu: numpy's legacy np.random.normal(0, 1, n) on a RandomState state -- MT19937 twists, tempering, two words per
  double, the polar method with four words per attempt, the Gaussian cache -- vectorised over attempts, with the values and
  the final state (key, pos, has_gauss, gauss).  `log` is the C library's (math.log), which legacy_gauss calls.
- aug_emu: the notebooks' augmentation of one item, in their draw order, on the global np.random (its noise is numpy's own
  np.random.normal): the host-path callable the device augmenter is compared with.
- intensity: the float32 roundings of x * s + t and of the noise add, for the robustness check."""
import math
import numpy as np

N, M_ = 624, 397
UPPER, LOWER, MATRIX_A = np.uint32(0x80000000), np.uint32(0x7fffffff), np.uint32(0x9908b0df)


def twist(key):
    """one MT19937 generation (mt19937_gen) of a uint32 [624] key -> the new key; three dependency levels of <= 227 words"""
    old, new = key, np.empty_like(key)

    def mix(a, b, c):
        y = (a & UPPER) | (b & LOWER)
        return c ^ (y >> np.uint32(1)) ^ np.where(y & np.uint32(1), MATRIX_A, np.uint32(0))
    k = N - M_
    new[:k] = mix(old[:k], old[1:k + 1], old[M_:])
    new[k:2 * k] = mix(old[k:2 * k], old[k + 1:2 * k + 1], new[:k])
    new[2 * k:N - 1] = mix(old[2 * k:N - 1], old[2 * k + 1:N], new[k:N - 1 - k])
    new[N - 1:] = mix(old[N - 1:], new[:1], new[M_ - 1:M_])
    return new


def temper(y):
    y = y ^ (y >> np.uint32(11))
    y = y ^ ((y << np.uint32(7)) & np.uint32(0x9d2c5680))
    y = y ^ ((y << np.uint32(15)) & np.uint32(0xefc60000))
    return y ^ (y >> np.uint32(18))


def normal_emu(state, n):
    """(values float64 [n], state after) of np.random.normal(0, 1, n) from a legacy get_state() tuple"""
    name, key, pos, has_gauss, gauss = state
    key = np.asarray(key, np.uint32)
    pos, has_gauss = int(pos), int(bool(has_gauss))
    if n == 0:
        return np.zeros(0), (name, key.copy(), pos, has_gauss, float(gauss))
    out = [np.array([gauss])] if has_gauss else []
    M = (n - has_gauss + 1) // 2
    if M == 0:
        return np.array([gauss]), (name, key.copy(), pos, 0, 0.0)
    A = int(math.ceil((M + 6 * math.sqrt(M) + 32) / (math.pi / 4)))
    while True:
        blocks = [key]
        while len(blocks) * N < pos + 4 * A:
            blocks.append(twist(blocks[-1]))
        words = temper(np.concatenate(blocks)[pos:pos + 4 * A]).reshape(A, 4).astype(np.float64)
        u = ((np.floor(words[:, 0::2] / 32) * 67108864.0) + np.floor(words[:, 1::2] / 64)) / 9007199254740992.0
        x1, x2 = 2.0 * u[:, 0] - 1.0, 2.0 * u[:, 1] - 1.0
        r2 = x1 * x1 + x2 * x2
        acc = np.flatnonzero(~((r2 >= 1.0) | (r2 == 0.0)))
        if len(acc) >= M:
            break
        A *= 2
    a = acc[:M]
    r = r2[a]
    f = np.sqrt(-2.0 * np.array([math.log(v) for v in r]) / r)
    pairs = np.stack([f * x2[a], f * x1[a]], axis=1).ravel()
    vals = np.concatenate(out + [pairs])
    cached = len(vals) > n
    c = pos + 4 * (int(a[-1]) + 1)
    t = (c - 1) // N
    new = (name, blocks[t].copy(), c - t * N, int(cached), float(vals[n]) if cached else 0.0)
    return vals[:n], new


def fliprot(x, y, axis):
    """random_fliprot of the 3-D notebook (the 2-D notebook's for axis = all axes)"""
    perm = tuple(np.random.permutation(axis))
    tr = np.arange(y.ndim)
    for a, p in zip(axis, perm):
        tr[a] = p
    tr = tuple(int(v) for v in tr)
    x = x.transpose(tr + tuple(range(y.ndim, x.ndim)))
    y = y.transpose(tr)
    for ax in axis:
        if np.random.rand() > 0.5:
            x, y = np.flip(x, axis=ax), np.flip(y, axis=ax)
    return x, y


def aug_emu(x, y, axis=None, scale=(0.6, 2), shift=(-0.2, 0.2), noise=0.02):
    """the notebooks' augmenter (x float32 patch, y label patch) on the global np.random"""
    axis = tuple(range(y.ndim)) if axis is None else tuple(axis)
    x, y = fliprot(x, y, axis)
    x = x * np.random.uniform(*scale) + np.random.uniform(*shift)
    if noise is not None:
        sig = noise * np.random.uniform(0, 1)
        x = x + sig * np.random.normal(0, 1, x.shape)
    return x, y


def intensity(x, s, t):
    """float32(float32(x * float32(s)) + float32(t)): numpy's float32 array with Python floats"""
    x = np.asarray(x, np.float32)
    return (x * np.float32(s)).astype(np.float32) + np.float32(t)


def noise_add(x32, sig, n):
    """float32(float64(x) + sig * n)"""
    return (x32.astype(np.float64) + sig * np.asarray(n, np.float64)).astype(np.float32)
