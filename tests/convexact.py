"""Exactly representable operands for the tensor-core convolution kernels (csrc/unet_tc.cu) and float64 restatements of
what those kernels compute.

k_conv_wg takes pre-split operands: activation planes (hi, lo) in fp16, weight planes (W_hi, W_lo) in fp16 and a power of
two w_scale.  Its documented arithmetic is

    y = (hi.W_hi + lo.W_hi + hi.W_lo) * 2^-s + b      (the lo.W_lo term is dropped), then ReLU, then a hi/lo fp16 split.

Built here from small integers times powers of two, every product and every partial sum of that expression is an integer
multiple of one quantum and stays below 2^22 quanta (worst_case_bits proves it for each accumulator).  fp32 then holds
every partial sum exactly, so the kernel's result has a single correct value whatever the summation order, the MMA's
internal alignment, the truncating accumulator adder or sdb_tc_set_split_acc -- and the tests compare it with the float64
references below by value equality, element by element, in both output planes.  Only `prob` goes through expf and a
division; it is compared within 4 float32 ulps.

The case tables at the end are shared by tests/test_cpu_conv_exact.py (bounds, mutants, instance coverage) and
tests/test_gpu_conv_exact.py (the kernels).  Pure numpy / torch on the CPU."""
import math
import re
import itertools
import numpy as np

# ------------------------------------------------------------------------------------------------ recipes
# a: |hi| and |W_hi| <= a (integers); the lo planes are integers in [-a, a] times lo_q; bias = integers in [-b_int, b_int]
# times b_q.  The fused features -> heads path multiplies the feature quantum by the head-weight quantum, so its operands
# are smaller: head weights are integers in [-hw_int, hw_int] times hw_q, head biases integers times hb_q.
PARAMS = {
    "conv": dict(a=2, lo_q=2.0 ** -6, w_scale=2.0 ** 4, b_int=64, b_q=2.0 ** -10),
    "heads": dict(a=2, lo_q=2.0 ** -6, w_scale=2.0 ** 4, b_int=64, b_q=2.0 ** -10),
    "fused": dict(a=1, lo_q=2.0 ** -5, w_scale=2.0 ** 4, b_int=64, b_q=2.0 ** -9, hw_int=1, hw_q=2.0 ** -3, hb_int=64,
                  hb_q=2.0 ** -12),
    # stem: fp32 input and weights (no split); x = integers * x_q, W = integers * w_q
    "stem": dict(x_int=8, x_q=2.0 ** -3, w_int=8, w_q=2.0 ** -4, b_int=64, b_q=2.0 ** -7),
}


def worst_case_bits(p, K, n_head_in=128):
    """log2 of the largest |partial sum| / quantum any accumulator can reach with recipe `p` over K = taps * Cin terms.

    main:       hi.W_hi alone (split_acc = 1), quantum 1
    correction: lo.W_hi + hi.W_lo (split_acc = 1), quantum lo_q
    combined:   all three products in one accumulator (split_acc = 0, and the epilogue's acc + cor), quantum lo_q
    output:     combined * 2^-s + b, quantum min(lo_q / w_scale, b_q) -- below 2^22 the hi/lo fp16 split is exact too
    head:       (fused) sum over n_head_in features of |f| * |w_head| + |b_head|, quantum = feature quantum * hw_q"""
    a, q = p["a"], p["lo_q"]
    hh = K * a * a                                   # in units of 1
    cor = 2 * K * a * (a * q)                        # in units of 1
    out = {"main": hh / 1.0, "correction": cor / q, "combined": (hh + cor) / q}
    y_max = (hh + cor) / p["w_scale"] + p["b_int"] * p["b_q"]
    y_q = min(q / p["w_scale"], p["b_q"])
    out["output"] = y_max / y_q
    if "hw_q" in p:
        f_max = y_max                                # ReLU does not enlarge it
        h_q = y_q * p["hw_q"]
        assert (p["hb_q"] / h_q).is_integer(), "the head bias quantum must be a multiple of the head-sum quantum"
        out["head"] = (n_head_in * f_max * p["hw_int"] * p["hw_q"] + p["hb_int"] * p["hb_q"]) / h_q
    return {k: math.log2(v) for k, v in out.items()}


def stem_worst_case_bits(p, cin):
    K = 9 * cin
    q = min(p["x_q"] * p["w_q"], p["b_q"])
    return math.log2((K * p["x_int"] * p["x_q"] * p["w_int"] * p["w_q"] + p["b_int"] * p["b_q"]) / q)


# ------------------------------------------------------------------------------------------------ generators
def _ints(rng, shape, r):
    return rng.integers(-r, r + 1, size=shape).astype(np.float64)


def _f16(a):
    h = a.astype(np.float16)
    assert np.array_equal(h.astype(np.float64), a), "operand not exactly representable in fp16"
    return h


def gen_conv(case):
    """split activation planes of both sources and split weights for a 3x3 / 3x3x3 (or fused features) case.
    2-D: activations [n, h, w, c]; 3-D: one volume [d, h, w, c].  Weights [taps][cout][cin] (tap = dz*9 + dy*3 + dx)."""
    fam = case["family"]
    p = PARAMS["fused" if fam == "fused" else "conv"]
    rng = np.random.default_rng(case["seed"])
    lead = (case["d"],) if fam == "conv3d" else (case["n"],)
    sp = lead + (case["h"], case["w"])
    cin = case["c0"] + case["c1"]
    cout = 128 if fam == "fused" else case["cout"]
    taps = 27 if fam == "conv3d" else 9
    a, q = p["a"], p["lo_q"]
    D = dict(
        x_hi=_f16(_ints(rng, sp + (cin,), a)), x_lo=_f16(_ints(rng, sp + (cin,), a) * q),
        w_hi=_f16(_ints(rng, (taps, cout, cin), a)), w_lo=_f16(_ints(rng, (taps, cout, cin), a) * q),
        bias=(_ints(rng, (cout,), p["b_int"]) * p["b_q"]).astype(np.float32), w_scale=p["w_scale"])
    if fam == "fused":
        R = case["R"]
        hw = np.zeros((128, 36)); hb = np.zeros(36)
        hw[:, :R] = _ints(rng, (128, R), p["hw_int"]) * p["hw_q"]
        hw[:, 32] = _ints(rng, (128,), p["hw_int"]) * p["hw_q"]
        hb[:R] = _ints(rng, (R,), p["hb_int"]) * p["hb_q"]
        hb[32] = _ints(rng, (1,), p["hb_int"])[0] * p["hb_q"]
        D["heads_w"], D["heads_b"] = hw.astype(np.float32), hb.astype(np.float32)
    return D


def gen_heads(case):
    """1x1 heads: features [n, h, w, cfeat] split planes, head weights [np][cfeat] split planes (row 0 prob, rows 1..R
    dist, rows > R zero as the executors pad them), bias [np]"""
    p = PARAMS["heads"]
    rng = np.random.default_rng(case["seed"])
    cf, npd, R = case["cfeat"], case["np"], case["R"]
    sp = (case["n"], case["h"], case["w"])
    a, q = p["a"], p["lo_q"]
    wh = np.zeros((npd, cf)); wl = np.zeros((npd, cf)); b = np.zeros(npd)
    wh[:R + 1] = _ints(rng, (R + 1, cf), a); wl[:R + 1] = _ints(rng, (R + 1, cf), a) * q
    b[:R + 1] = _ints(rng, (R + 1,), p["b_int"]) * p["b_q"]
    return dict(x_hi=_f16(_ints(rng, sp + (cf,), a)), x_lo=_f16(_ints(rng, sp + (cf,), a) * q),
                w_hi=_f16(wh), w_lo=_f16(wl), bias=b.astype(np.float32), w_scale=p["w_scale"])


def gen_stem(case):
    p = PARAMS["stem"]
    rng = np.random.default_rng(case["seed"])
    cin, cout = case["cin"], case["cout"]
    return dict(x=(_ints(rng, (case["n"], case["h"], case["w"], cin), p["x_int"]) * p["x_q"]).astype(np.float32),
                w=(_ints(rng, (3, 3, cin, cout), p["w_int"]) * p["w_q"]).astype(np.float32),
                bias=(_ints(rng, (cout,), p["b_int"]) * p["b_q"]).astype(np.float32))


# ------------------------------------------------------------------------------------------------ float64 references
def _taps(nd):
    return [(dz, dy, dx) for dz in (range(3) if nd == 3 else (1,)) for dy in range(3) for dx in range(3)]


def conv_taps(x, W, nd, mutants=(), order=1, dtype=np.float64):
    """'same' 3x3 (nd 2: x [n, h, w, c]) or 3x3x3 (nd 3: x [d, h, w, c], one volume) convolution with W [taps][cout][cin],
    as a sum over taps of shifted-input x W^T products, taps visited in `order` (1 forwards, -1 backwards).
    mutants: 'swap_dydx' reads tap (dy, dx) at (dx, dy); 'dz_wrong' reads the plane z-1 for the dz = +1 taps."""
    x = np.asarray(x, dtype)
    x5 = x[:, None] if nd == 2 else x[None]                      # [B, D, H, W, C]
    B, Dd, H, Wd, _ = x5.shape
    xp = np.pad(x5, ((0, 0), (1, 1), (1, 1), (1, 1), (0, 0)))
    out = np.zeros((B, Dd, H, Wd, W.shape[1]), dtype)
    taps = list(enumerate(_taps(nd)))[::order]
    for t, (dz, dy, dx) in taps:
        if "swap_dydx" in mutants: dy, dx = dx, dy
        if "dz_wrong" in mutants and dz == 2: dz = 0
        out += xp[:, dz:dz + Dd, dy:dy + H, dx:dx + Wd, :] @ np.asarray(W[t], dtype).T
    return out[:, 0] if nd == 2 else out[0]


def split16(y):
    """the epilogue's output split: hi = fp16(v), lo = fp16(v - hi), v the fp32 value"""
    y32 = np.asarray(y, np.float32)
    hi = y32.astype(np.float16)
    lo = (y32 - hi.astype(np.float32)).astype(np.float16)
    return hi, lo


def upsample(y, up, mutants=()):
    """nearest up-sampling written by the producing epilogue: 2x2 over (h, w) (up 1, 2-D) or 2x2x2 over (d, h, w) (up 2, 3-D).
    mutant 'up_replica': the odd replicas along the first up-sampled axis take the next source row / plane."""
    if not up:
        return y
    axes = (1, 2) if up == 1 else (0, 1, 2)
    out = y
    for ax in axes:
        out = np.repeat(out, 2, axis=ax)
    if "up_replica" in mutants:
        a0 = axes[0]
        n = y.shape[a0]
        nxt = np.take(y, np.minimum(np.arange(n) + 1, n - 1), axis=a0)
        for ax in axes[1:]:
            nxt = np.repeat(nxt, 2, axis=ax)
        sl = [slice(None)] * out.ndim; sl[a0] = slice(1, None, 2)
        out[tuple(sl)] = nxt
    return out


def _sources(D, c0, kc, mutants):
    xh = D["x_hi"].astype(np.float64); xl = D["x_lo"].astype(np.float64)
    if "swap_src" in mutants:                                   # source 1's channels first, source 0's after
        xh = np.concatenate([xh[..., c0:], xh[..., :c0]], -1); xl = np.concatenate([xl[..., c0:], xl[..., :c0]], -1)
    if "shift_cblock" in mutants:                               # every K block reads the next block's channels
        xh = np.roll(xh, -kc, axis=-1); xl = np.roll(xl, -kc, axis=-1)
    return xh, xl


def conv_pre(D, nd, c0, kc=32, mutants=(), order=1, dtype=np.float64):
    """(hi.W_hi + lo.W_hi + hi.W_lo) of the split operands, before scale and bias; `lo_whi`, `hi_wlo` drop a product,
    `lo_wlo` adds the dropped one"""
    xh, xl = _sources(D, c0, kc, mutants)
    wh = D["w_hi"].astype(np.float64); wl = D["w_lo"].astype(np.float64)
    y = conv_taps(xh, wh, nd, mutants, order, dtype)
    if "lo_whi" not in mutants: y = y + conv_taps(xl, wh, nd, mutants, order, dtype)
    if "hi_wlo" not in mutants: y = y + conv_taps(xh, wl, nd, mutants, order, dtype)
    if "lo_wlo" in mutants: y = y + conv_taps(xl, wl, nd, mutants, order, dtype)
    return y


def _bias_act(pre, D, relu, mutants, dtype=np.float64):
    b = np.asarray(D["bias"], dtype)
    if "shift_bias" in mutants: b = np.roll(b, 1)
    y = pre * dtype(1.0 / D["w_scale"])
    if relu and "relu_before_bias" in mutants:
        return np.maximum(y, 0) + b
    y = y + b
    return np.maximum(y, 0) if relu else y


def conv_ref(case, D, mutants=()):
    """float64 output of sdb_conv3x3_tc / sdb_conv3x3x3_tc (up-sampled if the case asks), before the hi/lo split"""
    nd = 3 if case["family"] == "conv3d" else 2
    kc = instance(case)[1]
    y = _bias_act(conv_pre(D, nd, case["c0"], kc, mutants), D, case["relu"], mutants)
    return upsample(y, case["up"], mutants)


def sigmoid64(v):
    v = np.asarray(v, np.float64)
    return 1.0 / (1.0 + np.exp(-v))


def heads_ref(D, R, mutants=()):
    """(prob, dist) of sdb_heads_tc in float64: logits = (hi.W_hi + lo.W_hi + hi.W_lo) / w_scale + b over the padded rows;
    prob = sigmoid(row 0), dist = rows 1..R.  mutant 'dist_row': dist takes rows 2..R+1."""
    xh = D["x_hi"].astype(np.float64); xl = D["x_lo"].astype(np.float64)
    wh = D["w_hi"].astype(np.float64); wl = D["w_lo"].astype(np.float64)
    z = xh @ wh.T
    if "lo_whi" not in mutants: z = z + xl @ wh.T
    if "hi_wlo" not in mutants: z = z + xh @ wl.T
    if "lo_wlo" in mutants: z = z + xl @ wl.T
    b = D["bias"].astype(np.float64)
    if "shift_bias" in mutants: b = np.roll(b, 1)
    z = z / D["w_scale"] + b
    r0 = 2 if "dist_row" in mutants else 1
    zp = np.concatenate([z, np.zeros(z.shape[:-1] + (2,))], -1)
    return sigmoid64(z[..., 0]), zp[..., r0:r0 + R]


def fused_ref(case, D, mutants=()):
    """(prob logit, prob, dist) of sdb_conv3x3_heads_tc in float64: features f = act(conv(...) / w_scale + b) (never stored),
    then heads on the [128][36] weights: dist_r = f . w[:, r] + b[r] (r < R), prob = sigmoid(f . w[:, 32] + b[32]).
    mutant 'dist_row': dist_r uses column r + 1."""
    f = _bias_act(conv_pre(D, 2, case["c0"], 32, mutants), D, case["relu"], mutants)
    hw = D["heads_w"].astype(np.float64); hb = D["heads_b"].astype(np.float64)
    o = f @ hw + hb
    r0 = 1 if "dist_row" in mutants else 0
    logit = o[..., 32]
    return logit, sigmoid64(logit), o[..., r0:r0 + case["R"]]


def stem_ref(D, relu, mutants=()):
    """sdb_stem_split in float64: 3x3 'same' conv of the fp32 input with the Keras kernel (3, 3, cin, cout) + bias, ReLU"""
    W = np.asarray(D["w"], np.float64).reshape(9, D["w"].shape[2], D["w"].shape[3]).transpose(0, 2, 1)
    y = conv_taps(D["x"], W, 2, mutants)
    return _bias_act(y, dict(bias=D["bias"], w_scale=1.0), relu, mutants)


def maxpool_split_ref(hi, lo, pool):
    """max of the fp32 values hi + lo over (pz, py, px) windows of [d, h, w, c] planes, re-split (k_maxpool*_split)"""
    v = hi.astype(np.float32) + lo.astype(np.float32)
    d, h, w, c = v.shape
    pz, py, px = pool
    m = v.reshape(d // pz, pz, h // py, py, w // px, px, c).max(axis=(1, 3, 5))
    return split16(m)


def weights_split_ref(w, scale):
    """sdb_split_weights(_3d): Keras (k..., cin, cout) fp32 kernel times scale -> [tap][cout][cin] fp16 hi / lo"""
    cin, cout = w.shape[-2], w.shape[-1]
    v = (np.asarray(w, np.float32) * np.float32(scale)).reshape(-1, cin, cout).transpose(0, 2, 1)
    return split16(v)


# ------------------------------------------------------------------------------------------------ kernel instances
def _k64(c0, c1):
    return c0 % 64 == 0 and c1 % 64 == 0


def instance(case):
    """(N, KC, FUSE) of the k_conv_wg instantiation a case launches: a Python copy of pick_kc, nt = min(cout, 128) and the
    np choice in unet_tc.cu"""
    fam = case["family"]
    if fam in ("conv2d", "conv3d"):
        kc = 32 if (case["variant"] == 4 or not _k64(case["c0"], case["c1"])) else 64
        return (min(case["cout"], 128), kc, False)
    if fam == "heads":
        return (case["np"], 64, False)
    return (128, 32, True)


def instances_in_source(path):
    """every (N, KC, FUSE) that unet_tc.cu instantiates (SDB_WG(N, KC) and launch_wg<N, KC[, true]>)"""
    src = open(path).read()
    out = {(int(n), int(k), False) for n, k in re.findall(r"SDB_WG\((\d+),\s*(\d+)\)", src)}
    for n, k, f in re.findall(r"launch_wg<(\d+),\s*(\d+)(?:,\s*(true))?>\(", src):
        out.add((int(n), int(k), f == "true"))
    return out


ALL_INSTANCES = {(n, kc, False) for n in (32, 64, 128) for kc in (32, 64)} | {(n, 64, False) for n in (48, 80, 112, 144)} \
    | {(128, 32, True)}

VARIANTS = (0, 1, 3, 4)


# ------------------------------------------------------------------------------------------------ case tables
# A reduced cross product: every parameter value appears, and variants / split_acc rotate so that each of the 11
# instances runs under split_acc 0 and 1 and each family under variants 0, 1, 3 and 4 (test_cpu_conv_exact.py checks it).
MIXES_2D = [(0, 32), (0, 64), (0, 96), (32, 32), (32, 64), (64, 32), (64, 64), (0, 256)]
EDGES = [(1, 1), (1, 17), (7, 15), (8, 16), (9, 17), (3, 130)]


def _conv2d_cases():
    cases = []
    for i, ((c0, c1), cout) in enumerate(itertools.product(MIXES_2D, (32, 64, 128, 256))):
        h, w = EDGES[i % len(EDGES)]
        cases.append(dict(family="conv2d", c0=c0, c1=c1, cout=cout, n=(1, 3)[(i // 3) % 2], h=h, w=w, relu=(i // 2) % 2,
                          up=1 if i % 5 == 4 else 0, variant=VARIANTS[i % 4], split=(i // 4) % 2, seed=1000 + i))
    return cases


def _conv3d_cases():
    cases = []
    for i, ((c0, c1), cout) in enumerate(itertools.product(MIXES_2D, (32, 64, 128))):
        h, w = EDGES[(i + 2) % len(EDGES)]
        cases.append(dict(family="conv3d", c0=c0, c1=c1, cout=cout, d=(1, 2, 3)[i % 3], h=h, w=w, relu=(i // 2) % 2,
                          up=2 if i % 4 == 1 else 0, variant=VARIANTS[(i // 3) % 4], split=(i // 2) % 2, seed=2000 + i))
    return cases


def _heads_cases():
    cases = []
    small_R = {48: 33, 80: 61, 112: 97, 144: 131}            # R < np - 1 and not a multiple of 8
    # (n, h, w): the 3-D executor's (1, d*h, w) view of a 3 x 5 x 23 volume, and 2-D images with ragged tiles
    shapes = [(1, 3 * 5, 23), (2, 9, 17), (1, 1, 130), (2, 8, 16)]
    for i, (npd, r, cf) in enumerate(itertools.product((48, 80, 112, 144), (0, 1), (64, 128, 256))):
        n, h, w = shapes[i % len(shapes)]
        cases.append(dict(family="heads", np=npd, R=npd - 1 if r == 0 else small_R[npd], cfeat=cf, n=n, h=h, w=w,
                          variant=VARIANTS[(i // 3) % 4], split=i % 2, seed=3000 + i))
    return cases


def _fused_cases():
    cases = []
    for i, R in enumerate((1, 2, 7, 8, 9, 15, 16, 17, 31, 32)):
        for j, (c0, c1) in enumerate(((0, 32), (0, 64), (32, 32))):
            k = 3 * i + j
            h, w = EDGES[k % len(EDGES)]
            cases.append(dict(family="fused", R=R, c0=c0, c1=c1, n=(1, 2)[k % 2], h=h, w=w, relu=(k // 2) % 2,
                              variant=VARIANTS[k % 4], split=(k // 4) % 2, seed=4000 + k))
    return cases


# Persistent-grid cases: more 8 x 16-pixel tiles than the H100's 132 SMs, so each CTA sweeps several tiles and the producer
# runs ahead across tile boundaries (ring parity, accumulator restart, epilogue overlap).  Variant 1 launches one CTA per tile.
PERSISTENT = [
    dict(family="conv2d", c0=0, c1=64, cout=256, n=3, h=64, w=136, relu=1, up=0, variant=0, split=1, seed=1100),
    dict(family="conv2d", c0=32, c1=32, cout=32, n=2, h=61, w=133, relu=0, up=1, variant=4, split=0, seed=1101),
    dict(family="conv3d", c0=0, c1=64, cout=128, d=8, h=64, w=80, relu=1, up=0, variant=3, split=0, seed=2100),
    dict(family="conv3d", c0=32, c1=32, cout=64, d=5, h=27, w=83, relu=1, up=2, variant=0, split=1, seed=2101),
    dict(family="heads", np=144, R=131, cfeat=128, n=1, h=12 * 30, w=83, variant=0, split=1, seed=3100),
    dict(family="heads", np=48, R=33, cfeat=64, n=2, h=64, w=136, variant=4, split=0, seed=3101),
    dict(family="fused", R=32, c0=0, c1=32, n=2, h=128, w=136, relu=1, variant=0, split=1, seed=4100),
    dict(family="fused", R=17, c0=32, c1=32, n=1, h=95, w=141, relu=0, variant=3, split=0, seed=4101),
]


def n_tiles(case):
    """tiles of one launch: 8 x 16 pixels per image (or z plane) and output-channel block"""
    imgs = case["d"] if case["family"] == "conv3d" else case["n"]
    n_nb = max(1, case["cout"] // 128) if case["family"] in ("conv2d", "conv3d") else 1
    return -(-case["h"] // 8) * -(-case["w"] // 16) * imgs * n_nb


CONV2D_CASES = _conv2d_cases() + [c for c in PERSISTENT if c["family"] == "conv2d"]
CONV3D_CASES = _conv3d_cases() + [c for c in PERSISTENT if c["family"] == "conv3d"]
HEADS_CASES = _heads_cases() + [c for c in PERSISTENT if c["family"] == "heads"]
FUSED_CASES = _fused_cases() + [c for c in PERSISTENT if c["family"] == "fused"]
ALL_CASES = CONV2D_CASES + CONV3D_CASES + HEADS_CASES + FUSED_CASES

STEM_CASES = [dict(family="stem", cin=cin, cout=cout, n=(1, 2)[i % 2], h=(5, 16, 1, 9)[i % 4], w=(7, 33, 1, 130)[i % 4],
                   relu=i % 2, seed=5000 + i)
              for i, (cin, cout) in enumerate(itertools.product((1, 2, 3, 4), (32, 64)))]


def K_of(case):
    fam = case["family"]
    if fam == "heads":
        return case["cfeat"]
    return (27 if fam == "conv3d" else 9) * (case["c0"] + case["c1"])


def case_id(case):
    fam = case["family"]
    if fam in ("conv2d", "conv3d"):
        sp = ("n%d" % case["n"]) if fam == "conv2d" else ("d%d" % case["d"])
        return "%s-c%d+%d-o%d-%s-%dx%d-r%d-up%d-v%d-s%d" % (fam, case["c0"], case["c1"], case["cout"], sp, case["h"], case["w"],
                                                           case["relu"], case["up"], case["variant"], case["split"])
    if fam == "heads":
        return "heads-np%d-R%d-cf%d-n%d-%dx%d-v%d-s%d" % (case["np"], case["R"], case["cfeat"], case["n"], case["h"], case["w"],
                                                        case["variant"], case["split"])
    if fam == "fused":
        return "fused-R%d-c%d+%d-n%d-%dx%d-r%d-v%d-s%d" % (case["R"], case["c0"], case["c1"], case["n"], case["h"], case["w"],
                                                         case["relu"], case["variant"], case["split"])
    return "stem-ci%d-co%d-n%d-%dx%d-r%d" % (case["cin"], case["cout"], case["n"], case["h"], case["w"], case["relu"])


# ------------------------------------------------------------------------------------------------ mutants
CONV_MUTANTS = ("lo_whi", "hi_wlo", "lo_wlo", "swap_dydx", "dz_wrong", "swap_src", "shift_cblock", "shift_bias",
                "up_replica", "relu_before_bias")
HEADS_MUTANTS = ("lo_whi", "hi_wlo", "lo_wlo", "shift_bias", "dist_row")
FUSED_MUTANTS = ("lo_whi", "hi_wlo", "lo_wlo", "swap_dydx", "swap_src", "shift_cblock", "shift_bias", "dist_row",
                 "relu_before_bias")
STEM_MUTANTS = ("swap_dydx", "shift_bias", "relu_before_bias")


def mutant_applies(case, m):
    """whether a case can express the error at all (a second source to swap, a second K block, up-sampling, ReLU, z taps)"""
    fam = case["family"]
    if m == "dz_wrong": return fam == "conv3d" and case["d"] > 1
    if m == "swap_src": return case.get("c0", 0) > 0
    if m == "shift_cblock": return case["c0"] + case["c1"] > instance(case)[1]
    if m == "up_replica": return bool(case.get("up")) and (case["d"] if fam == "conv3d" else case["h"]) > 1
    if m == "relu_before_bias": return bool(case["relu"])
    if m == "swap_dydx": return (case["h"] > 1 or case["w"] > 1)
    return True


# ------------------------------------------------------------------------------------------------ comparison
def first_mismatch(got, want, what):
    """'' when got == want by value (so -0 == +0), else a message naming the count and the first differing element"""
    got = np.asarray(got, np.float64); want = np.asarray(want, np.float64)
    if got.shape != want.shape:
        return "%s: shape %s != %s" % (what, got.shape, want.shape)
    bad = ~((got == want) | (np.isnan(got) & np.isnan(want)))
    if not bad.any():
        return ""
    idx = tuple(int(i) for i in np.argwhere(bad)[0])
    return "%s: %d of %d elements differ; first at %s: got %r, want %r" % (what, int(bad.sum()), bad.size, idx, got[idx], want[idx])


def prob_mismatch(got, want64, ulps=4):
    """'' when every float32 prob is within `ulps` float32 ulps of the float64 sigmoid"""
    got = np.asarray(got, np.float64); want64 = np.asarray(want64, np.float64)
    tol = ulps * np.spacing(np.abs(want64).astype(np.float32)).astype(np.float64)
    bad = ~(np.abs(got - want64) <= tol)
    if not bad.any():
        return ""
    idx = tuple(int(i) for i in np.argwhere(bad)[0])
    return "prob: %d elements beyond %d ulps; first at %s: got %r, want %r" % (int(bad.sum()), ulps, idx, got[idx], want64[idx])
