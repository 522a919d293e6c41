"""Exactly representable operands for the fp32 CUDA-core network kernels (csrc/unet_simt.cu) and float64 restatements of
what those kernels compute.

The kernels are plain fp32 (fmaf chains, one thread or one register tile per output):
  sdb_conv3_nd         'same' 3x3 / 3x3x3 convolution of [nearest-upsample(in_lo), in_skip] (k_conv3x3<COUT_T, KZ>, tiles of
                       16 x 16 pixels x COUT_T channels, K in chunks of 8 channels) or, for 1..4 input channels and no second
                       source, of the input alone (k_conv3x3_stem<COUT, KZ>, one thread per pixel)
  sdb_conv_generic_nd  any kernel extent and per-axis stride with TensorFlow's 'same' padding (ResNet backbone)
  sdb_maxpool_nd       max over (pz, py, px) windows
  sdb_add_act          a + b, optional ReLU (ResNet residual sum)
  sdb_heads_2d         1x1 heads: prob = sigmoid(f . w_p + b_p), dist = f . w_d + b_d (k_heads<128>)
  sdb_class_head       softmax(f . W + b) over up to 32 outputs

Operands are small integers times powers of two: x = ints[-a, a] * x_q, W = ints[-a, a] * w_q, b = ints * b_q with b_q a
multiple of x_q * w_q.  Every product and every partial sum is then an integer multiple of x_q * w_q, and worst_case_bits
proves it stays below 2^24 quanta, so fp32 holds every partial sum exactly: the result has a single correct value whatever
the fmaf order, channel chunking or tiling, and the GPU tests compare it with the float64 references below by value, element
by element.  Only prob (expf and a division) and the softmax carry a tolerance, derived from their operation counts.

The case tables are shared by tests/test_cpu_simt_exact.py (bounds, mutants, instance and executor coverage) and
tests/test_gpu_simt_exact.py (the kernels).  Pure numpy."""
import itertools
import math
import re
import numpy as np

from convexact import _bias_act, conv_taps, first_mismatch, prob_mismatch, sigmoid64  # noqa: F401  (shared with the GPU test)

# ------------------------------------------------------------------------------------------------ recipe
PARAMS = dict(a=4, x_q=2.0 ** -3, w_q=2.0 ** -4, b_int=256, b_q=2.0 ** -7)


def worst_case_bits(p, K):
    """log2 of the largest |partial sum| / quantum an accumulator over K = taps * Cin products (plus the bias, which some
    kernels add first and some last) can reach with recipe `p`; the quantum is x_q * w_q"""
    q = p["x_q"] * p["w_q"]
    assert (p["b_q"] / q).is_integer(), "the bias quantum must be a multiple of x_q * w_q"
    return math.log2((K * p["a"] * p["x_q"] * p["a"] * p["w_q"] + p["b_int"] * p["b_q"]) / q)


def K_of(case):
    fam = case["family"]
    if fam in ("conv", "stem"):
        return case["kz"] * 9 * (case["cin_skip"] + case["cin_lo"])
    if fam == "generic":
        return int(np.prod(case["k"])) * case["cin"]
    if fam == "heads":
        return 128
    if fam == "class":
        return case["cf"]
    return 0


def class_head_ulps(C):
    """bound, in float32 ulps of the float64 softmax value, on k_class_head's error for C outputs with exact logits:
    acc - max is exact (below 2^24 quanta), each expf is within 2 ulp (CUDA math table, no fast-math), the C - 1 float32
    additions of the sum and the final division each round once.  With u = 2^-24:
        exp:      |e' / e - 1| <= 2 ulp <= 4u
        sum:      S' / S in [(1 - 4u)(1 - u)^(C-1), (1 + 4u)(1 + u)^(C-1)]
        quotient: p' / p in [(1 - 4u)(1 - u) / ((1 + 4u)(1 + u)^(C-1)), (1 + 4u)(1 + u) / ((1 - 4u)(1 - u)^(C-1))]
    and one float32 ulp at p is more than p * u, so |p' - p| < rel * p < rel / u ulps."""
    u = 2.0 ** -24
    hi = (1 + 4 * u) * (1 + u) / ((1 - 4 * u) * (1 - u) ** (C - 1)) - 1
    lo = 1 - (1 - 4 * u) * (1 - u) / ((1 + 4 * u) * (1 + u) ** (C - 1))
    return int(math.ceil(max(hi, lo) / u))


# ------------------------------------------------------------------------------------------------ generators
def _ints(rng, shape, r):
    return rng.integers(-r, r + 1, size=shape).astype(np.float64)


def _x(rng, shape):
    return (_ints(rng, shape, PARAMS["a"]) * PARAMS["x_q"]).astype(np.float32)


def _w(rng, shape):
    return (_ints(rng, shape, PARAMS["a"]) * PARAMS["w_q"]).astype(np.float32)


def _b(rng, n):
    return (_ints(rng, (n,), PARAMS["b_int"]) * PARAMS["b_q"]).astype(np.float32)


def lo_shape(case):
    uz, uy, ux = case["up"]
    return (case["n"], case["d"] // uz, case["h"] // uy, case["w"] // ux, case["cin_lo"])


def gen(case):
    """operands of one case, float32, in the layouts the kernels take (NDHWC activations, Keras (k..., Cin, Cout) kernels)"""
    fam = case["family"]
    rng = np.random.default_rng(case["seed"])
    if fam in ("conv", "stem"):
        sp = (case["n"], case["d"], case["h"], case["w"])
        cin = case["cin_skip"] + case["cin_lo"]
        return dict(skip=_x(rng, sp + (case["cin_skip"],)), lo=_x(rng, lo_shape(case)) if case["cin_lo"] else None,
                    w=_w(rng, (case["kz"], 3, 3, cin, case["cout"])), bias=_b(rng, case["cout"]))
    if fam == "generic":
        return dict(x=_x(rng, (case["n"], case["d"], case["h"], case["w"], case["cin"])),
                    w=_w(rng, tuple(case["k"]) + (case["cin"], case["cout"])), bias=_b(rng, case["cout"]))
    if fam == "maxpool":      # any float32 values: the max is exact
        return dict(x=rng.standard_normal((case["n"], case["d"], case["h"], case["w"], case["c"])).astype(np.float32))
    if fam == "add":          # any float32 values: the reference is numpy's correctly rounded float32 sum
        return dict(a=rng.standard_normal(case["size"]).astype(np.float32), b=rng.standard_normal(case["size"]).astype(np.float32))
    if fam == "heads":
        R = case["R"]
        return dict(feat=_x(rng, (case["npix"], 128)), wp=_w(rng, (128, 1)), bp=_b(rng, 1), wd=_w(rng, (128, R)), bd=_b(rng, R))
    if fam == "class":
        return dict(feat=_x(rng, (case["npix"], case["cf"])), w=_w(rng, (case["cf"], case["C"])), bias=_b(rng, case["C"]))
    raise ValueError(fam)


# ------------------------------------------------------------------------------------------------ float64 references
def upsample_nd(lo, up, mutants=()):
    """nearest up-sampling of lo [n, d', h', w', c] by (uz, uy, ux): out[z, y, x] = lo[z // uz, y // uy, x // ux].
    mutants: 'up_axes' divides each coordinate by another axis' factor (factors rotated, reads clamped to the source);
    'up_replica' makes the odd replicas along the first up-sampled axis read the next source row (clamped)."""
    up = tuple(int(v) for v in up)
    f = (up[1], up[2], up[0]) if "up_axes" in mutants else up
    idx = []
    for ax in range(3):
        n_lo = lo.shape[1 + ax]
        o = np.arange(n_lo * up[ax])
        idx.append(np.minimum(o // f[ax], n_lo - 1))
    if "up_replica" in mutants:
        ax = next(a for a in range(3) if up[a] > 1)
        o = np.arange(len(idx[ax]))
        idx[ax] = np.minimum(idx[ax] + (o % up[ax] == 1), lo.shape[1 + ax] - 1)
    return lo[:, idx[0]][:, :, idx[1]][:, :, :, idx[2]]


def conv3_ref(case, D, mutants=()):
    """sdb_conv3_nd in float64: 'same' 3x3 (kz 1) or 3x3x3 (kz 3) cross-correlation of [upsample(lo), skip] (the up-sampled
    source first, as csbdeep concatenates) with the Keras kernel (kz, 3, 3, Cin, Cout), then bias, then optional ReLU.
    mutants: 'swap_src' (skip first), 'shift_chunk' (every 8-channel chunk reads the next chunk's channels),
    'shift_cout_tile' (output channels rotated by 32), the tap mutants of convexact.conv_taps, the up-sampling mutants of
    upsample_nd and the bias mutants of convexact._bias_act."""
    x = D["skip"].astype(np.float64)
    if case["cin_lo"]:
        u = upsample_nd(D["lo"].astype(np.float64), case["up"], mutants)
        x = np.concatenate([x, u] if "swap_src" in mutants else [u, x], -1)
    if "shift_chunk" in mutants:
        x = np.roll(x, -8, axis=-1)
    kz, cin, cout = case["kz"], x.shape[-1], case["cout"]
    Wt = D["w"].astype(np.float64).reshape(kz * 9, cin, cout).transpose(0, 2, 1)        # [tap][cout][cin]
    if kz == 1:
        y = conv_taps(x[:, 0], Wt, 2, mutants)[:, None]
    else:
        y = np.stack([conv_taps(v, Wt, 3, mutants) for v in x])
    if "shift_cout_tile" in mutants:
        y = np.roll(y, 32, axis=-1)
    return _bias_act(y, dict(bias=D["bias"], w_scale=1.0), case["relu"], mutants)


def same_padding(n, k, s, mutants=()):
    """TensorFlow 'same': out = ceil(n / s), pad_total = max((out - 1) * s + k - n, 0), pad_before = pad_total // 2 (the odd
    row goes after).  mutant 'pad_ceil': pad_before = ceil(pad_total / 2)."""
    out = -(-n // s)
    total = max((out - 1) * s + k - n, 0)
    return out, total, ((total + 1) // 2 if "pad_ceil" in mutants else total // 2)


def generic_ref(case, D, mutants=()):
    """sdb_conv_generic_nd in float64: out[o] = sum over taps t of x[o * s - pad_before + t] . W[t] (zero outside), + bias,
    optional ReLU; per axis (z, y, x).  mutants: 'pad_ceil', 'stride_axes' (input coordinates use the strides rotated
    (sy, sx, sz); output extents stay right), 'flip_kernel' (convolution instead of correlation), bias mutants."""
    x = D["x"].astype(np.float64)
    W = D["w"].astype(np.float64)
    if "flip_kernel" in mutants:
        W = W[::-1, ::-1, ::-1]
    ext = x.shape[1:4]
    k, s = tuple(case["k"]), tuple(case["s"])
    s_in = (s[1], s[2], s[0]) if "stride_axes" in mutants else s
    geo = [same_padding(ext[a], k[a], s[a], mutants) for a in range(3)]
    outs = [g[0] for g in geo]
    y = np.zeros((x.shape[0],) + tuple(outs) + (W.shape[-1],))
    for t in itertools.product(*(range(v) for v in k)):
        idx, ok = [], []
        for a in range(3):
            i = np.arange(outs[a]) * s_in[a] - geo[a][2] + t[a]
            ok.append((i >= 0) & (i < ext[a]))
            idx.append(np.clip(i, 0, ext[a] - 1))
        m = ok[0][:, None, None] & ok[1][None, :, None] & ok[2][None, None, :]
        if not m.any():
            continue
        xs = x[:, idx[0]][:, :, idx[1]][:, :, :, idx[2]] * m[None, ..., None]
        y += xs @ W[t]
    return _bias_act(y, dict(bias=D["bias"], w_scale=1.0), case["relu"], mutants)


def maxpool_ref(case, D, mutants=()):
    """sdb_maxpool_nd: max over (pz, py, px) windows.  mutant 'pool_axes': the window extents are rotated (py, px, pz) while
    the output stride stays (pz, py, px); reads clamped to the input."""
    x = D["x"]
    pool = tuple(case["pool"])
    ext = (pool[1], pool[2], pool[0]) if "pool_axes" in mutants else pool
    outs = [x.shape[1 + a] // pool[a] for a in range(3)]
    m = np.full((x.shape[0],) + tuple(outs) + (x.shape[-1],), -np.inf, np.float32)
    for t in itertools.product(*(range(v) for v in ext)):
        idx = [np.minimum(np.arange(outs[a]) * pool[a] + t[a], x.shape[1 + a] - 1) for a in range(3)]
        m = np.maximum(m, x[:, idx[0]][:, :, idx[1]][:, :, :, idx[2]])
    return m


def add_ref(case, D):
    y = D["a"] + D["b"]                                                   # float32, correctly rounded
    return np.maximum(y, np.float32(0)) if case["relu"] else y


def heads_ref(case, D, mutants=()):
    """sdb_heads_2d in float64: logits z = f . [w_p | w_d] + [b_p | b_d] (exact); prob = sigmoid(z_0), dist = z_1..R.
    mutants: 'shift_bias' (bias vector rotated by one), 'dist_row' (dist takes rows 2..R+1)"""
    f = D["feat"].astype(np.float64)
    W = np.concatenate([D["wp"], D["wd"]], 1).astype(np.float64)
    b = np.concatenate([D["bp"], D["bd"]]).astype(np.float64)
    if "shift_bias" in mutants:
        b = np.roll(b, 1)
    z = f @ W + b
    r0 = 2 if "dist_row" in mutants else 1
    zp = np.concatenate([z, np.zeros((z.shape[0], 1))], 1)
    return sigmoid64(z[:, 0]), zp[:, r0:r0 + case["R"]]


def class_ref(case, D, mutants=()):
    """sdb_class_head in float64: softmax over the C exact logits f . W + b.  mutants: 'shift_bias', 'class_col' (output
    columns rotated by one)"""
    b = D["bias"].astype(np.float64)
    if "shift_bias" in mutants:
        b = np.roll(b, 1)
    z = D["feat"].astype(np.float64) @ D["w"].astype(np.float64) + b
    e = np.exp(z - z.max(1, keepdims=True))
    p = e / e.sum(1, keepdims=True)
    return np.roll(p, 1, axis=1) if "class_col" in mutants else p


def softmax_mismatch(got, want64, C):
    return prob_mismatch(got, want64, class_head_ulps(C))


def logit_bits(case):
    """bits of max |acc - max acc| / quantum in k_class_head: twice the accumulator bound"""
    return worst_case_bits(PARAMS, K_of(case)) + 1


# ------------------------------------------------------------------------------------------------ dispatch of sdb_conv3_nd
def conv3_instance(cin_skip, cin_lo, cout, kz):
    """the kernel sdb_conv3_nd launches: a Python copy of its dispatch"""
    if cin_lo == 0 and cin_skip + cin_lo <= 4:
        return "k_conv3x3_stem<%d, %d>" % (cout, kz)
    return "k_conv3x3<%d, %d>" % (64 if cout % 64 == 0 else 32, kz)


def instance(case):
    fam = case["family"]
    if fam in ("conv", "stem"):
        return conv3_instance(case["cin_skip"], case["cin_lo"], case["cout"], case["kz"])
    if fam == "heads":
        return "k_heads<128>"
    return None


def instances_in_source(path):
    """every k_conv3x3<N, KZ>, k_conv3x3_stem<N, KZ> and k_heads<CF> that unet_simt.cu launches"""
    src = open(path).read()
    out = {"k_conv3x3<%s, %s>" % m for m in re.findall(r"\(k_conv3x3<(\d+),\s*(\d+)>\)", src)}
    out |= {"k_conv3x3_stem<%s, %s>" % m for m in re.findall(r"\(k_conv3x3_stem<(\d+),\s*(\d+)>\)", src)}
    out |= {"k_heads<%s>" % m for m in re.findall(r"\(k_heads<(\d+)>\)", src)}
    return out


# ------------------------------------------------------------------------------------------------ launch classes
def pad_class(n, k, s):
    total = same_padding(n, k, s)[1]
    return "0" if total == 0 else ("odd" if total % 2 else "even")


def conv3_class(cin_skip, cin_lo, cout, kz, up):
    inst = conv3_instance(cin_skip, cin_lo, cout, kz)
    if "stem" in inst:
        return ("conv3_nd", inst, "cin%d" % cin_skip)
    return ("conv3_nd", inst, tuple(int(v) for v in up) if cin_lo else None)


def generic_classes(k, s):
    """every (kernel, stride, per-axis padding class) an input of any extent can produce; the class of an axis depends on
    its extent only modulo the stride, so extents 1..4 reach them all"""
    per_axis = [sorted({pad_class(n, k[a], s[a]) for n in range(1, 5)}) for a in range(3)]
    return {("conv_generic_nd", tuple(k), tuple(s), pc) for pc in itertools.product(*per_axis)}


def case_class(case):
    fam = case["family"]
    if fam in ("conv", "stem"):
        return conv3_class(case["cin_skip"], case["cin_lo"], case["cout"], case["kz"], case["up"])
    if fam == "generic":
        pc = tuple(pad_class(case[ax], case["k"][a], case["s"][a]) for a, ax in enumerate("dhw"))
        return ("conv_generic_nd", tuple(case["k"]), tuple(case["s"]), pc)
    if fam == "maxpool":
        return ("maxpool_nd", tuple(case["pool"]))
    if fam == "add":
        return ("add_act",)
    if fam == "heads":
        return ("heads_2d", "k_heads<128>", case["R"])
    return ("class_head", case["cf"], case["C"])


def executor_classes(config):
    """launch classes of the fp32 CUDA-core executors of models/unet_device.py for `config`: UNetDeviceND for U-Nets (the
    2-D executor, the fp16-overflow fallback and the cross-check executor of the tensor-core paths, whose stem and class
    branch it also runs) and ResNetDeviceND for the 3-D ResNet backbone.  A walk over the layer lists with the executors'
    dispatch: which entry point, which kernel instance, which up-sampling / pool / stride pattern and padding class."""
    from stardist_b200.models.weights import unet_layers, resnet_layers
    nd = config.n_dim
    kz = 1 if nd == 2 else 3
    to3 = lambda t: (1,) + tuple(int(v) for v in t) if len(t) == 2 else tuple(int(v) for v in t)
    out = set()
    resnet = getattr(config, "backbone", "unet") == "resnet"
    layers = resnet_layers(config) if resnet else unet_layers(config)
    up = None
    for l in layers:
        kind = l["kind"]
        if kind == "conv" and resnet:
            if tuple(l["k"]) == (3, 3, 3) and tuple(l["stride"]) == (1, 1, 1) and l["cin"] > 4:
                out.add(conv3_class(l["cin"], 0, l["cout"], 3, (1, 1, 1)))
            else:
                out |= generic_classes(tuple(l["k"]), tuple(l["stride"]))
        elif kind == "conv":
            c_lo = l.get("cin_lo", 0) if up is not None else 0
            out.add(conv3_class(l["cin"] - c_lo, c_lo, l["cout"], kz, to3(up) if c_lo else None))
            up = None
        elif kind == "pool":
            out.add(("maxpool_nd", to3(l["pool"])))
        elif kind == "up":
            up = l["pool"]
        elif kind == "block_end":
            out.add(("add_act",))
        elif kind == "head" and l["name"] == "dist":
            out.add(("heads_2d", "k_heads<128>", l["cout"]))
            assert l["cin"] == 128, "sdb_heads_2d takes 128 feature channels"
        elif kind == "conv_class":
            out.add(conv3_class(l["cin"], 0, l["cout"], kz, None))
        elif kind == "head_class":
            out.add(("class_head", l["cin"], l["cout"]))
    return out


# ------------------------------------------------------------------------------------------------ case tables
# A reduced cross product: every listed value appears (test_cpu_simt_exact.py checks it), and the product's rotation keeps
# the float64 references cheap.
COUTS = (32, 64, 96, 128, 256)
MIXES = [(8, 0), (16, 0), (40, 0), (8, 8), (16, 8), (8, 24), (32, 32)]          # (cin_skip, cin_lo)
UPS = {1: [(1, 2, 2), (1, 2, 1), (1, 1, 2), (1, 4, 2)], 3: [(1, 2, 2), (2, 2, 2), (1, 2, 1), (2, 1, 1)]}
HW = [(1, 1), (15, 17), (16, 16), (17, 33), (33, 15), (1, 130), (130, 1), (16, 130)]
DEPTHS = (1, 2, 3, 5)


def _round_up(v, f):
    return -(-v // f) * f


def _conv_cases():
    cases = []
    for i, (cout, kz, (cs, cl)) in enumerate(itertools.product(COUTS, (1, 3), MIXES)):
        h, w = HW[i % len(HW)]
        up = UPS[kz][(i // 2) % len(UPS[kz])] if cl else (1, 1, 1)
        d = DEPTHS[(i // 3) % len(DEPTHS)] if kz == 3 else 1
        n = (1, 2, 3)[(i // 5) % 3]
        d, h, w = (_round_up(v, f) for v, f in zip((d, h, w), up))
        if h * w > 1000:                     # keep the references cheap: large planes run as one plane of one image
            n, d = 1, min(d, 2) if kz == 3 else 1
        cases.append(dict(family="conv", cin_skip=cs, cin_lo=cl, up=up, cout=cout, kz=kz, n=n, d=d, h=h, w=w,
                          relu=(i // 2) % 2, seed=6000 + i))
    # the largest K of the networks: 27 * 256 (3-D decoder, ResNet features), and cout 256 with two sources
    cases.append(dict(family="conv", cin_skip=128, cin_lo=128, up=(2, 2, 2), cout=32, kz=3, n=1, d=2, h=4, w=6, relu=1, seed=6100))
    cases.append(dict(family="conv", cin_skip=64, cin_lo=64, up=(1, 2, 2), cout=256, kz=1, n=2, h=18, w=20, d=1, relu=0, seed=6101))
    return cases


def _stem_cases():
    cases = []
    for i, (cin, cout, kz) in enumerate(itertools.product((1, 2, 3, 4), (32, 64), (1, 3))):
        h, w = HW[(i + 1) % len(HW)]
        d = DEPTHS[i % len(DEPTHS)] if kz == 3 else 1
        n = (1, 2)[(i // 2) % 2]
        if h * w > 1000:
            n = 1
        cases.append(dict(family="stem", cin_skip=cin, cin_lo=0, up=(1, 1, 1), cout=cout, kz=kz, n=n, d=d, h=h, w=w,
                          relu=i % 2, seed=6200 + i))
    # more than one 128-thread block and not a multiple of it; the 3-D tensor-core executor's stem at its test size
    cases.append(dict(family="stem", cin_skip=3, cin_lo=0, up=(1, 1, 1), cout=64, kz=1, n=2, d=1, h=37, w=45, relu=1, seed=6300))
    cases.append(dict(family="stem", cin_skip=1, cin_lo=0, up=(1, 1, 1), cout=32, kz=3, n=1, d=16, h=64, w=64, relu=1, seed=6301))
    return cases


KERNELS = [(7, 7, 7), (3, 3, 3), (1, 1, 1), (1, 3, 3)]
STRIDES = [(1, 1, 1), (2, 2, 2), (1, 2, 2), (2, 1, 1)]
ODD, EVEN = (5, 3, 1, 7), (4, 6, 2)


def _generic_cases():
    """every kernel x stride, and for each every odd / even combination of the extents along its strided axes (odd and
    even extents give odd and even pad_total there; extent 1 appears too)"""
    cases = []
    i = 0
    for k, s in itertools.product(KERNELS, STRIDES):
        strided = [a for a in range(3) if s[a] > 1]
        for par in itertools.product((0, 1), repeat=len(strided)):
            ext = [ODD[(i + a) % len(ODD)] if (a + i) % 3 else EVEN[(i + a) % len(EVEN)] for a in range(3)]
            for a, p in zip(strided, par):
                ext[a] = (ODD if p else EVEN)[(i + a) % (len(ODD) if p else len(EVEN))]
            cin = (1, 8, 32)[i % 3]
            cout = (32, 8, 64, 5)[i % 4]
            if k == (7, 7, 7) and cin == 32:
                cout = 8
            cases.append(dict(family="generic", k=k, s=s, cin=cin, cout=cout, n=(1, 2)[(i // 3) % 2], d=ext[0], h=ext[1],
                              w=ext[2], relu=(i // 2) % 2, seed=6400 + i))
            i += 1
    # 2-D (d = kz = sz = 1), including an even kernel extent
    for j, (k, s, hw) in enumerate([((1, 3, 3), (1, 2, 2), (9, 10)), ((1, 1, 1), (1, 2, 2), (7, 8)), ((1, 7, 7), (1, 1, 1), (5, 12)),
                                    ((1, 2, 4), (1, 1, 2), (6, 9)), ((1, 3, 3), (1, 1, 1), (1, 17))]):
        cases.append(dict(family="generic", k=k, s=s, cin=(8, 1, 32)[j % 3], cout=(16, 32)[j % 2], n=2, d=1, h=hw[0], w=hw[1],
                          relu=j % 2, seed=6500 + j))
    return cases


POOLS = [(1, 2, 2), (2, 2, 2), (1, 2, 1), (2, 1, 1), (1, 1, 2)]


def _maxpool_cases():
    cases = []
    for i, (pool, c) in enumerate(itertools.product(POOLS, (4, 32, 36))):
        ext = [(1, 2)[(i + a) % 2] * pool[a] * (3, 5, 7)[(i + a) % 3] for a in range(3)]
        cases.append(dict(family="maxpool", pool=pool, c=c, n=(1, 2)[i % 2], d=ext[0], h=ext[1], w=ext[2], seed=6600 + i))
    # more output float4s than the launch's 132 * 16 blocks of 256 threads: the grid-stride loop wraps
    cases.append(dict(family="maxpool", pool=(1, 2, 2), c=32, n=1, d=8, h=256, w=256, seed=6700))
    return cases


MAXPOOL_GRID = 132 * 16 * 256          # float4 outputs of one sweep of sdb_maxpool_nd's grid
ADD_GRID = 132 * 32 * 256              # elements of one sweep of sdb_add_act's grid


def _add_cases():
    return [dict(family="add", size=1, relu=1, seed=6800), dict(family="add", size=1000, relu=0, seed=6801),
            dict(family="add", size=4099, relu=1, seed=6802), dict(family="add", size=ADD_GRID + 12345, relu=1, seed=6803)]


HEADS_R = (1, 3, 31, 32, 33, 64, 96, 127, 128, 187, 255, 256)
HEADS_NPIX = (1, 31, 33, 4099)


def _heads_cases():
    return [dict(family="heads", R=R, npix=npix, seed=6900 + i) for i, (R, npix) in enumerate(itertools.product(HEADS_R, HEADS_NPIX))]


CLASS_C = (1, 2, 3, 4, 17, 32)
CLASS_NPIX = (1, 200, 1000, 4099)


def _class_cases():
    return [dict(family="class", C=C, cf=cf, npix=CLASS_NPIX[i % len(CLASS_NPIX)], seed=7000 + i)
            for i, (C, cf) in enumerate(itertools.product(CLASS_C, (32, 128)))]


CONV_CASES = _conv_cases()
STEM_CASES = _stem_cases()
GENERIC_CASES = _generic_cases()
MAXPOOL_CASES = _maxpool_cases()
ADD_CASES = _add_cases()
HEADS_CASES = _heads_cases()
CLASS_CASES = _class_cases()
ALL_CASES = CONV_CASES + STEM_CASES + GENERIC_CASES + MAXPOOL_CASES + ADD_CASES + HEADS_CASES + CLASS_CASES


def case_id(case):
    fam = case["family"]
    if fam in ("conv", "stem"):
        up = "-up%d%d%d" % tuple(case["up"]) if case["cin_lo"] else ""
        return "%s-k%d-c%d+%d%s-o%d-n%dx%dx%dx%d-r%d" % (fam, case["kz"], case["cin_skip"], case["cin_lo"], up, case["cout"],
                                                        case["n"], case["d"], case["h"], case["w"], case["relu"])
    if fam == "generic":
        return "generic-k%d%d%d-s%d%d%d-c%d-o%d-n%dx%dx%dx%d-r%d" % (tuple(case["k"]) + tuple(case["s"]) + (
            case["cin"], case["cout"], case["n"], case["d"], case["h"], case["w"], case["relu"]))
    if fam == "maxpool":
        return "maxpool-p%d%d%d-c%d-n%dx%dx%dx%d" % (tuple(case["pool"]) + (case["c"], case["n"], case["d"], case["h"], case["w"]))
    if fam == "add":
        return "add-%d-r%d" % (case["size"], case["relu"])
    if fam == "heads":
        return "heads-R%d-npix%d" % (case["R"], case["npix"])
    return "class-C%d-cf%d-npix%d" % (case["C"], case["cf"], case["npix"])


# ------------------------------------------------------------------------------------------------ mutants
CONV_MUTANTS = ("swap_dydx", "dz_wrong", "swap_src", "up_axes", "up_replica", "shift_chunk", "shift_cout_tile", "shift_bias",
                "relu_before_bias")
STEM_MUTANTS = ("swap_dydx", "dz_wrong", "shift_bias", "relu_before_bias")
GENERIC_MUTANTS = ("pad_ceil", "stride_axes", "flip_kernel", "shift_bias", "relu_before_bias")
MAXPOOL_MUTANTS = ("pool_axes",)
HEADS_MUTANTS = ("shift_bias", "dist_row")
CLASS_MUTANTS = ("shift_bias", "class_col")


def mutant_applies(case, m):
    """whether a case can express the error at all"""
    fam = case["family"]
    if m == "swap_dydx": return case["h"] > 1 or case["w"] > 1
    if m == "dz_wrong": return case["kz"] == 3 and case["d"] > 1
    if m == "swap_src": return case["cin_lo"] > 0
    if m == "up_axes": return case["cin_lo"] > 0 and len(set(case["up"])) > 1
    if m == "up_replica": return case["cin_lo"] > 0
    if m == "shift_chunk": return case["cin_skip"] + case["cin_lo"] > 8
    if m == "shift_cout_tile": return case["cout"] > 32
    if m == "relu_before_bias": return bool(case["relu"])
    if m == "pad_ceil": return any(pad_class(case[ax], case["k"][a], case["s"][a]) == "odd" for a, ax in enumerate("dhw"))
    if m == "stride_axes": return len(set(case["s"])) > 1
    if m == "flip_kernel": return max(case["k"]) > 1
    if m == "pool_axes": return len(set(case["pool"])) > 1
    if m in ("shift_bias", "class_col") and fam == "class": return case["C"] > 1
    return True
