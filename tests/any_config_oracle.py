"""float64 restatement of the generalised StarDist networks (any kernel extent, channel width, feature width and Keras
activation) and the cases of the csrc/unet_any.cu layer tests.

The activation table is written out from the TensorFlow / Keras definitions.  TensorFlow cannot be run next to these
tests, so agreement with TensorFlow's own float32 bits is not pinned; the device kernels are held to these float64
values within the bounds stated in tests/test_gpu_any_config.py.
"""
import itertools
import math

import numpy as np
import torch
import torch.nn.functional as F

from stardist_b200.models.weights import unet_layers, resnet_layers

SELU_ALPHA = 1.6732632423543772848170429916717
SELU_SCALE = 1.0507009873554804934193349852946


def act64(name, x):
    """Keras activation `name` on a float64 tensor"""
    if name == 'linear':
        return x
    if name == 'relu':
        return torch.clamp_min(x, 0.0)
    if name == 'elu':                                   # alpha = 1
        return torch.where(x > 0, x, torch.expm1(x))
    if name == 'selu':
        return SELU_SCALE * torch.where(x > 0, x, SELU_ALPHA * torch.expm1(x))
    if name == 'tanh':
        return torch.tanh(x)
    if name == 'sigmoid':
        return 1.0 / (1.0 + torch.exp(-x))
    if name == 'softplus':                              # log(1 + exp(x))
        return torch.logaddexp(torch.zeros_like(x), x)
    if name == 'softsign':
        return x / (1.0 + torch.abs(x))
    if name == 'exponential':
        return torch.exp(x)
    if name == 'swish':                                 # x * sigmoid(x)
        return x / (1.0 + torch.exp(-x))
    if name == 'gelu':                                  # approximate=False: 0.5 x (1 + erf(x / sqrt 2)) = 0.5 x erfc(-x / sqrt 2)
        return 0.5 * x * torch.special.erfc(-x / math.sqrt(2.0))
    raise KeyError(name)


ACTS = ('linear', 'relu', 'elu', 'selu', 'tanh', 'sigmoid', 'softplus', 'softsign', 'exponential', 'swish', 'gelu')


def tf_same_pad(size, k, s):
    """TensorFlow padding='same': (pad_before, pad_after) of one axis"""
    out = -(-size // s)
    total = max((out - 1) * s + k - size, 0)
    return total // 2, total - total // 2


def upsample(x, up):
    """nearest up-sampling of channels-last x [N, *sp, C] by the factors `up`"""
    for ax, u in enumerate(up):
        if u > 1:
            x = torch.repeat_interleave(x, int(u), dim=1 + ax)
    return x


def conv_same(x, k, b, stride=None, act='linear'):
    """act(conv(x) + b) as Keras Conv2D / Conv3D with padding='same' computes it: x [N, *sp, Cin], k (*ks, Cin, Cout)"""
    nd = x.dim() - 2
    ks = tuple(k.shape[:nd])
    stride = (1,) * nd if stride is None else tuple(stride)
    pads = []
    for ax in reversed(range(nd)):
        pads += list(tf_same_pad(x.shape[1 + ax], ks[ax], stride[ax]))
    xc = F.pad(x.movedim(-1, 1), pads)
    wc = k.permute(nd + 1, nd, *range(nd))
    y = (F.conv2d if nd == 2 else F.conv3d)(xc, wc, b, stride=stride)
    return act64(act, y.movedim(1, -1))


def maxpool(x, pool):
    nd = x.dim() - 2
    y = (F.max_pool2d if nd == 2 else F.max_pool3d)(x.movedim(-1, 1), tuple(pool), tuple(pool))
    return y.movedim(1, -1)


def _heads(W, feat, n_classes_base):
    wp, bp = W['prob']; wd, bd = W['dist']
    cf = feat.shape[-1]
    prob = torch.sigmoid(feat @ wp.reshape(cf, 1) + bp)[..., 0]
    dist = feat @ wd.reshape(cf, -1) + bd
    return prob, dist


def _class(config, W, base, act):
    if config.n_classes is None:
        return None
    x = base
    if 'features_class' in W:
        x = conv_same(x, *W['features_class'], act=act)
    wc, bc = W['prob_class']
    return torch.softmax(x @ wc.reshape(x.shape[-1], -1) + bc, dim=-1)


def forward(config, weights, x, device='cpu'):
    """(prob, dist, prob_class or None) float64 numpy of the model `config` with `weights` on x [N, *sp, Cin]"""
    W = {k: (torch.as_tensor(np.asarray(v[0]), dtype=torch.float64, device=device),
             torch.as_tensor(np.asarray(v[1]), dtype=torch.float64, device=device)) for k, v in weights.items()}
    x = torch.as_tensor(np.asarray(x), dtype=torch.float64, device=device)
    with torch.no_grad():
        if getattr(config, 'backbone', 'unet') == 'resnet':
            feat, base, act = _resnet(config, W, x)
        else:
            feat, base, act = _unet(config, W, x)
        prob, dist = _heads(W, feat, None)
        pc = _class(config, W, base, act)
    f = lambda t: None if t is None else t.cpu().numpy()
    return f(prob), f(dist), f(pc)


def _unet(config, W, x):
    skips, lo, up, base = {}, None, None, None
    for l in unet_layers(config):
        if l['kind'] == 'conv':
            if l['name'] == 'features':
                base = x
            inp = x if lo is None else torch.cat([upsample(lo, up), x], dim=-1)
            x = conv_same(inp, *W[l['name']], act=l['act'])
            lo = None
        elif l['kind'] == 'pool':
            if 'save_skip' in l:
                skips[l['save_skip']] = x
            x = maxpool(x, l['pool'])
        elif l['kind'] == 'up':
            lo, up = x, tuple(l['pool'])
            x = skips.pop(l['skip'])
    return x, (x if base is None else base), config.unet_activation


def _resnet(config, W, x):
    block_in = shortcut = base = None
    for l in resnet_layers(config):
        if l['kind'] == 'block_begin':
            block_in, shortcut = x, None
        elif l['kind'] == 'conv':
            if l['name'] == 'features':
                base = x
            y = conv_same(block_in if l['src'] == 'block_in' else x, *W[l['name']], stride=l['stride'], act=l['act'])
            if l['dst'] == 'shortcut':
                shortcut = y
            else:
                x = y
        elif l['kind'] == 'block_end':
            x = act64(l['act'], (block_in if shortcut is None else shortcut) + x)
            block_in = shortcut = None
    return x, (x if base is None else base), config.resnet_activation


# ------------------------------------------------------------------------------------------------ layer cases
VMAX = 3            # operands are integers in [-VMAX, VMAX]


def _conv_cases():
    """sdb_conv_any_nd cases: every kernel of KERNELS at strides 1 and 2, two (cin, cout) pairs each, so that every cin of
    CINS and every cout of COUTS occurs; and every kernel with an up-sampled source (2-D and 3-D factors)"""
    kernels = [(1, 3, 3), (5, 5), (2, 2), (7, 7, 7), (4, 1)]
    cins, couts = [1, 3, 5, 16, 40], [1, 16, 48, 96]
    out, i = [], 0
    for k, s in itertools.product(kernels, (1, 2)):
        nd = len(k)
        for _ in range(2):
            cin, cout = cins[i % len(cins)], couts[i % len(couts)]
            i += 1
            shape = (19, 37) if nd == 2 else (5, 11, 20)
            out.append(dict(id='k%s_s%d_ci%d_co%d' % (''.join(map(str, k)), s, cin, cout), nd=nd, k=k, s=(s,) * nd, n=2,
                            shape=shape, c_skip=cin, c_lo=0, up=(1,) * nd, cout=cout, act=('relu' if i % 2 else 'linear')))
    for j, k in enumerate(kernels):
        nd = len(k)
        ups = [(2, 2), (1, 2)] if nd == 2 else [(1, 2, 2), (2, 2, 2)]
        for u in ups:
            shape = (18, 34) if nd == 2 else (4, 10, 18)
            c_lo, c_skip, cout = [(16, 16, 48), (5, 3, 96), (40, 1, 16), (3, 5, 1)][(j + len(out)) % 4]
            out.append(dict(id='k%s_up%s_lo%d_sk%d_co%d' % (''.join(map(str, k)), ''.join(map(str, u)), c_lo, c_skip, cout), nd=nd,
                            k=k, s=(1,) * nd, n=2, shape=shape, c_skip=c_skip, c_lo=c_lo, up=u, cout=cout, act='relu'))
    return out


CONV_CASES = _conv_cases()


def max_partial(case, vmax=VMAX):
    """largest |partial sum| the convolution forms on a case: every tap times every input channel, plus the bias"""
    return int(np.prod(case['k'])) * (case['c_skip'] + case['c_lo']) * vmax * vmax + vmax


def gen_conv(case, seed=0):
    """(skip [n, *shape, c_skip], lo [n, *shape / up, c_lo] or None, kernel (*k, cin, cout), bias) float32 integers"""
    rng = np.random.default_rng(seed + sum(map(ord, case['id'])))
    r = lambda *s: rng.integers(-VMAX, VMAX + 1, size=s).astype(np.float32)
    n, shape = case['n'], tuple(case['shape'])
    skip = r(n, *shape, case['c_skip'])
    lo = None
    if case['c_lo']:
        lo = r(n, *(s // u for s, u in zip(shape, case['up'])), case['c_lo'])
    k = r(*case['k'], case['c_lo'] + case['c_skip'], case['cout'])
    b = r(case['cout'])
    return skip, lo, k, b


def conv_ref(case, skip, lo, k, b):
    t = lambda a: torch.from_numpy(a).double()
    x = t(skip)
    if lo is not None:
        x = torch.cat([upsample(t(lo), case['up']), x], dim=-1)
    return conv_same(x, t(k), t(b), stride=case['s'], act=case['act']).numpy()
