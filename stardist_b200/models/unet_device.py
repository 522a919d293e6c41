"""Device executor of the U-Net forward pass: walks weights.unet_layers() and launches the CUDA
kernels of libstardist_b200.so on NHWC float32 tensors (torch is only the memory substrate).

Reference: `keras_model.predict(x[np.newaxis])` at stardist/models/base.py:408-410 for the graph
built in model2d.py:310-349.  The decoder's UpSampling+Concatenate is never materialised: the
conv kernel reads [upsample(x_lo), skip] through its loader address math.
"""
import os
import numpy as np
import torch
from .. import _lib as L
from .weights import unet_layers, resnet_layers


# Keras activation name -> activation id of the csrc/unet_any.cu kernels (0 and 1 are also the `relu` flag of unet_simt.cu)
ACTIVATIONS = {'linear': 0, 'relu': 1, 'elu': 2, 'selu': 3, 'tanh': 4, 'sigmoid': 5, 'softplus': 6, 'softsign': 7,
               'exponential': 8, 'swish': 9, 'gelu': 10}


def act_id(name):
    """activation id of a Keras activation name; NotImplementedError naming it for any other (e.g. 'hard_sigmoid', whose
    definition changed between Keras versions)"""
    if name not in ACTIVATIONS:
        raise NotImplementedError("activation %r is not supported (supported: %s)" % (name, ", ".join(ACTIVATIONS)))
    return ACTIVATIONS[name]


def check_activations(layers):
    """act_id of every activation of a layer list, so that an unsupported one raises before anything touches the device"""
    for l in layers:
        if l['kind'] in ('conv', 'conv_class', 'block_end'):
            act_id(l['act'])


# One predicate per unet_simt.cu kernel: the layers it accepts run on it, every other layer on csrc/unet_any.cu.
def conv3_accepts(nd, k, stride, cin_skip, cin_lo, cout, act):
    """sdb_conv3_nd: 3^d kernels at stride 1 with ReLU or linear; its stem variant takes cin <= 4 without an up-sampled
    source and cout 32 or 64, its tiled variant input channels in multiples of 8 and output channels in multiples of 32"""
    if tuple(k) != (3,) * nd or tuple(stride) != (1,) * nd or act not in ('relu', 'linear'):
        return False
    if cin_lo == 0 and cin_skip <= 4:
        return cout in (32, 64)
    return cin_skip % 8 == 0 and cin_lo % 8 == 0 and cout % 32 == 0


def conv_generic_accepts(act):
    """sdb_conv_generic_nd: any kernel extent and stride, ReLU or linear"""
    return act in ('relu', 'linear')


def maxpool_accepts(c):
    """sdb_maxpool_nd: channel counts that are multiples of 4"""
    return c % 4 == 0


def heads_accept(cf, n_rays):
    """sdb_heads_2d: 128 feature channels, and its weight and output tables within 200 KB of shared memory"""
    return cf == 128 and (160 * (n_rays + 1) + 32 * 129) * 4 <= 200 * 1024


def add_act_accepts(act):
    """sdb_add_act: ReLU or linear"""
    return act in ('relu', 'linear')


# Training (csrc/unet_train.cu): the layers these predicates accept take the backward kernels of the default family, every
# other layer the unet_any.cu / any-extent entry points.
def conv_wgrad_accepts(nd, k):
    """sdb_conv_wgrad_nd: 1^d and 3^d kernels, and (1, 3, 3) in 3-D; sdb_conv_wgrad_any_nd takes every other extent"""
    k = tuple(k)
    return k in ((1,) * nd, (3,) * nd) or (nd == 3 and k == (1, 3, 3))


def conv_dgrad3_accepts(nd, k, cin, cout):
    """input gradient as sdb_conv3_nd of dY (cout channels) with the flipped kernel (cin outputs): 3^d kernels whose
    transposed shape that kernel takes (in particular every cin % 32 == 0 layer with cout a multiple of 8); every other layer
    runs sdb_conv_dgrad_any_nd"""
    return conv3_accepts(nd, k, (1,) * nd, cout, 0, cin, 'linear')


def keeps_preactivation(act):
    """training keeps the pre-activation z of layers whose activation derivative needs it (every activation but ReLU and
    linear, whose backward reads the output)"""
    return act not in ('relu', 'linear')


class UNetDeviceND:
    """exact-fp32 CUDA-core executor for 2-D (NHWC) and 3-D (NDHWC) U-Nets: csrc/unet_simt.cu for the layers its kernels
    accept (see the *_accepts predicates), csrc/unet_any.cu for every other kernel extent, channel count, feature width and
    activation"""

    def __init__(self, config, weights, device=None):
        if config.unet_batch_norm:
            raise NotImplementedError("unet_batch_norm=True is not supported on this path")
        self.layers = unet_layers(config)
        check_activations(self.layers)
        L.require_cuda()
        self.config = config
        self.nd = config.n_dim
        self.device = torch.device("cuda") if device is None else torch.device(device)
        self._upload(weights)

    def _upload(self, weights):
        self.w = {}
        for name, (k, b) in weights.items():
            self.w[name] = (torch.from_numpy(np.ascontiguousarray(k, dtype=np.float32)).to(self.device),
                            torch.from_numpy(np.ascontiguousarray(b, dtype=np.float32)).to(self.device))

    @staticmethod
    def _dhw(x):
        return (1,) + tuple(x.shape[1:3]) if x.dim() == 4 else tuple(x.shape[1:4])

    def _conv(self, x, x_lo, name, act, up, stride=None, keep_z=False):
        """act(conv(x) + bias) with 'same' padding; the input channels are [upsample(x_lo), x] when x_lo is given.
        keep_z=True (activations other than ReLU / linear) returns (z, act(z)): the same kernel runs linear and sdb_act_any
        applies the activation, which gives the fused result bit for bit."""
        lib = L.load()
        k, b = self.w[name]
        n = x.shape[0]; d, h, w = self._dhw(x); c_skip = x.shape[-1]
        c_lo = 0 if x_lo is None else x_lo.shape[-1]
        cout = k.shape[-1]
        assert k.shape[-2] == c_skip + c_lo, (name, k.shape, c_skip, c_lo)
        ks = tuple(k.shape[:-2])
        stride = (1,) * self.nd if stride is None else tuple(stride)
        uz, uy, ux = ((1,) + tuple(up)) if len(up) == 2 else tuple(up)
        if conv3_accepts(self.nd, ks, stride, c_skip, c_lo, cout, act):
            assert not keep_z
            out = torch.empty(tuple(x.shape[:-1]) + (cout,), dtype=torch.float32, device=x.device)
            L.check(lib.sdb_conv3_nd(L.ptr(x), L.ptr(x_lo), n, d, h, w, c_skip, c_lo, int(uz), int(uy), int(ux), L.ptr(k), L.ptr(b), cout,
                                    1 if self.nd == 2 else 3, 1 if act == 'relu' else 0, L.ptr(out), L.stream_ptr()))
            return out
        (kz, ky, kx), (sz, sy, sx) = ((1,) + ks, (1,) + stride) if self.nd == 2 else (ks, stride)
        osp = tuple(-(-s // t) for s, t in zip(x.shape[1:-1], stride))
        out = torch.empty((n,) + osp + (cout,), dtype=torch.float32, device=x.device)
        L.check(lib.sdb_conv_any_nd(L.ptr(x), L.ptr(x_lo), n, d, h, w, c_skip, c_lo, int(uz), int(uy), int(ux), L.ptr(k), L.ptr(b), cout,
                                   kz, ky, kx, sz, sy, sx, 0 if keep_z else act_id(act), L.ptr(out), L.stream_ptr()))
        if keep_z:
            y = torch.empty_like(out)
            L.check(lib.sdb_act_any(L.ptr(out), out.numel(), act_id(act), L.ptr(y), L.stream_ptr()))
            return out, y
        return out

    def _class_branch(self, base, keep=False):
        """prob_class [N,...,n_classes+1] from the backbone output `base` (fp32, channels last), or None.  keep=True stores
        self.saved_class = (base, the prob_class layer's input, prob_class) for the backward pass, and in
        self.saved_class_z the pre-activation of features_class when its activation is neither ReLU nor linear."""
        if self.config.n_classes is None:
            return None
        lib = L.load()
        x, z = base, None
        if 'features_class' in self.w:
            act = self.config.unet_activation if getattr(self.config, 'backbone', 'unet') == 'unet' else self.config.resnet_activation
            if keep and keeps_preactivation(act):
                z, x = self._conv(base, None, 'features_class', act, (1,) * self.nd, keep_z=True)
            else:
                x = self._conv(base, None, 'features_class', act, (1,) * self.nd)
        wc, bc = self.w['prob_class']
        C = int(wc.shape[-1]); cf = int(x.shape[-1])
        npix = int(np.prod(x.shape[:-1]))
        out = torch.empty(tuple(x.shape[:-1]) + (C,), dtype=torch.float32, device=x.device)
        L.check(lib.sdb_class_head(L.ptr(x), npix, cf, L.ptr(wc.reshape(cf, C).contiguous()), L.ptr(bc), C, L.ptr(out), L.stream_ptr()))
        if keep:
            self.saved_class, self.saved_class_z = (base, x, out), z
        return out

    def _pool(self, x, pool):
        lib = L.load()
        n = x.shape[0]; d, h, w = self._dhw(x); c = x.shape[-1]
        pz, py, px = ((1,) + tuple(pool)) if len(pool) == 2 else tuple(pool)
        osp = (h // py, w // px) if self.nd == 2 else (d // pz, h // py, w // px)
        out = torch.empty((n,) + osp + (c,), dtype=torch.float32, device=x.device)
        fn = lib.sdb_maxpool_nd if maxpool_accepts(c) else lib.sdb_maxpool_any_nd
        L.check(fn(L.ptr(x), n, d, h, w, c, int(pz), int(py), int(px), L.ptr(out), L.stream_ptr()))
        return out

    def _heads(self, feat):
        lib = L.load()
        cf = feat.shape[-1]
        npix = int(np.prod(feat.shape[:-1]))
        R = self.config.n_rays
        (wp, bp), (wd, bd) = self.w['prob'], self.w['dist']
        prob = torch.empty(tuple(feat.shape[:-1]), dtype=torch.float32, device=feat.device)
        dist = torch.empty(tuple(feat.shape[:-1]) + (R,), dtype=torch.float32, device=feat.device)
        fn = lib.sdb_heads_2d if heads_accept(cf, R) else lib.sdb_heads_any
        L.check(fn(L.ptr(feat), npix, cf, L.ptr(wp), L.ptr(bp), L.ptr(wd), L.ptr(bd), R, L.ptr(prob), L.ptr(dist), L.stream_ptr()))
        return prob, dist

    def forward(self, x, keep=False):
        """x: float32 [N,(D,)H,W,Cin] on the device -> (prob [N,...], dist [N,...,R]).
        keep=True stores in self.saved, per entry of self.layers, what the backward pass reads: for a convolution its
        inputs (x, x_lo, up), its output y and, for activations other than ReLU / linear, its pre-activation z (the layer then
        runs linear and its activation as a separate pass, with the same y), for a pooling its input x; self.saved_feat is
        the heads' input and, for multi-class models, self.saved_class the class branch's (see _class_branch)."""
        assert x.dtype == torch.float32 and x.is_cuda and x.is_contiguous()
        skips = {}
        lo, up = None, (1,) * self.nd
        base = None
        saved = [None] * len(self.layers) if keep else None
        for i, l in enumerate(self.layers):
            kind = l['kind']
            if kind == 'conv':
                if l['name'] == 'features': base = x
                if keep and keeps_preactivation(l['act']):
                    z, y = self._conv(x, lo, l['name'], l['act'], up, keep_z=True)
                else:
                    z, y = None, self._conv(x, lo, l['name'], l['act'], up)
                if keep:
                    saved[i] = dict(x=x, lo=lo, up=up, y=y, z=z)
                x = y
                lo, up = None, (1,) * self.nd
            elif kind == 'pool':
                if 'save_skip' in l:
                    skips[l['save_skip']] = x
                if keep:
                    saved[i] = dict(x=x)
                x = self._pool(x, l['pool'])
            elif kind == 'up':
                lo, up = x, tuple(l['pool'])           # consumed by the next conv together with the skip
                x = skips.pop(l['skip'])
            elif kind == 'head':
                break
        feat = x
        if keep:
            self.saved, self.saved_feat = saved, feat
        prob, dist = self._heads(feat)
        self.prob_class = self._class_branch(feat if base is None else base, keep=keep)
        return prob, dist


UNetDevice2D = UNetDeviceND


class ResNetDeviceND(UNetDeviceND):
    """3-D ResNet backbone (stardist/models/model3d.py:402-447, csbdeep resnet_block) on the fp32 CUDA-core kernels:
    the stride-1 3^3 convolutions run on the tiled kernel of the U-Net path (sdb_conv3_nd), the 7^3 stem, the strided
    3^3 convolution that opens a pooling block and the strided 1^3 shortcut projection on the generic kernel
    (sdb_conv_generic_nd, TensorFlow 'same' padding), the residual sum on sdb_add_act.  Layers none of these accept
    (activations other than ReLU / linear, channel counts sdb_conv3_nd does not take) run on csrc/unet_any.cu."""

    def __init__(self, config, weights, device=None):
        self.layers = resnet_layers(config)
        check_activations(self.layers)
        L.require_cuda()
        self.config = config
        self.nd = config.n_dim
        self.device = torch.device("cuda") if device is None else torch.device(device)
        self._upload(weights)

    def _conv_layer(self, x, l):
        lib = L.load()
        k, b = self.w[l['name']]
        act = l['act']
        if tuple(l['k']) == (3, 3, 3) and tuple(l['stride']) == (1, 1, 1) and l['cin'] > 4:
            if conv3_accepts(3, l['k'], l['stride'], l['cin'], 0, l['cout'], act):
                return self._conv(x, None, l['name'], act, (1, 1, 1))
        elif conv_generic_accepts(act):
            n, d, h, w, cin = x.shape
            kz, ky, kx = l['k']; sz, sy, sx = l['stride']
            cout = k.shape[-1]
            out = torch.empty((n, -(-d // sz), -(-h // sy), -(-w // sx), cout), dtype=torch.float32, device=x.device)
            L.check(lib.sdb_conv_generic_nd(L.ptr(x), n, d, h, w, cin, L.ptr(k), L.ptr(b), cout, kz, ky, kx, sz, sy, sx,
                                           1 if act == 'relu' else 0, L.ptr(out), L.stream_ptr()))
            return out
        return self._conv(x, None, l['name'], act, (1, 1, 1), stride=l['stride'])

    def forward(self, x):
        lib = L.load()
        assert x.dtype == torch.float32 and x.is_cuda and x.is_contiguous() and x.dim() == 5
        block_in = shortcut = base = None
        for l in self.layers:
            kind = l['kind']
            if kind == 'block_begin':
                block_in, shortcut = x, None
            elif kind == 'conv':
                if l['name'] == 'features': base = x
                y = self._conv_layer(block_in if l['src'] == 'block_in' else x, l)
                if l['dst'] == 'shortcut': shortcut = y
                else: x = y
            elif kind == 'block_end':
                s = block_in if shortcut is None else shortcut
                assert s.shape == x.shape
                out = torch.empty_like(x)
                if add_act_accepts(l['act']):
                    L.check(lib.sdb_add_act(L.ptr(s), L.ptr(x), x.numel(), 1 if l['act'] == 'relu' else 0, L.ptr(out), L.stream_ptr()))
                else:
                    L.check(lib.sdb_add_act_any(L.ptr(s), L.ptr(x), x.numel(), act_id(l['act']), L.ptr(out), L.stream_ptr()))
                x, block_in, shortcut = out, None, None
            elif kind == 'head':
                break
        feat = x
        prob, dist = self._heads(feat)
        self.prob_class = self._class_branch(feat if base is None else base)
        return prob, dist


def tc_weight_scale(k):
    """power of two that brings max|w| into [1024, 2048): the fp16 'lo' parts of all but negligible
    weights then stay in the normal range (no precision loss), and products stay far from overflow"""
    m = float(np.max(np.abs(k)))
    if not np.isfinite(m) or m <= 0:
        return 1.0
    return float(2.0 ** (10 - int(np.floor(np.log2(m)))))


class UNetDevice2DTC:
    """wgmma / TMA executor (csrc/unet_tc.cu).  Activations are [2, N, H, W, C] float16
    tensors (plane 0 = hi, plane 1 = lo, value = hi + lo); convolutions run as three fp16 tensor-core
    passes with fp32 accumulation in registers.  The Cin<=4 stem, 2x2 max-pooling and the 1x1 heads are
    small CUDA-core kernels on the same split format; nearest up-sampling is written by the
    producing convolution's epilogue."""

    def __init__(self, config, weights, device=None):
        lib = L.require_cuda()
        self.config = config
        self.device = torch.device("cuda") if device is None else torch.device(device)
        self.layers = unet_layers(config)
        if config.unet_batch_norm:
            raise NotImplementedError("unet_batch_norm=True is not supported on this path")
        if tuple(config.unet_kernel_size) != (3, 3) or tuple(config.unet_pool) != (2, 2):
            raise NotImplementedError("only 3x3 kernels and 2x2 pooling are supported")
        self.w = {}
        self._simt = None
        self.prob_class = None
        for name, (k, b) in weights.items():
            kd = torch.from_numpy(np.ascontiguousarray(k, dtype=np.float32)).to(self.device)
            bd = torch.from_numpy(np.ascontiguousarray(b, dtype=np.float32)).to(self.device)
            ent = dict(k=kd, b=bd)
            if k.ndim == 4 and k.shape[0] == 3 and k.shape[2] % 32 == 0:
                cin, cout = k.shape[2], k.shape[3]
                ws = torch.empty((2, 9, cout, cin), dtype=torch.float16, device=self.device)
                ent['scale'] = tc_weight_scale(k)
                L.check(lib.sdb_split_weights(L.ptr(kd), cin, cout, ent['scale'], L.ptr(ws[0]), L.ptr(ws[1]), L.stream_ptr()))
                ent['split'] = ws
            self.w[name] = ent
        # 1x1 heads as one tensor-core GEMM: rows = [prob | dist_0..R-1 | zero padding], K = feature channels
        R = config.n_rays
        kp, kd = self.w['prob']['k'], self.w['dist']['k']
        cf = kp.shape[-2]
        self.heads_np = next((v for v in (48, 80, 112, 144) if v >= R + 1), None)
        if self.heads_np is not None and cf % 64 == 0:
            Wf = torch.zeros((self.heads_np, cf), dtype=torch.float32, device=self.device)
            Wf[0] = kp.reshape(cf, 1)[:, 0]
            Wf[1:R + 1] = kd.reshape(cf, R).t()
            sc = tc_weight_scale(Wf.cpu().numpy())
            Ws = Wf * sc
            hi = Ws.to(torch.float16)
            lo = (Ws - hi.float()).to(torch.float16)
            self.heads_w = torch.stack([hi, lo]).reshape(2, 1, self.heads_np, cf).contiguous()
            self.heads_scale = sc
            self.heads_b = torch.zeros(self.heads_np, dtype=torch.float32, device=self.device)
            self.heads_b[0] = self.w['prob']['b'][0]
            self.heads_b[1:R + 1] = self.w['dist']['b']
        else:
            self.heads_w = None
        # fused features+heads (sdb_conv3x3_heads_tc): fp32 head weights [cf][36], columns 0..R-1 dist, 32 prob
        self.fuse_heads = (R <= 32 and cf == 128 and os.environ.get("STARDIST_B200_FUSE_HEADS", "1") != "0")
        if self.fuse_heads:
            Wh = torch.zeros((cf, 36), dtype=torch.float32, device=self.device)
            Wh[:, :R] = kd.reshape(cf, R)
            Wh[:, 32] = kp.reshape(cf)
            bh = torch.zeros(36, dtype=torch.float32, device=self.device)
            bh[:R] = self.w['dist']['b']
            bh[32] = self.w['prob']['b'][0]
            self.fuse_w, self.fuse_b = Wh.contiguous(), bh

    def _class_branch_split(self, base_split):
        """multi-class branch of the tensor-core executor: the backbone output (split fp16 planes) is merged to fp32 and
        runs through the CUDA-core 3x3 convolution + softmax head (classification models only; not on the bench path)"""
        if self.config.n_classes is None:
            return None
        lib = L.load()
        if self._simt is None:
            self._simt = UNetDeviceND(self.config, {k: (v['k'].cpu().numpy(), v['b'].cpu().numpy()) for k, v in self.w.items()
                                                   if k in ('features_class', 'prob_class')})
        base = torch.empty(tuple(base_split.shape[1:]), dtype=torch.float32, device=base_split.device)
        L.check(lib.sdb_merge_split(L.ptr(base_split[0]), L.ptr(base_split[1]), base.numel(), L.ptr(base), L.stream_ptr()))
        return self._simt._class_branch(base)

    @staticmethod
    def supported(config):
        ch = [l['cin'] for l in unet_layers(config) if l['kind'] == 'conv'] + [l['cout'] for l in unet_layers(config) if l['kind'] == 'conv']
        first = next(l for l in unet_layers(config) if l['kind'] == 'conv')
        ok_first = first['cin'] <= 4 and first['cout'] in (32, 64)
        rest = [l for l in unet_layers(config) if l['kind'] == 'conv'][1:]
        ok_rest = all(l['cin'] % 32 == 0 and l['cout'] in (32, 64, 128, 256) for l in rest)
        # every pooling layer -- incl. the grid stem's, which follows config.grid and may be (2,1) / (1,2) -- must be 2x2:
        # sdb_maxpool_split pools both axes (anisotropic grids run on the generic CUDA-core executor)
        ok_pool = all(tuple(l['pool']) == (2, 2) for l in unet_layers(config) if l['kind'] == 'pool')
        return (ok_first and ok_rest and ok_pool and config.net_conv_after_unet == 128 and not config.unet_batch_norm
                and tuple(config.unet_kernel_size) == (3, 3) and tuple(config.unet_pool) == (2, 2))

    def _forward_tc(self, x):
        lib = L.load()
        assert x.dtype == torch.float32 and x.is_cuda and x.is_contiguous()
        st = L.stream_ptr()
        n, h, w, _ = x.shape
        layers = self.layers
        skips = {}
        lo = None          # (tensor [2,n,h,w,c]) up-sampled source waiting for its concat conv
        cur = None         # current activation (split)
        first = True
        for i, l in enumerate(layers):
            kind = l['kind']
            if kind == 'conv':
                relu = 1 if l['act'] == 'relu' else 0
                if l['act'] not in ('relu', 'linear'):
                    raise NotImplementedError("activation %s" % l['act'])
                nxt = layers[i + 1]['kind'] if i + 1 < len(layers) else None
                up2x = 1 if nxt == 'up' else 0
                ent = self.w[l['name']]
                cout = ent['k'].shape[-1]
                if first:
                    out = torch.empty((2, n, h, w, cout), dtype=torch.float16, device=x.device)
                    L.check(lib.sdb_stem_split(L.ptr(x), n, h, w, x.shape[-1], L.ptr(ent['k']), L.ptr(ent['b']), cout, relu,
                                               L.ptr(out[0]), L.ptr(out[1]), st))
                    first = False
                else:
                    _, n_, hh, ww, c1 = cur.shape
                    c0 = 0 if lo is None else lo.shape[-1]
                    oh, ow = (2 * hh, 2 * ww) if up2x else (hh, ww)
                    ws = ent['split']
                    if l['name'] == 'features':
                        self.prob_class = self._class_branch_split(cur) if lo is None else None
                    if self.fuse_heads and l['name'] == 'features' and c1 + c0 <= 64 and cout == 128:
                        R = self.config.n_rays
                        prob = torch.empty((n_, hh, ww), dtype=torch.float32, device=x.device)
                        dist = torch.empty((n_, hh, ww, R), dtype=torch.float32, device=x.device)
                        L.check(lib.sdb_conv3x3_heads_tc(L.ptr(lo[0]) if lo is not None else L.ptr(None), L.ptr(lo[1]) if lo is not None else L.ptr(None), c0,
                                                         L.ptr(cur[0]), L.ptr(cur[1]), c1, n_, hh, ww, L.ptr(ws[0]), L.ptr(ws[1]), ent['scale'], L.ptr(ent['b']),
                                                         relu, L.ptr(self.fuse_w), L.ptr(self.fuse_b), R, L.ptr(prob), L.ptr(dist), st))
                        L.check(lib.sdb_tc_error_check(st))
                        return prob, dist
                    out = torch.empty((2, n_, oh, ow, cout), dtype=torch.float16, device=x.device)
                    L.check(lib.sdb_conv3x3_tc(L.ptr(lo[0]) if lo is not None else L.ptr(None), L.ptr(lo[1]) if lo is not None else L.ptr(None), c0,
                                               L.ptr(cur[0]), L.ptr(cur[1]), c1, n_, hh, ww, L.ptr(ws[0]), L.ptr(ws[1]), ent['scale'], L.ptr(ent['b']),
                                               cout, relu, up2x, L.ptr(out[0]), L.ptr(out[1]), st))
                    lo = None
                cur = out
            elif kind == 'pool':
                if 'save_skip' in l:
                    skips[l['save_skip']] = cur
                _, n_, hh, ww, c = cur.shape
                out = torch.empty((2, n_, hh // 2, ww // 2, c), dtype=torch.float16, device=x.device)
                L.check(lib.sdb_maxpool_split(L.ptr(cur[0]), L.ptr(cur[1]), n_, hh, ww, c, L.ptr(out[0]), L.ptr(out[1]), st))
                cur = out
            elif kind == 'up':
                lo = cur                        # already written at 2x resolution by its producer
                cur = skips.pop(l['skip'])
                assert lo.shape[2] == cur.shape[2] and lo.shape[3] == cur.shape[3]
            elif kind == 'head':
                break
        _, n_, hh, ww, cf = cur.shape
        R = self.config.n_rays
        prob = torch.empty((n_, hh, ww), dtype=torch.float32, device=x.device)
        dist = torch.empty((n_, hh, ww, R), dtype=torch.float32, device=x.device)
        if self.heads_w is not None:
            L.check(lib.sdb_heads_tc(L.ptr(cur[0]), L.ptr(cur[1]), cf, n_, hh, ww, L.ptr(self.heads_w[0]), L.ptr(self.heads_w[1]),
                                    self.heads_scale, L.ptr(self.heads_b), self.heads_np, R, L.ptr(prob), L.ptr(dist), st))
        else:
            L.check(lib.sdb_heads_split(L.ptr(cur[0]), L.ptr(cur[1]), n_ * hh * ww, cf, L.ptr(self.w['prob']['k']), L.ptr(self.w['prob']['b']),
                                       L.ptr(self.w['dist']['k']), L.ptr(self.w['dist']['b']), R, L.ptr(prob), L.ptr(dist), st))
        L.check(lib.sdb_tc_error_check(st))
        return prob, dist


class UNetDevice3DTC:
    """tensor-core executor of the 3-D U-Net (model3d.py:360-399) for ONE volume: activations are [2, D, H, W, C] float16
    planes (hi, lo); every 3x3x3 convolution with Cin % 32 == 0 runs on sdb_conv3x3x3_tc (k_conv_wg: z planes as the
    tensor map's image axis, 27 taps), the Cin <= 4 stem on the CUDA-core kernel followed by sdb_split_f32, pooling on
    sdb_maxpool3d_split, nearest 2x2x2 up-sampling written by the producing convolution, the 1x1x1 heads on the
    tensor-core heads kernel over the volume viewed as a [D*H, W] image."""

    def __init__(self, config, weights, device=None):
        lib = L.require_cuda()
        self.config = config
        self.device = torch.device("cuda") if device is None else torch.device(device)
        self.layers = unet_layers(config)
        self.prob_class = None
        self._simt = UNetDeviceND(config, weights, device=self.device)       # stem conv, class branch
        self.w = {}
        for name, (k, b) in weights.items():
            kd = torch.from_numpy(np.ascontiguousarray(k, dtype=np.float32)).to(self.device)
            bd = torch.from_numpy(np.ascontiguousarray(b, dtype=np.float32)).to(self.device)
            ent = dict(k=kd, b=bd)
            if k.ndim == 5 and k.shape[0] == 3 and k.shape[3] % 32 == 0:
                cin, cout = k.shape[3], k.shape[4]
                ws = torch.empty((2, 27, cout, cin), dtype=torch.float16, device=self.device)
                ent['scale'] = tc_weight_scale(k)
                L.check(lib.sdb_split_weights_3d(L.ptr(kd), cin, cout, ent['scale'], L.ptr(ws[0]), L.ptr(ws[1]), L.stream_ptr()))
                ent['split'] = ws
            self.w[name] = ent
        R = config.n_rays
        kp, kd = self.w['prob']['k'], self.w['dist']['k']
        cf = kp.shape[-2]
        self.heads_np = next(v for v in (48, 80, 112, 144) if v >= R + 1)
        Wf = torch.zeros((self.heads_np, cf), dtype=torch.float32, device=self.device)
        Wf[0] = kp.reshape(cf, 1)[:, 0]
        Wf[1:R + 1] = kd.reshape(cf, R).t()
        sc = tc_weight_scale(Wf.cpu().numpy())
        Ws = Wf * sc
        hi = Ws.to(torch.float16)
        lo = (Ws - hi.float()).to(torch.float16)
        self.heads_w = torch.stack([hi, lo]).reshape(2, 1, self.heads_np, cf).contiguous()
        self.heads_scale = sc
        self.heads_b = torch.zeros(self.heads_np, dtype=torch.float32, device=self.device)
        self.heads_b[0] = self.w['prob']['b'][0]
        self.heads_b[1:R + 1] = self.w['dist']['b']

    @staticmethod
    def supported(config):
        if config.n_dim != 3 or getattr(config, 'backbone', 'unet') != 'unet' or config.unet_batch_norm:
            return False
        convs = [l for l in unet_layers(config) if l['kind'] == 'conv']
        ok_first = convs[0]['cin'] <= 4 and convs[0]['cout'] % 32 == 0
        ok_rest = all(l['cin'] % 32 == 0 and l.get('cin_lo', 0) % 32 == 0 and l['cout'] in (32, 64, 128) for l in convs[1:])
        return (ok_first and ok_rest and tuple(config.unet_kernel_size) == (3, 3, 3) and tuple(config.unet_pool) == (2, 2, 2)
                and config.net_conv_after_unet % 64 == 0 and config.net_conv_after_unet > 0 and config.n_rays + 1 <= 144
                and config.unet_activation in ('relu', 'linear') and config.unet_last_activation in ('relu', 'linear'))

    def _forward_tc(self, x, stop_before_features=False):
        lib = L.load()
        assert x.dtype == torch.float32 and x.is_cuda and x.is_contiguous() and x.dim() == 5
        if x.shape[0] != 1:
            raise NotImplementedError("the 3-D tensor-core executor takes one volume per call")
        st = L.stream_ptr()
        layers = self.layers
        skips = {}
        lo = None
        cur = None
        base = None
        first = True
        for i, l in enumerate(layers):
            kind = l['kind']
            if kind == 'conv':
                relu = 1 if l['act'] == 'relu' else 0
                nxt = layers[i + 1]['kind'] if i + 1 < len(layers) else None
                up2x = 2 if nxt == 'up' else 0
                ent = self.w[l['name']]
                cout = ent['k'].shape[-1]
                if first:
                    y = self._simt._conv(x, None, l['name'], l['act'], (1, 1, 1))          # [1,D,H,W,cout] fp32
                    out = torch.empty((2,) + tuple(y.shape[1:]), dtype=torch.float16, device=x.device)
                    L.check(lib.sdb_split_f32(L.ptr(y), y.numel(), L.ptr(out[0]), L.ptr(out[1]), st))
                    first = False
                else:
                    _, d, h, w, c1 = cur.shape
                    c0 = 0 if lo is None else lo.shape[-1]
                    od, oh, ow = (2 * d, 2 * h, 2 * w) if up2x else (d, h, w)
                    if l['name'] == 'features':
                        base = cur
                        if stop_before_features and lo is None:
                            return cur, ent, relu                      # forward_candidates runs features + heads slab by slab
                    out = torch.empty((2, od, oh, ow, cout), dtype=torch.float16, device=x.device)
                    ws = ent['split']
                    L.check(lib.sdb_conv3x3x3_tc(L.ptr(lo[0]) if lo is not None else L.ptr(None), L.ptr(lo[1]) if lo is not None else L.ptr(None), c0,
                                                 L.ptr(cur[0]), L.ptr(cur[1]), c1, d, h, w, L.ptr(ws[0]), L.ptr(ws[1]), ent['scale'], L.ptr(ent['b']),
                                                 cout, relu, up2x, L.ptr(out[0]), L.ptr(out[1]), st))
                    lo = None
                cur = out
            elif kind == 'pool':
                if 'save_skip' in l:
                    skips[l['save_skip']] = cur
                _, d, h, w, c = cur.shape
                pz, py, px = (int(v) for v in l['pool'])
                out = torch.empty((2, d // pz, h // py, w // px, c), dtype=torch.float16, device=x.device)
                L.check(lib.sdb_maxpool3d_split(L.ptr(cur[0]), L.ptr(cur[1]), d, h, w, c, pz, py, px, L.ptr(out[0]), L.ptr(out[1]), st))
                cur = out
            elif kind == 'up':
                lo = cur
                cur = skips.pop(l['skip'])
                assert tuple(lo.shape[1:4]) == tuple(cur.shape[1:4])
            elif kind == 'head':
                break
        _, d, h, w, cf = cur.shape
        R = self.config.n_rays
        prob = torch.empty((1, d, h, w), dtype=torch.float32, device=x.device)
        dist = torch.empty((1, d, h, w, R), dtype=torch.float32, device=x.device)
        L.check(lib.sdb_heads_tc(L.ptr(cur[0]), L.ptr(cur[1]), cf, 1, d * h, w, L.ptr(self.heads_w[0]), L.ptr(self.heads_w[1]),
                                self.heads_scale, L.ptr(self.heads_b), self.heads_np, R, L.ptr(prob), L.ptr(dist), st))
        L.check(lib.sdb_tc_error_check(st))
        self.prob_class = None
        if self.config.n_classes is not None:
            b32 = torch.empty((1,) + tuple(base.shape[1:]), dtype=torch.float32, device=x.device)
            L.check(lib.sdb_merge_split(L.ptr(base[0]), L.ptr(base[1]), b32.numel(), L.ptr(b32), st))
            self.prob_class = self._simt._class_branch(b32)
        return prob, dist

    def forward_candidates(self, x, prob_thresh, slab=16):
        """Sparse forward pass for large volumes (SURVEY H7, the reference's own per-tile sparse gather base.py:580-593):
        the 128-channel `features` map (17 GB at 128x512x512) and the dense dist map (12.9 GB) are never materialised.
        The last two layers run over z-slabs of `slab` planes (+1 halo plane each side for the 3x3x3 convolution); of every
        slab only the prob planes (into the full prob map) and the dist rows of voxels with prob > prob_thresh (into a compact
        store) survive.  Returns (prob [1,D,H,W], store [n_rows,R] float32, slot int32[D*H*W]) with store[slot[flat]] =
        dist row of voxel `flat` for every voxel above the threshold; values are those of forward() (same kernels)."""
        import ctypes
        lib = L.load()
        st = L.stream_ptr()
        r = self._forward_tc(x, stop_before_features=True)
        if not (isinstance(r, tuple) and len(r) == 3 and isinstance(r[1], dict)):
            raise NotImplementedError("forward_candidates: architecture without a plain `features` layer")
        cur, ent, relu = r
        _, D, H, W, c1 = cur.shape
        R = self.config.n_rays
        cf = int(ent['k'].shape[-1])
        ws = ent['split']
        dev = x.device
        prob = torch.empty((1, D, H, W), dtype=torch.float32, device=dev)
        slot = torch.empty(D * H * W, dtype=torch.int32, device=dev)
        thr = float(np.float32(prob_thresh))
        stores, rows = [], 0
        plane = H * W
        feat = torch.empty((2, min(D, slab + 2), H, W, cf), dtype=torch.float16, device=dev)
        dist_slab = torch.empty((min(D, slab), H, W, R), dtype=torch.float32, device=dev)
        for z0 in range(0, D, slab):
            s = min(slab, D - z0)
            za, zb = max(0, z0 - 1), min(D, z0 + s + 1)
            sd = zb - za
            f = feat[:, :sd]
            if sd != feat.shape[1]:
                f = torch.empty((2, sd, H, W, cf), dtype=torch.float16, device=dev)
            L.check(lib.sdb_conv3x3x3_tc(L.ptr(None), L.ptr(None), 0, L.ptr(cur[0, za:zb]), L.ptr(cur[1, za:zb]), c1, sd, H, W,
                                         L.ptr(ws[0]), L.ptr(ws[1]), ent['scale'], L.ptr(ent['b']), cf, relu, 0, L.ptr(f[0]), L.ptr(f[1]), st))
            o = z0 - za
            pslab = prob[0, z0:z0 + s]
            L.check(lib.sdb_heads_tc(L.ptr(f[0, o:o + s]), L.ptr(f[1, o:o + s]), cf, 1, s * H, W, L.ptr(self.heads_w[0]), L.ptr(self.heads_w[1]),
                                    self.heads_scale, L.ptr(self.heads_b), self.heads_np, R, L.ptr(pslab), L.ptr(dist_slab), st))
            cnt = ctypes.c_int(0)
            L.check(lib.sdb_count_above(L.ptr(pslab), s * plane, thr, ctypes.byref(cnt), st))
            n = int(cnt.value)
            if n > 0:
                store = torch.empty((n, R), dtype=torch.float32, device=dev)
                L.check(lib.sdb_store_rows_above(L.ptr(pslab), L.ptr(dist_slab), s * plane, R, thr, z0 * plane, rows, n, L.ptr(store), L.ptr(slot), st))
                # rows of this slab are numbered from `rows` in the concatenated store; the kernel numbers them from 0
                stores.append(store)
                rows += n
        L.check(lib.sdb_tc_error_check(st))
        self.prob_class = None
        store = torch.cat(stores) if stores else torch.empty((0, R), dtype=torch.float32, device=dev)
        return prob, store, slot


def _forward_guarded(self, x):
    """tensor-core forward pass; if an activation left the fp16 range of the split representation (|v| > 65504: raw
    16-bit images, un-normalised floats -- the reference only warns about those, base.py:414) the pass is repeated on the
    exact-fp32 CUDA-core executor, which has float32's range like the reference network"""
    try:
        return self._forward_tc(x)
    except L.StarDistB200Error as e:
        if 'fp16 overflow' not in str(e):
            raise
    import warnings
    warnings.warn("stardist_b200: activations exceed the fp16 range of the tensor-core path (un-normalised input?); "
                  "running this prediction on the fp32 CUDA-core kernels instead")
    if getattr(self, '_fp32', None) is None:
        self._fp32 = UNetDeviceND(self.config, {k: (v['k'].cpu().numpy(), v['b'].cpu().numpy()) for k, v in self.w.items()})
    out = self._fp32.forward(x)
    self.prob_class = self._fp32.prob_class
    return out


UNetDevice2DTC.forward = _forward_guarded
UNetDevice3DTC.forward = _forward_guarded
