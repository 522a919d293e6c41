"""Training of the StarDist U-Net on the device: loss, backward pass and Adam (csrc/unet_train.cu) behind
StarDist2D.train / StarDist3D.train.

Reference: stardist/models/model2d.py:352-481 / model3d.py `train`, the losses of stardist/models/base.py:34-50,
:108-126 (the multi-class cross-entropy) and :315-347, Keras' Adam, ReduceLROnPlateau and csbdeep's checkpointing
(restated on the host below).  The forward pass is UNetDeviceND's (exact fp32 CUDA cores) with its activations kept; DESIGN.md 4.2 states the data flow and the loss.
Under the 'mixed_bfloat16' policy of stardist_b200.mixed_precision the trainer runs its own forward pass and every
convolution, head and gradient between layers on the bf16 tensor-core kernels of csrc/unet_train_bf16.cu instead.
"""
import warnings
import numpy as np

from .. import _lib as L
from ..utils import _raise

ADAM_BETA_1, ADAM_BETA_2, ADAM_EPSILON = 0.9, 0.999, 1e-7     # tf.keras.optimizers.Adam defaults

_tensor_float_32 = False


def enable_tensor_float_32_execution(enabled):
    """TensorFlow's tf.config.experimental.enable_tensor_float_32_execution for training: when on, the weight gradients of the
    1^d / 3^d / (1, 3, 3) convolutions and the input gradients of the 3^d ones run on the TF32 tensor cores (operands rounded to
    10 mantissa bits, fp32 accumulation; DESIGN.md 4.2).  Off by default, unlike TensorFlow: the backward pass is then exact
    fp32.  The forward pass, the loss and prediction never change.  A UNetTrainer (and so train()) reads the switch once,
    when it is constructed."""
    global _tensor_float_32
    _tensor_float_32 = bool(enabled)


def tensor_float_32_execution_enabled():
    """whether trainers constructed from now on run their convolution gradients in TF32"""
    return _tensor_float_32


def check_trainable(config, optimizer=None, policy=None):
    """NotImplementedError for every setting this trainer does not cover under `policy` (default: the global mixed-precision
    policy); runs before anything touches the device"""
    if getattr(config, 'backbone', 'unet') != 'unet':
        raise NotImplementedError("training of the '%s' backbone is not supported (U-Net only)" % config.backbone)
    if config.train_dist_loss not in ('mae', 'mse'):
        raise NotImplementedError("train_dist_loss=%r is not supported ('mae' or 'mse')" % config.train_dist_loss)
    if getattr(config, 'train_shape_completion', False):
        raise NotImplementedError("train_shape_completion=True is not supported")
    if getattr(config, 'unet_batch_norm', False):
        raise NotImplementedError("unet_batch_norm=True is not supported")
    if optimizer is not None:
        raise NotImplementedError("optimizer=%r: only the default Adam(train_learning_rate) is supported" % (optimizer,))
    ks = tuple(int(v) for v in config.unet_kernel_size)
    if len(ks) != config.n_dim or not all(1 <= v <= 7 for v in ks):
        raise NotImplementedError("unet_kernel_size=%r: kernel extents 1..7 per axis are supported" % (ks,))
    from .unet_device import act_id
    for a in (config.unet_activation, config.unet_last_activation):
        act_id(a)
    if getattr(config, 'n_classes', None) is not None:
        from .weights import unet_layers
        if config.n_classes + 1 > 32:
            raise NotImplementedError("n_classes=%d: multi-class training supports n_classes + 1 <= 32" % config.n_classes)
        for l in unet_layers(config):
            if l['kind'] == 'conv_class' and l['cin'] % 32:
                raise NotImplementedError("layer %s: %d input channels; the input gradient needs a multiple of 32" % (l['name'], l['cin']))
    from ..mixed_precision import global_policy
    if (global_policy() if policy is None else policy).name == 'mixed_bfloat16':
        check_bf16(config)


def check_bf16(config):
    """NotImplementedError naming the first layer the mixed_bfloat16 kernels do not take (unet_device.conv_bf16_accepts)"""
    from .unet_device import conv_bf16_accepts
    from .weights import unet_layers
    for l in unet_layers(config):
        if l['kind'] in ('conv', 'conv_class'):
            lo = l.get('cin_lo', 0)
            if not conv_bf16_accepts(config.n_dim, l['k'], l['cin'] - lo, lo, l['cout'], l['act']):
                raise NotImplementedError(
                    "policy 'mixed_bfloat16': layer %s (kernel %s, %d -> %d channels, activation %r) is outside the bf16 family: "
                    "kernels 1^d, 3^d or (1, 3, 3), ReLU or linear, output channels a multiple of 32, input channels <= 4 (stem) "
                    "or a multiple of 8" % (l['name'], tuple(l['k']), l['cin'], l['cout'], l['act']))


def adam_coef(n):
    """float32 [n]: sqrt(1 - beta2^t) / (1 - beta1^t) for t = 1..n, in float32 on the host"""
    t = np.arange(1, n + 1, dtype=np.float32)
    one = np.float32(1)
    return (np.sqrt(one - np.float32(ADAM_BETA_2) ** t) / (one - np.float32(ADAM_BETA_1) ** t)).astype(np.float32)


class UNetTrainer:
    """Device parameters (one flat float32 buffer), Adam's m and v, the forward activations and the backward buffers of
    one U-Net.  step() runs forward, loss, backward and Adam without reading anything back to the host."""

    bf16 = False        # set from the mixed-precision policy at construction

    def __init__(self, config, weights, learning_rate=None):
        import torch
        from .unet_device import UNetDeviceND
        from ..mixed_precision import global_policy
        self.policy = global_policy()
        self.bf16 = self.policy.name == 'mixed_bfloat16'
        check_trainable(config, policy=self.policy)
        lib = L.require_cuda()
        self.tf32 = tensor_float_32_execution_enabled() and not self.bf16
        self.config, self.nd = config, config.n_dim
        self.net = UNetDeviceND(config, weights)
        self.layers = self.net.layers
        self.names = [l['name'] for l in self.layers if l['kind'] in ('conv', 'head', 'conv_class', 'head_class')]
        self.n_classes = config.n_classes
        self.shapes = {n: (tuple(np.shape(weights[n][0])), tuple(np.shape(weights[n][1]))) for n in self.names}
        # offset of every layer in the flat buffer, in layer order.  The 1-float prob and R-float dist biases leave the
        # offsets after them unaligned; the class layers that follow start at a multiple of 32 floats, because the forward
        # convolution loads its weights as float4.  The gaps hold zeros with zero gradients, which Adam leaves at zero.
        self.offsets, off = {}, 0
        for n in self.names:
            if n in ('features_class', 'prob_class'):
                off = -(-off // 32) * 32
            self.offsets[n] = off
            off += int(np.prod(self.shapes[n][0])) + int(np.prod(self.shapes[n][1]))
        total = off
        dev = self.net.device
        self.params = (torch.zeros if self.n_classes is not None else torch.empty)(total, dtype=torch.float32, device=dev)
        self.grad = torch.zeros(total, dtype=torch.float32, device=dev)
        self.m = torch.zeros(total, dtype=torch.float32, device=dev)
        self.v = torch.zeros(total, dtype=torch.float32, device=dev)
        self.pview, self.gview = {}, {}
        for n in self.names:
            ks, bs = self.shapes[n]
            nk, nb = int(np.prod(ks)), int(np.prod(bs))
            off = self.offsets[n]
            self.pview[n] = (self.params[off:off + nk].view(ks), self.params[off + nk:off + nk + nb].view(bs))
            self.gview[n] = (self.grad[off:off + nk].view(ks), self.grad[off + nk:off + nk + nb].view(bs))
            self.pview[n][0].copy_(torch.from_numpy(np.ascontiguousarray(weights[n][0], np.float32)))
            self.pview[n][1].copy_(torch.from_numpy(np.ascontiguousarray(weights[n][1], np.float32)))
        self.net.w = dict(self.pview)            # the forward pass reads the trained parameters in place
        self.lr = np.float32(config.train_learning_rate if learning_rate is None else learning_rate)
        self.state = torch.zeros(3, dtype=torch.int32, device=dev)        # (t, skipped steps, last step skipped)
        self.coef = torch.empty(0, dtype=torch.float32, device=dev)
        self.n_calls = 0
        self._bufs = {}
        if self.n_classes is not None:
            self.class_w = torch.from_numpy(np.asarray(config.train_class_weights, np.float32)).to(dev)

    # ---------------------------------------------------------------------------------------------- buffers
    def _buf(self, key, shape, zero=False, bf16=False):
        import torch
        b = self._bufs.get(key)
        if b is None or tuple(b.shape) != tuple(shape):
            b = (torch.zeros if zero else torch.empty)(tuple(shape), dtype=torch.bfloat16 if bf16 else torch.float32,
                                                       device=self.net.device)
            self._bufs[key] = b
        return b

    def _workspace(self, floats):
        b = self._bufs.get('work')
        if b is None or b.numel() < floats:
            b = self._buf('work', (int(floats),))
        return b

    @staticmethod
    def _dhw(t):
        return (1,) + tuple(t.shape[1:3]) if t.dim() == 4 else tuple(t.shape[1:4])

    # ---------------------------------------------------------------------------------------------- kernels
    def _wgrad(self, x, lo, up, k, dy, ldy, cout, dw, db):
        """weight and bias gradient of a stride-1 'same' convolution with kernel extents k over the input [upsample(lo), x]"""
        from .unet_device import conv_wgrad_accepts
        lib = L.load()
        n = x.shape[0]; d, h, w = self._dhw(x)
        c_skip = x.shape[-1]; c_lo = 0 if lo is None else lo.shape[-1]
        kz, ky, kx = ((1,) + tuple(k)) if self.nd == 2 else tuple(k)
        uz, uy, ux = ((1,) + tuple(up)) if len(up) == 2 else tuple(up)
        need = int(lib.sdb_conv_wgrad_workspace(n * d * h * w, kz * ky * kx, c_skip + c_lo, cout))
        work = self._workspace(need)
        if self.bf16:
            import torch
            L.check(lib.sdb_conv_wgrad_bf16_nd(L.ptr(x), L.ptr(lo), n, d, h, w, c_skip, c_lo, int(uz), int(uy), int(ux), kz, ky, L.ptr(dy),
                                               1 if dy.dtype == torch.bfloat16 else 0, ldy, cout, L.ptr(work), work.numel(), L.ptr(dw),
                                               L.ptr(db), L.stream_ptr()))
        elif conv_wgrad_accepts(self.nd, k):
            wgrad = lib.sdb_conv_wgrad_tf32_nd if self.tf32 else lib.sdb_conv_wgrad_nd
            L.check(wgrad(L.ptr(x), L.ptr(lo), n, d, h, w, c_skip, c_lo, int(uz), int(uy), int(ux), kz, ky, L.ptr(dy), ldy,
                          cout, L.ptr(work), work.numel(), L.ptr(dw), L.ptr(db), L.stream_ptr()))
        else:
            L.check(lib.sdb_conv_wgrad_any_nd(L.ptr(x), L.ptr(lo), n, d, h, w, c_skip, c_lo, int(uz), int(uy), int(ux), kz, ky, kx, L.ptr(dy),
                                              ldy, cout, L.ptr(work), work.numel(), L.ptr(dw), L.ptr(db), L.stream_ptr()))

    def _loss(self, prob, dist, prob_t, dam, dhead, out, state):
        lib = L.load()
        c = self.config
        npix = prob.numel(); R = c.n_rays
        assert prob_t.numel() == npix and dam.numel() == npix * (R + 1) and dist.numel() == npix * R
        work = self._buf('loss_work', (int(lib.sdb_stardist_loss_workspace(npix)) // 4,))
        stats = self._buf('loss_stats', (2,))
        w0, w1 = (float(v) for v in c.train_loss_weights[:2])
        prob_t, dam = prob_t.contiguous(), dam.contiguous()
        L.check(lib.sdb_stardist_loss(L.ptr(prob), L.ptr(dist), L.ptr(prob_t), L.ptr(dam), npix, R,
                                      1 if c.train_dist_loss == 'mae' else 0, float(c.train_background_reg), w0, w1, L.ptr(work),
                                      L.ptr(stats), L.ptr(dhead), L.ptr(out), L.ptr(state), L.stream_ptr()))

    def _class_loss(self, s, pc_t, dclass, out):
        """out[4] = the class loss, out[0] += w2 * it; dclass (or None) = dL/d(prob_class logits)"""
        lib = L.load()
        C = self.n_classes + 1
        npix = s.numel() // C
        pc_t = pc_t.contiguous()
        assert pc_t.numel() == s.numel(), (tuple(pc_t.shape), tuple(s.shape))
        work = self._buf('class_loss_work', (int(lib.sdb_stardist_class_loss_workspace(npix)) // 4,))
        L.check(lib.sdb_stardist_class_loss(L.ptr(s), L.ptr(pc_t), npix, C, L.ptr(self.class_w), float(self.config.train_loss_weights[2]),
                                            L.ptr(work), L.ptr(dclass), L.ptr(out[0:1]), L.ptr(out[4:5]), L.stream_ptr()))

    def _dgrad(self, key, name, g, x_shape, cin, cout, k):
        """input gradient of the stride-1 convolution `name` (kernel extents k, x_shape [..., cin] -> cout): the correlation of g
        with the flipped kernel, on sdb_conv3_nd (sdb_conv_dgrad_tf32_nd in TF32 mode) where conv_dgrad3_accepts takes the layer,
        else on sdb_conv_dgrad_any_nd"""
        from .unet_device import conv_dgrad3_accepts
        lib = L.load()
        st = L.stream_ptr()
        taps = int(np.prod(k))
        if self.bf16:
            kz, ky, kx = ((1,) + tuple(k)) if self.nd == 2 else tuple(k)
            n = x_shape[0]; d, h, w = (1,) + tuple(x_shape[1:3]) if len(x_shape) == 4 else tuple(x_shape[1:4])
            wfb = self._buf(('wflip_bf16', key), (taps * cout * cin,), bf16=True)
            L.check(lib.sdb_weights_bf16(L.ptr(self.pview[name][0]), taps, cin, cout, 1, cout, L.ptr(wfb), st))
            gin = self._buf(('gin', key), tuple(x_shape[:-1]) + (cin,), bf16=True)
            L.check(lib.sdb_conv_bf16_nd(L.ptr(g), None, n, d, h, w, cout, 0, 1, 1, 1, kz, ky, kx, L.ptr(wfb), None, cin, 0, 0,
                                         L.ptr(gin), st))
            return gin
        wf = self._buf(('wflip', key), (taps, cout, cin))
        L.check(lib.sdb_conv_flip_weights(L.ptr(self.pview[name][0]), taps, cin, cout, L.ptr(wf), st))
        n = x_shape[0]; d, h, w = (1,) + tuple(x_shape[1:3]) if len(x_shape) == 4 else tuple(x_shape[1:4])
        gin = self._buf(('gin', key), tuple(x_shape[:-1]) + (cin,))
        if conv_dgrad3_accepts(self.nd, k, cin, cout) and self.tf32:
            L.check(lib.sdb_conv_dgrad_tf32_nd(L.ptr(g), n, d, h, w, cout, L.ptr(wf), cin, 1 if self.nd == 2 else 3, 3, L.ptr(gin), st))
        elif conv_dgrad3_accepts(self.nd, k, cin, cout):
            zb = self._buf(('zero_bias', cin), (cin,), zero=True)
            L.check(lib.sdb_conv3_nd(L.ptr(g), None, n, d, h, w, cout, 0, 1, 1, 1, L.ptr(wf), L.ptr(zb), cin,
                                     1 if self.nd == 2 else 3, 0, L.ptr(gin), st))
        else:
            kz, ky, kx = ((1,) + tuple(k)) if self.nd == 2 else tuple(k)
            L.check(lib.sdb_conv_dgrad_any_nd(L.ptr(g), n, d, h, w, cout, L.ptr(wf), cin, kz, ky, kx, L.ptr(gin), st))
        return gin

    def _act_backward(self, g, act, y, z):
        """g *= act'(pre-activation) in place: from the output y for ReLU, from the kept pre-activation z for the activations
        other than ReLU / linear"""
        lib = L.load()
        if act == 'relu' and self.bf16:
            L.check(lib.sdb_relu_backward_bf16(L.ptr(g), L.ptr(y), g.numel(), L.stream_ptr()))
        elif act == 'relu':
            L.check(lib.sdb_relu_backward(L.ptr(g), L.ptr(y), g.numel(), L.stream_ptr()))
        elif act != 'linear':
            from .unet_device import act_id
            L.check(lib.sdb_act_backward(L.ptr(g), L.ptr(z), g.numel(), act_id(act), L.stream_ptr()))

    def _class_backward(self, dclass, g):
        """the class branch's parameter gradients from dclass = dL/d(softmax logits) per output pixel.  Returns the input
        gradient of features_class (the caller adds it to the features layer's), or None when there is no features_class: the
        prob_class layer then reads the heads' input, and its share is added to g, the heads' input gradient."""
        lib = L.load()
        st = L.stream_ptr()
        base, xc, _ = self.net.saved_class
        C = self.n_classes + 1
        cf = xc.shape[-1]; npix = xc.numel() // cf
        ones = (1,) * self.nd
        self._wgrad(xc, None, ones, ones, dclass, C, C, *self.gview['prob_class'])
        wc = self.pview['prob_class'][0]
        if self.bf16:
            wcb = self._buf('wclass_bwd_bf16', (cf * C,), bf16=True)
            L.check(lib.sdb_weights_bf16(L.ptr(wc), 1, cf, C, 1, C, L.ptr(wcb), st))
        if 'features_class' not in self.pview:
            if self.bf16:
                L.check(lib.sdb_gemm_bf16_f32in(L.ptr(dclass), npix, C, L.ptr(wcb), cf, 1, L.ptr(g), st))
            else:
                L.check(lib.sdb_class_head_backward(L.ptr(xc), L.ptr(dclass), npix, cf, L.ptr(wc), C, 0, 1, L.ptr(g), st))
            return None
        gc = self._buf('dfeat_class', xc.shape, bf16=self.bf16)
        act = self.config.unet_activation
        if self.bf16:
            L.check(lib.sdb_gemm_bf16_f32in(L.ptr(dclass), npix, C, L.ptr(wcb), cf, 0, L.ptr(gc), st))
            self._act_backward(gc, act, xc, None)
        else:
            L.check(lib.sdb_class_head_backward(L.ptr(xc), L.ptr(dclass), npix, cf, L.ptr(wc), C, 1 if act == 'relu' else 0, 0, L.ptr(gc), st))
        if act != 'relu' and not self.bf16:
            self._act_backward(gc, act, xc, self.net.saved_class_z)
        k = tuple(self.pview['features_class'][0].shape[:self.nd])
        self._wgrad(base, None, ones, k, gc, cf, cf, *self.gview['features_class'])
        return self._dgrad('class', 'features_class', gc, base.shape, base.shape[-1], cf, k)

    def _backward(self, dhead, dclass=None):
        """gradient of every parameter into self.grad from dhead = (dL/d prob logit, dL/d dist) and, for multi-class models,
        dclass = dL/d(prob_class logits) per output pixel"""
        import torch
        lib = L.load()
        st = L.stream_ptr()
        net, R = self.net, self.config.n_rays
        feat = net.saved_feat
        cf = feat.shape[-1]; npix = feat.numel() // cf
        ones = (1,) * self.nd
        dh = dhead.view(-1)
        self._wgrad(feat, None, ones, ones, dh, R + 1, 1, *self.gview['prob'])
        self._wgrad(feat, None, ones, ones, dh[1:], R + 1, R, *self.gview['dist'])
        g = self._buf('dfeat', feat.shape, bf16=self.bf16)
        if self.bf16:
            whb = self._buf('wheads_bwd_bf16', (cf * (R + 1),), bf16=True)
            L.check(lib.sdb_weights_bf16(L.ptr(self.pview['prob'][0]), 1, cf, 1, 1, R + 1, L.ptr(whb), st))
            L.check(lib.sdb_weights_bf16(L.ptr(self.pview['dist'][0]), 1, cf, R, 1, R + 1, L.ptr(whb[1:]), st))
            L.check(lib.sdb_gemm_bf16_f32in(L.ptr(dhead), npix, R + 1, L.ptr(whb), cf, 0, L.ptr(g), st))
        else:
            L.check(lib.sdb_heads_backward(L.ptr(feat), L.ptr(dhead), npix, cf, L.ptr(self.pview['prob'][0]), L.ptr(self.pview['dist'][0]),
                                           R, 0, L.ptr(g), st))
        gin_class = None if dclass is None else self._class_backward(dclass, g)
        first = next(i for i, l in enumerate(self.layers) if l['kind'] == 'conv')
        skip_grad = {}
        for i in reversed(range(len(self.layers))):
            l = self.layers[i]
            a = net.saved[i]
            if l['kind'] == 'conv':
                self._act_backward(g, l['act'], a['y'], a['z'])
                x, lo, up = a['x'], a['lo'], a['up']
                cout = l['cout']
                self._wgrad(x, lo, up, l['k'], g, cout, cout, *self.gview[l['name']])
                if i == first:
                    break                                    # the network input needs no gradient
                n = x.shape[0]; d, h, w = self._dhw(x)
                gin = self._dgrad(i, l['name'], g, x.shape, l['cin'], cout, l['k'])
                if gin_class is not None and l['name'] == 'features':
                    if self.bf16:
                        L.check(lib.sdb_add_bf16(L.ptr(gin), L.ptr(gin_class), gin.numel(), L.ptr(gin), st))
                    else:
                        L.check(lib.sdb_add_act(L.ptr(gin), L.ptr(gin_class), gin.numel(), 0, L.ptr(gin), st))
                if lo is not None:
                    up_layer = self.layers[i - 1]
                    assert up_layer['kind'] == 'up'
                    uz, uy, ux = ((1,) + tuple(up)) if len(up) == 2 else tuple(up)
                    dlo = self._buf(('dlo', i), lo.shape, bf16=self.bf16)
                    dskip = self._buf(('dskip', i), x.shape, bf16=self.bf16)
                    split = lib.sdb_decoder_split_bf16 if self.bf16 else lib.sdb_decoder_split
                    L.check(split(L.ptr(gin), n, d, h, w, lo.shape[-1], x.shape[-1], int(uz), int(uy), int(ux), L.ptr(dlo), L.ptr(dskip), st))
                    skip_grad[up_layer['skip']] = dskip
                    g = dlo
                else:
                    g = gin
            elif l['kind'] == 'pool':
                x = a['x']
                n = x.shape[0]; d, h, w = self._dhw(x)
                pz, py, px = ((1,) + tuple(l['pool'])) if self.nd == 2 else tuple(l['pool'])
                if 'save_skip' in l:
                    gx, acc = skip_grad.pop(l['save_skip']), 1
                else:
                    gx, acc = self._buf(('gpool', i), x.shape, bf16=self.bf16), 0
                pool_bwd = lib.sdb_maxpool_backward_bf16_nd if self.bf16 else lib.sdb_maxpool_backward_nd
                L.check(pool_bwd(L.ptr(x), L.ptr(g), n, d, h, w, x.shape[-1], int(pz), int(py), int(px), acc, L.ptr(gx), st))
                g = gx

    # ---------------------------------------------------------------------------------------------- mixed_bfloat16 forward
    def _forward_bf16(self, x):
        """the forward pass under 'mixed_bfloat16': the input rounded to bf16 once, every convolution on sdb_conv_bf16_nd with bf16
        kernels copied from the fp32 parameters, bf16 max pooling, fp32 prob / dist / prob_class from bf16 features.  Keeps in
        self.net what _backward reads, as UNetDeviceND.forward(keep=True) does, with bf16 tensors."""
        import torch
        lib = L.load()
        st = L.stream_ptr()
        net, nd = self.net, self.nd
        ones = (1,) * nd
        cur = self._buf('x_bf16', x.shape, bf16=True)
        L.check(lib.sdb_cast_bf16(L.ptr(x), x.numel(), L.ptr(cur), st))
        skips, saved = {}, [None] * len(self.layers)
        lo, up, base = None, ones, None
        for i, l in enumerate(self.layers):
            kind = l['kind']
            if kind == 'conv':
                if l['name'] == 'features':
                    base = cur
                y = self._conv_bf16(cur, lo, up, l)
                saved[i] = dict(x=cur, lo=lo, up=up, y=y, z=None)
                cur, lo, up = y, None, ones
            elif kind == 'pool':
                if 'save_skip' in l:
                    skips[l['save_skip']] = cur
                saved[i] = dict(x=cur)
                n = cur.shape[0]; d, h, w = self._dhw(cur); c = cur.shape[-1]
                pz, py, px = ((1,) + tuple(l['pool'])) if nd == 2 else tuple(l['pool'])
                osp = (h // py, w // px) if nd == 2 else (d // pz, h // py, w // px)
                out = torch.empty((n,) + osp + (c,), dtype=torch.bfloat16, device=cur.device)
                L.check(lib.sdb_maxpool_bf16_nd(L.ptr(cur), n, d, h, w, c, int(pz), int(py), int(px), L.ptr(out), st))
                cur = out
            elif kind == 'up':
                lo, up = cur, tuple(l['pool'])
                cur = skips.pop(l['skip'])
            elif kind == 'head':
                break
        feat = cur
        net.saved, net.saved_feat = saved, feat
        R, cf = self.config.n_rays, feat.shape[-1]
        npix = feat.numel() // cf
        whb = self._buf('wheads_bf16', ((R + 1) * cf,), bf16=True)
        L.check(lib.sdb_weights_bf16(L.ptr(self.pview['prob'][0]), 1, cf, 1, 0, cf, L.ptr(whb), st))
        L.check(lib.sdb_weights_bf16(L.ptr(self.pview['dist'][0]), 1, cf, R, 0, cf, L.ptr(whb[cf:]), st))
        prob = torch.empty(tuple(feat.shape[:-1]), dtype=torch.float32, device=feat.device)
        dist = torch.empty(tuple(feat.shape[:-1]) + (R,), dtype=torch.float32, device=feat.device)
        L.check(lib.sdb_heads_bf16(L.ptr(feat), npix, cf, L.ptr(whb), L.ptr(self.pview['prob'][1]), L.ptr(self.pview['dist'][1]), R,
                                   L.ptr(prob), L.ptr(dist), st))
        net.prob_class = None
        if self.n_classes is not None:
            base = feat if base is None else base
            xc = base
            if 'features_class' in self.pview:
                fl = next(l for l in self.layers if l['name'] == 'features_class')
                xc = self._conv_bf16(base, None, ones, fl)
            C = self.n_classes + 1
            wcb = self._buf('wclass_bf16', (C * xc.shape[-1],), bf16=True)
            L.check(lib.sdb_weights_bf16(L.ptr(self.pview['prob_class'][0]), 1, xc.shape[-1], C, 0, xc.shape[-1], L.ptr(wcb), st))
            logits = self._buf('class_logits', tuple(xc.shape[:-1]) + (C,))
            out = torch.empty(tuple(xc.shape[:-1]) + (C,), dtype=torch.float32, device=xc.device)
            L.check(lib.sdb_class_head_bf16(L.ptr(xc), npix, xc.shape[-1], L.ptr(wcb), L.ptr(self.pview['prob_class'][1]), C,
                                            L.ptr(logits), L.ptr(out), st))
            net.saved_class, net.saved_class_z, net.prob_class = (base, xc, out), None, out
        return prob, dist

    def _conv_bf16(self, x, lo, up, l):
        """act(conv([upsample(lo), x]) + bias) of layer l as bf16, from a bf16 copy of its fp32 kernel"""
        import torch
        lib = L.load()
        st = L.stream_ptr()
        name, cout = l['name'], l['cout']
        k = tuple(l['k'])
        taps = int(np.prod(k))
        n = x.shape[0]; d, h, w = self._dhw(x)
        c_skip, c_lo = x.shape[-1], 0 if lo is None else lo.shape[-1]
        cin = c_skip + c_lo
        wb = self._buf(('wb', name), (taps * cout * cin,), bf16=True)
        L.check(lib.sdb_weights_bf16(L.ptr(self.pview[name][0]), taps, cin, cout, 0, cin, L.ptr(wb), st))
        kz, ky, kx = ((1,) + k) if self.nd == 2 else k
        uz, uy, ux = ((1,) + tuple(up)) if len(up) == 2 else tuple(up)
        y = torch.empty(tuple(x.shape[:-1]) + (cout,), dtype=torch.bfloat16, device=x.device)
        L.check(lib.sdb_conv_bf16_nd(L.ptr(x), L.ptr(lo), n, d, h, w, c_skip, c_lo, int(uz), int(uy), int(ux), kz, ky, kx, L.ptr(wb),
                                     L.ptr(self.pview[name][1]), cout, 1 if l['act'] == 'relu' else 0, 0, L.ptr(y), st))
        return y

    # ---------------------------------------------------------------------------------------------- public
    def _forward_loss(self, x, prob_t, dam, dhead, out, state, prob_class_t=None, dclass=None):
        import torch
        x = x if x.is_contiguous() else x.contiguous()
        if self.bf16:
            prob, dist = self._forward_bf16(x)
        else:
            prob, dist = self.net.forward(x, keep=dhead is not None)
        self._loss(prob, dist, prob_t, dam, dhead, out, state)
        if self.n_classes is not None:
            self._class_loss(self.net.prob_class, prob_class_t, dclass, out)

    def saved_activations(self):
        """the distinct device tensors the last forward pass kept for the backward pass"""
        net, seen, out = self.net, set(), []
        ts = [v for a in net.saved if a is not None for v in a.values() if hasattr(v, 'data_ptr')] + [net.saved_feat]
        if self.n_classes is not None:
            ts += list(net.saved_class[:2])            # the third entry is the fp32 prob_class output
        for t in ts:
            if t is not None and t.data_ptr() not in seen:
                seen.add(t.data_ptr())
                out.append(t)
        return out

    def _n_out(self):
        return 4 if self.n_classes is None else 5

    def _dclass(self, prob_class_t):
        """the dL/d(prob_class logits) buffer of a multi-class model (None for single-class ones)"""
        if self.n_classes is None:
            return None
        if prob_class_t is None:
            raise ValueError("a multi-class model needs the prob_class target")
        return self._buf('dclass', (prob_class_t.numel() // (self.n_classes + 1), self.n_classes + 1))

    def step(self, x, prob_t, dam, prob_class_t=None, out=None):
        """one training step on a batch (CUDA tensors as StarDistData*.batch_device gives them; prob_class_t for multi-class
        models); returns the device float32 [4] (loss, prob_loss, dist_loss, skipped) or, for multi-class models, [5] (loss,
        prob_loss, dist_loss, skipped, prob_class_loss) -- or writes it into `out`"""
        import torch
        lib = L.load()
        dclass = self._dclass(prob_class_t)
        if self.n_calls + 1 > self.coef.numel():
            self.coef = torch.from_numpy(adam_coef(max(1024, 2 * (self.n_calls + 1)))).to(self.net.device)
        self.n_calls += 1
        out = self._buf('out', (self._n_out(),)) if out is None else out
        npix = prob_t.numel()
        dhead = self._buf('dhead', (npix, self.config.n_rays + 1))
        self._forward_loss(x, prob_t, dam, dhead, out, self.state, prob_class_t, dclass)
        self._backward(dhead, dclass)
        one = np.float32(1)
        L.check(lib.sdb_adam_step(L.ptr(self.params), L.ptr(self.grad), L.ptr(self.m), L.ptr(self.v), self.params.numel(),
                                  float(self.lr), float(one - np.float32(ADAM_BETA_1)), float(one - np.float32(ADAM_BETA_2)),
                                  float(np.float32(ADAM_EPSILON)), L.ptr(self.coef), L.ptr(self.state), L.stream_ptr()))
        return out

    def evaluate(self, x, prob_t, dam, prob_class_t=None):
        """forward pass and loss only: device float32 [4] (loss, prob_loss, dist_loss, n_p == 0), [5] with prob_class_loss
        for multi-class models"""
        import torch
        if self.n_classes is not None and prob_class_t is None:
            raise ValueError("a multi-class model needs the prob_class target")
        out = torch.empty(self._n_out(), dtype=torch.float32, device=self.net.device)
        self._forward_loss(x, prob_t, dam, None, out, None, prob_class_t)
        return out

    def gradients(self, x, prob_t, dam, prob_class_t=None):
        """dict name -> (d kernel, d bias) numpy of the loss on one batch, without updating anything"""
        import torch
        dclass = self._dclass(prob_class_t)
        out = torch.empty(self._n_out(), dtype=torch.float32, device=self.net.device)
        dhead = self._buf('dhead', (prob_t.numel(), self.config.n_rays + 1))
        self._forward_loss(x, prob_t, dam, dhead, out, None, prob_class_t, dclass)
        self._backward(dhead, dclass)
        return {n: (self.gview[n][0].cpu().numpy(), self.gview[n][1].cpu().numpy()) for n in self.names}

    def weights(self):
        """the current parameters as a weights dict (name -> (kernel, bias) float32 numpy)"""
        host = self.params.cpu().numpy()
        out = {}
        for n in self.names:
            ks, bs = self.shapes[n]
            nk, nb = int(np.prod(ks)), int(np.prod(bs))
            off = self.offsets[n]
            out[n] = (host[off:off + nk].reshape(ks).copy(), host[off + nk:off + nk + nb].reshape(bs).copy())
        return out


# ------------------------------------------------------------------------------------------------------ callbacks
class ReduceLROnPlateau:
    """keras.callbacks.ReduceLROnPlateau on 'val_loss' in mode 'min' (restated: on_epoch_end returns the new lr)"""

    def __init__(self, factor=0.1, patience=10, min_delta=1e-4, cooldown=0, min_lr=0, **ignored):
        if factor >= 1.0:
            raise ValueError("ReduceLROnPlateau does not support a factor >= 1.0")
        self.factor, self.patience, self.min_delta = float(factor), int(patience), float(min_delta)
        self.cooldown, self.min_lr = int(cooldown), float(min_lr)
        self.best, self.wait, self.cooldown_counter = np.inf, 0, 0

    def on_epoch_end(self, current, lr):
        lr = np.float32(lr)
        if self.cooldown_counter > 0:
            self.cooldown_counter -= 1
            self.wait = 0
        if np.less(current, self.best - self.min_delta):
            self.best, self.wait = current, 0
        elif not self.cooldown_counter > 0:
            self.wait += 1
            if self.wait >= self.patience:
                if lr > np.float32(self.min_lr):
                    lr = np.float32(max(float(lr) * self.factor, self.min_lr))
                    self.cooldown_counter, self.wait = self.cooldown, 0
        return lr


class BestCheckpoint:
    """csbdeep's best checkpoint (keras ModelCheckpoint(save_best_only=True) on 'val_loss'): saved when strictly lower"""

    def __init__(self):
        self.best = np.inf

    def improved(self, current):
        if np.less(current, self.best):
            self.best = current
            return True
        return False


class History:
    """the per-epoch record of train(), like the History object Keras' fit returns"""

    KEYS = ('loss', 'prob_loss', 'dist_loss', 'val_loss', 'val_prob_loss', 'val_dist_loss', 'lr')
    KEYS_CLASSES = ('loss', 'prob_loss', 'dist_loss', 'prob_class_loss', 'val_loss', 'val_prob_loss', 'val_dist_loss',
                    'val_prob_class_loss', 'lr')

    def __init__(self, multiclass=False):
        self.history = {k: [] for k in (self.KEYS_CLASSES if multiclass else self.KEYS)}
        self.epoch = []


# ------------------------------------------------------------------------------------------------------ train()
def train(model, X, Y, validation_data, classes='auto', augmenter=None, seed=None, epochs=None, steps_per_epoch=None, workers=1,
          optimizer=None):
    """StarDist2D.train / StarDist3D.train (stardist/models/model2d.py:352-481, model3d.py): returns a History.  X, Y and
    validation_data's X, Y may be lazy sequences; they go to the generators as given, and the validation patches are made once."""
    config = model.config
    check_trainable(config, optimizer)
    multi = config.n_classes is not None
    if multi:
        classes = model._parse_classes_arg(classes, len(X))
    elif classes != 'auto' and classes is not None:
        warnings.warn("Ignoring given classes as n_classes is set to None")
    if seed is not None:
        np.random.seed(seed)
    if epochs is None:
        epochs = config.train_epochs
    if steps_per_epoch is None:
        steps_per_epoch = config.train_steps_per_epoch
    isinstance(validation_data, (list, tuple)) or _raise(ValueError())
    if multi and len(validation_data) == 2:
        validation_data = tuple(validation_data) + ('auto',)
    n_vd = 3 if multi else 2
    len(validation_data) == n_vd or _raise(ValueError('len(validation_data) = %d, but should be %d' % (len(validation_data), n_vd)))
    classes_val = model._parse_classes_arg(validation_data[2], len(validation_data[0])) if multi else None
    patch_size = config.train_patch_size
    axes = config.axes.replace('C', '')
    div_by = model._axes_div_by(axes)
    [(p % d == 0) or _raise(ValueError("'train_patch_size' must be divisible by {d} along axis '{a}'".format(a=a, d=d)))
     for p, d, a in zip(patch_size, div_by, axes)]

    import torch
    from .data import StarDistData2D, StarDistData3D
    L.require_cuda()
    kw = dict(patch_size=config.train_patch_size, grid=config.grid, foreground_prob=config.train_foreground_only,
              sample_ind_cache=config.train_sample_cache)
    if config.n_dim == 2:
        Data = StarDistData2D
        kw.update(n_rays=config.n_rays)
    else:
        from ..rays3d import rays_from_json
        Data = StarDistData3D
        kw.update(rays=rays_from_json(config.rays_json), anisotropy=config.anisotropy)
    n_val = len(validation_data[0])
    n_take = config.train_n_val_patches if config.train_n_val_patches is not None else n_val
    if multi:
        data_val = Data(validation_data[0], validation_data[1], batch_size=n_take, length=1, n_classes=config.n_classes,
                        classes=classes_val, **kw)
        (xv,), (pv, dv, cv) = data_val.batch_device(0)
        model.data_train = Data(X, Y, batch_size=config.train_batch_size, augmenter=augmenter, length=epochs * steps_per_epoch,
                                n_classes=config.n_classes, classes=classes, **kw)
    else:
        data_val = Data(validation_data[0], validation_data[1], batch_size=n_take, length=1, **kw)
        (xv,), (pv, dv) = data_val.batch_device(0)
        model.data_train = Data(X, Y, batch_size=config.train_batch_size, augmenter=augmenter, length=epochs * steps_per_epoch, **kw)

    trainer = UNetTrainer(config, model.weights)
    rlr = ReduceLROnPlateau(**config.train_reduce_lr) if config.train_reduce_lr is not None else None
    best_ckpt = BestCheckpoint()
    logdir = getattr(model, 'logdir', None)
    if logdir is not None:
        logdir.mkdir(parents=True, exist_ok=True)
        with open(logdir / 'config.json', 'w') as f:
            f.write(config.to_json())
    hist = History(multi)
    # per-step rows (loss, prob_loss, dist_loss, skipped[, prob_class_loss]); the history's losses are the columns `cols`
    log = torch.empty((steps_per_epoch, 5 if multi else 4), dtype=torch.float32, device=trainer.net.device)
    cols = [0, 1, 2, 4] if multi else [0, 1, 2]
    names = [k for k in hist.history if k != 'lr']
    bs = int(config.train_batch_size)
    best_weights = None
    for epoch in range(epochs):
        for s in range(steps_per_epoch):
            (x,), targets = model.data_train.batch_device(epoch * steps_per_epoch + s)
            trainer.step(x, *targets, out=log[s])
        # validation over batches of train_batch_size, weighted by batch size (Keras' evaluate)
        vals = []
        for b0 in range(0, n_take, bs):
            b1 = min(n_take, b0 + bs)
            vt = (cv[b0:b1],) if multi else ()
            vals.append((b1 - b0, trainer.evaluate(xv[b0:b1], pv[b0:b1], dv[b0:b1], *vt)))
        steps = log.cpu().numpy()
        vrows = np.stack([v.cpu().numpy() for _, v in vals])
        vw = np.array([n for n, _ in vals], np.float64)
        ok = steps[:, 3] == 0
        if not ok.all():
            warnings.warn("epoch %d: %d training batch(es) without any labelled pixel (all prob targets < 0) were skipped"
                          % (epoch + 1, int((~ok).sum())))
        tr = steps[ok][:, cols].astype(np.float64).mean(axis=0) if ok.any() else np.full(len(cols), np.nan)
        va = (vrows[:, cols].astype(np.float64) * vw[:, None]).sum(axis=0) / vw.sum()
        for k, v in zip(names, list(tr) + list(va)):
            hist.history[k].append(float(v))
        hist.history['lr'].append(float(trainer.lr))
        hist.epoch.append(epoch)
        if rlr is not None:
            trainer.lr = rlr.on_epoch_end(va[0], trainer.lr)
        if best_ckpt.improved(va[0]):
            best_weights = trainer.weights()
            if logdir is not None:
                _save_weights(logdir / 'weights.npz', best_weights)
        if logdir is not None:
            _save_weights(logdir / 'weights_last.npz', trainer.weights())
    # csbdeep's _training_finished: with a model folder the best checkpoint is loaded, otherwise the last weights stay
    final = trainer.weights()
    model.weights = best_weights if (logdir is not None and best_weights is not None) else final
    model._net = None
    return hist


def _save_weights(path, weights):
    np.savez(path, **{('%s/kernel' % k): v[0] for k, v in weights.items()}, **{('%s/bias' % k): v[1] for k, v in weights.items()})
