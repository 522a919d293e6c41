"""StarDistBase: prediction orchestration, device resident.

Mirrors the prediction half of stardist/models/base.py:
  _predict_setup (:371-443), _predict_generator/predict (:446-529), _predict_sparse_generator/
  predict_sparse (:541-642), _predict_instances_generator/predict_instances (:645-790),
  predict_instances_big (:838-983), thresholds handling (:230-252), _compute_receptive_field
  (:1068-1098), _axes_tile_overlap (:1101-1111), StarDistPadAndCropResizer (:1162-1211),
  optimize_thresholds (:986-1043), _guess_n_tiles (:1046-1055).
Training is in models/train.py; export is out of scope (DESIGN.md).

Differences by design: the network, thresholding, sort, NMS and label painting all run as CUDA
kernels on tensors that stay in HBM; only the final labels / polygons are copied to the host.
"""
import json, math, numbers, warnings, functools
from collections import namedtuple
from pathlib import Path
import numpy as np
import torch

from .. import _lib as L
from ..utils import (_raise, axes_check_and_normalize, axes_dict, move_image_axes, _is_floatarray,
                     _is_power_of_2)
from .weights import glorot_uniform_weights

Thresholds = namedtuple('Thresholds', ('prob', 'nms'))


class NoNormalizer:
    def before(self, x, axes):
        return x

    def after(self, mean, scale, axes):
        return mean, scale


class PercentileNormalizer:
    """csbdeep.data.PercentileNormalizer (percentile based input normalization)"""

    def __init__(self, pmin=2, pmax=99.8, do_after=True, dtype=np.float32, **kwargs):
        self.pmin, self.pmax, self._do_after, self.dtype, self.kwargs = pmin, pmax, do_after, dtype, kwargs

    def before(self, x, axes):
        from ..utils import normalize_mi_ma
        axes = axes_check_and_normalize(axes, x.ndim)
        channel = axes_dict(axes)['C']
        axis = None if channel is None else tuple((d for d in range(x.ndim) if d != channel))
        self.mi = np.percentile(x, self.pmin, axis=axis, keepdims=True).astype(self.dtype, copy=False)
        self.ma = np.percentile(x, self.pmax, axis=axis, keepdims=True).astype(self.dtype, copy=False)
        return normalize_mi_ma(x, self.mi, self.ma, dtype=self.dtype, **self.kwargs)


class StarDistPadAndCropResizer:
    """stardist/models/base.py:1162-1211 (pads at the END of each axis, mode 'reflect')"""

    def __init__(self, grid, mode='reflect', **kwargs):
        assert isinstance(grid, dict)
        self.mode = mode
        self.grid = grid
        self.kwargs = kwargs

    def plan(self, shape, axes, axes_div_by):
        """the bookkeeping of before() for an array of the given shape, without touching data (the device path pads in HBM)"""
        assert all(a % g == 0 for g, a in zip((self.grid.get(a, 1) for a in axes), axes_div_by))
        axes = axes_check_and_normalize(axes, len(shape))
        self.pad = {a: (0, (div_n - s % div_n) % div_n) for a, div_n, s in zip(axes, axes_div_by, shape)}
        self.padded_shape = {a: s + self.pad[a][1] for a, s in zip(axes, shape)}
        if 'C' in self.padded_shape:
            del self.padded_shape['C']
        return tuple(s + self.pad[a][1] for a, s in zip(axes, shape))

    def before(self, x, axes, axes_div_by):
        assert all(a % g == 0 for g, a in zip((self.grid.get(a, 1) for a in axes), axes_div_by))
        axes = axes_check_and_normalize(axes, x.ndim)

        def _split(v):
            return 0, v  # only pad at the end
        self.pad = {a: _split((div_n - s % div_n) % div_n) for a, div_n, s in zip(axes, axes_div_by, x.shape)}
        if all(self.pad[a] == (0, 0) for a in axes):
            x_pad = x          # nothing to pad: np.pad would only copy
        else:
            x_pad = np.pad(x, tuple(self.pad[a] for a in axes), mode=self.mode, **self.kwargs)
        self.padded_shape = dict(zip(axes, x_pad.shape))
        if 'C' in self.padded_shape:
            del self.padded_shape['C']
        return x_pad

    def crop_slices(self, axes, shape):
        axes = axes_check_and_normalize(axes, len(shape))
        assert all(s_pad == s * g for s, s_pad, g in zip(shape,
                                                         (self.padded_shape.get(a, _s) for a, _s in zip(axes, shape)),
                                                         (self.grid.get(a, 1) for a in axes)))
        return tuple(
            slice(0, -(math.floor(p[1] / g)) if p[1] >= g else None)
            for p, g in zip((self.pad.get(a, (0, 0)) for a in axes), (self.grid.get(a, 1) for a in axes)))

    def after(self, x, axes):
        return x[self.crop_slices(axes, x.shape)]

    def point_bounds(self, axes):
        """filter_points: a candidate is kept iff point < padded_shape - pad (per spatial axis)"""
        return tuple(self.padded_shape[a] - self.pad[a][1] for a in axes if a.lower() in ('z', 'y', 'x'))

    def filter_points(self, ndim, points, axes):
        assert points.ndim == 2
        axes = axes_check_and_normalize(axes, ndim)
        bounds = np.array(self.point_bounds(axes))
        return np.where(np.all(points < bounds, 1))


class StarDistBase:
    """Common prediction logic of StarDist2D / StarDist3D."""

    def __init__(self, config, name=None, basedir='.', weights=None, seed=0):
        self.name = name
        self.basedir = None if basedir is None else Path(basedir)
        self.logdir = None if (basedir is None or name is None) else self.basedir / name
        if config is None:
            if self.logdir is None or not (self.logdir / 'config.json').exists():
                raise FileNotFoundError("config file doesn't exist: %s" % (None if self.logdir is None else str((self.logdir / 'config.json').resolve())))
            with open(self.logdir / 'config.json') as f:
                cfg = json.load(f)
            config = self._config_class(**cfg)
        isinstance(config, self._config_class) or _raise(ValueError("Invalid configuration of type '%s', was expecting type '%s'." % (type(config).__name__, self._config_class.__name__)))
        self.config = config
        # thresholds (base.py:230-252)
        threshs = dict(prob=None, nms=None)
        if self.logdir is not None and (self.logdir / 'thresholds.json').exists():
            with open(self.logdir / 'thresholds.json') as f:
                threshs = json.load(f)
            if threshs.get('prob') is not None and not (0 < threshs['prob'] < 1):
                threshs['prob'] = None
            if threshs.get('nms') is not None and not (0 < threshs['nms'] < 1):
                threshs['nms'] = None
        if threshs.get('prob') is None or threshs.get('nms') is None:
            default = dict(prob=0.5, nms=0.4)
            for k in default:
                if threshs.get(k) is None:
                    threshs[k] = default[k]
        self.thresholds = dict(prob=threshs['prob'], nms=threshs['nms'])
        # weights: explicit dict > <logdir>/weights.npz > seeded Glorot-uniform (Keras default init)
        if weights is None and self.logdir is not None and (self.logdir / 'weights.npz').exists():
            weights = load_weights_npz(self.logdir / 'weights.npz')
        if weights is None and self.logdir is not None:
            # Keras checkpoints of a trained reference model (csbdeep BaseModel._find_and_load_weights: best, then last)
            for fname in (getattr(config, 'train_checkpoint', None) or 'weights_best.h5', 'weights_best.h5', 'weights_last.h5'):
                if fname and (self.logdir / fname).exists():
                    from ..io import h5lite
                    weights = h5lite.read_keras_weights(str(self.logdir / fname))
                    break
        if weights is None:
            weights = glorot_uniform_weights(config, seed=seed)
        else:
            from .weights import canonicalize_auto_names
            weights = canonicalize_auto_names(config, weights)
            self._check_weights(config, weights)
        self.weights = weights
        self._net = None
        self._stats = {}

    @staticmethod
    def _check_weights(config, weights):
        """every conv / head layer of the architecture must be present with the expected kernel shape"""
        from .weights import net_layers
        for l in net_layers(config):
            if l['kind'] not in ('conv', 'head', 'conv_class', 'head_class'):
                continue
            if l['name'] not in weights:
                raise ValueError("weights for layer '%s' are missing" % l['name'])
            k = np.asarray(weights[l['name']][0])
            want = tuple(l['k']) + (l['cin'], l['cout'])
            if tuple(k.shape) != want:
                raise ValueError("layer '%s': kernel shape %s, expected %s" % (l['name'], tuple(k.shape), want))

    # ------------------------------------------------------------------ properties
    @property
    def thresholds(self):
        return self._thresholds

    @thresholds.setter
    def thresholds(self, d):
        self._thresholds = Thresholds(**d)

    # optional per-stage CUDA-event timing (bench.py): set model._events = [] to collect
    def _mark(self, name):
        ev = getattr(self, '_events', None)
        if ev is not None:
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            ev.append((name, e))

    def _is_multiclass(self):
        return self.config.n_classes is not None

    @property
    def net(self):
        if self._net is None:
            self._net = self._build()
        return self._net

    def prepare_for_training(self, optimizer=None):
        """checks that train() covers this model; only the default optimizer (Adam with train_learning_rate) is supported"""
        from .train import check_trainable
        check_trainable(self.config, optimizer)

    def save_weights(self, path):
        np.savez(path, **{('%s/kernel' % k): v[0] for k, v in self.weights.items()},
                 **{('%s/bias' % k): v[1] for k, v in self.weights.items()})

    # ------------------------------------------------------------------ helpers shared with the reference
    def _normalize_axes(self, img, axes):
        if axes is None:
            axes = self.config.axes
            assert 'C' in axes
            if img.ndim == len(axes) - 1 and self.config.n_channel_in == 1:
                axes = axes.replace('C', '')
        return axes_check_and_normalize(axes, img.ndim)

    def _make_permute_axes(self, img_axes_in, net_axes_in, net_axes_out=None):
        if net_axes_out is None:
            net_axes_out = net_axes_in
        channel_in = axes_dict(img_axes_in)['C']

        def _permute_axes(data, undo=False):
            if data is None:
                return None
            if undo:
                if channel_in is not None:
                    return move_image_axes(data, net_axes_out, img_axes_in, True)
                else:
                    data = move_image_axes(data, net_axes_out, img_axes_in + 'C', True)
                    if data.shape[-1] == 1:
                        data = data[..., 0]
                    return data
            else:
                return move_image_axes(data, img_axes_in, net_axes_in, True)
        return _permute_axes

    def _check_normalizer(self, normalizer):
        if normalizer is None:
            return NoNormalizer()
        hasattr(normalizer, 'before') or _raise(ValueError("normalizer must provide .before(x, axes)"))
        return normalizer

    def _device_prep_plan(self, x, axes_net, normalizer, zoom):
        """Can normalisation / zoom / reflect padding of this input run in HBM (stardist_b200/prep.py)?  Conditions: single
        input channel, a dtype whose values the float32 upload preserves, no normaliser or this module's PercentileNormalizer
        with its plain arguments.  Returns the plan (dict) or None (host path, as the reference does it)."""
        import os
        from .. import prep
        if os.environ.get("STARDIST_B200_PREP", "device") != "device" or not torch.cuda.is_available():
            return None
        if not isinstance(x, np.ndarray) or x.dtype not in prep.EXACT_IN_F32 or self.config.n_channel_in != 1 or x.shape[-1] != 1:
            return None
        norm = None
        if isinstance(normalizer, PercentileNormalizer):
            kw = dict(normalizer.kwargs)
            if type(normalizer) is not PercentileNormalizer or set(kw) - {'clip', 'eps'} or np.dtype(normalizer.dtype) != np.float32:
                return None
            norm = (normalizer.pmin, normalizer.pmax, bool(kw.get('clip', False)), kw.get('eps', 1e-20))
        elif not isinstance(normalizer, NoNormalizer):
            return None
        if zoom is not None and x.dtype.kind not in 'iuf':
            return None
        if zoom is not None and x.dtype == np.float16:
            return None
        return dict(norm=norm, zoom=None if zoom is None else tuple(zoom), src_dtype=x.dtype)

    def _predict_setup(self, img, axes, normalizer, n_tiles, _zoom=None):
        """ Shared setup code between `predict` and `predict_sparse` (base.py:371-443) """
        if n_tiles is None:
            n_tiles = [1] * img.ndim
        try:
            n_tiles = tuple(n_tiles)
            img.ndim == len(n_tiles) or _raise(TypeError())
        except TypeError:
            raise ValueError("n_tiles must be an iterable of length %d" % img.ndim)
        all(np.isscalar(t) and 1 <= t and int(t) == t for t in n_tiles) or _raise(
            ValueError("all values of n_tiles must be integer values >= 1"))
        n_tiles = tuple(map(int, n_tiles))
        axes = self._normalize_axes(img, axes)
        axes_net = self.config.axes
        _permute_axes = self._make_permute_axes(axes, axes_net)
        x = _permute_axes(img)  # x has axes_net semantics
        channel = axes_dict(axes_net)['C']
        self.config.n_channel_in == x.shape[channel] or _raise(ValueError())
        axes_net_div_by = self._axes_div_by(axes_net)
        grid = tuple(self.config.grid)
        len(grid) == len(axes_net) - 1 or _raise(ValueError())
        grid_dict = dict(zip(axes_net.replace('C', ''), grid))
        normalizer = self._check_normalizer(normalizer)
        resizer = StarDistPadAndCropResizer(grid=grid_dict)
        self._dev_prep = None
        zoom_net = None
        if _zoom is not None:                      # per image axis -> network axis order (the channel factor is 1)
            zd = dict(zip(axes, _zoom))
            zoom_net = tuple(zd.get(a, 1) for a in axes_net)
        plan = self._device_prep_plan(x, axes_net, normalizer, zoom_net)
        if plan is not None and (plan['norm'] is not None or plan['zoom'] is not None or
                                 any(s % d for s, d in zip(x.shape, axes_net_div_by))):
            # normalisation / zoom / padding happen in HBM after the upload (_to_device); only the bookkeeping here
            shape_z = tuple(x.shape) if zoom_net is None else tuple(int(round(s * z)) for s, z in zip(x.shape, zoom_net))
            plan.update(normalizer=normalizer, shape_z=shape_z, padded=resizer.plan(shape_z, axes_net, axes_net_div_by))
            self._dev_prep = plan
            if plan['norm'] is None and not _is_floatarray(x):
                warnings.warn("Predicting on non-float input... ( forgot to normalize? )")
        else:
            if _zoom is not None:
                from scipy import ndimage as ndi
                x = ndi.zoom(x, zoom_net, order=1)
            x = normalizer.before(x, axes_net)
            x = resizer.before(x, axes_net, axes_net_div_by)
            if not _is_floatarray(x):
                warnings.warn("Predicting on non-float input... ( forgot to normalize? )")
        # tiles refer to the axes of the input image; the network sees them in axes_net order (base.py:419-424)
        n_tiles = _permute_axes(np.empty(n_tiles, dtype=bool)).shape
        n_tiles[channel] == 1 or _raise(ValueError("cannot tile the channel axis"))
        return x, axes, axes_net, axes_net_div_by, _permute_axes, resizer, n_tiles, grid, grid_dict, channel

    def _pinned(self, key, shape, dtype):
        """persistent pinned staging buffers (one per role, grown in powers of two): torch's caching host
        allocator sporadically takes ~60 ms for a 4 MB pinned block (cudaHostAlloc / cudaFreeHost)"""
        pool = self.__dict__.setdefault('_pin_pool', {})
        nbytes = int(np.prod(shape, dtype=np.int64)) * torch.empty((), dtype=dtype).element_size()
        buf = pool.get(key)
        if buf is None or buf.numel() < nbytes:
            cap = 1 << max(12, int(nbytes - 1).bit_length())
            buf = torch.empty(cap, dtype=torch.uint8, pin_memory=torch.cuda.is_available())
            pool[key] = buf
        return buf[:nbytes].view(dtype).view(tuple(shape))

    @staticmethod
    def _stage_fill(stage, x):
        """host array x (any dtype / strides) -> float32 staging tensor stage[0] (same shape).  Large float arrays go through torch's
        multi-threaded copy (a 134 MB volume: 3-6 ms instead of 27-38 ms with np.copyto on 8 cores), everything else, and
        anything torch refuses (byte-swapped, unsupported dtypes), through numpy; both are IEEE conversions to float32."""
        if x.dtype in (np.float32, np.float64) and x.size >= (1 << 23):      # volumes; a 1024^2 image stays on the single memcpy
            try:
                stage[0].copy_(torch.from_numpy(x if x.flags.c_contiguous else np.ascontiguousarray(x)))
                return
            except (TypeError, ValueError, RuntimeError):
                pass
        np.copyto(stage.numpy()[0], x, casting='unsafe')

    def _to_device(self, x):
        """host float array (axes_net semantics, channels last) -> pinned staging buffer -> device [1,...,C] float32"""
        x = np.asarray(x)
        stage = self._pinned('in', (1,) + x.shape, torch.float32)
        self._stage_fill(stage, x)
        self._stats['h2d_bytes'] = self._stats.get('h2d_bytes', 0) + stage.numel() * 4
        x_dev = stage.to(self.net.device, non_blocking=True)
        plan, self._dev_prep = getattr(self, '_dev_prep', None), None
        if plan is None:
            return x_dev
        from .. import prep
        t = x_dev[0, ..., 0]                                  # single channel: the spatial array, contiguous
        if plan['zoom'] is not None:
            t = prep.zoom_device(t, plan['zoom'][:-1], plan['src_dtype'])
        if plan['norm'] is not None:
            pmin, pmax, clip, eps = plan['norm']
            mi, ma = prep.normalize_device(t, tuple(t.shape), pmin, pmax, plan['src_dtype'], clip=clip, eps=eps)
            nz = plan['normalizer']                            # PercentileNormalizer.before leaves mi / ma behind
            nz.mi = np.asarray(mi, np.float32).reshape((1,) * x.ndim); nz.ma = np.asarray(ma, np.float32).reshape((1,) * x.ndim)
        t = prep.pad_reflect_end_device(t.unsqueeze(-1), plan['padded'][:-1])
        return t.unsqueeze(0)

    def _to_host(self, tensors, copy_threads=False):
        """device tensors -> numpy arrays: asynchronous copies into persistent pinned buffers, ONE stream
        synchronisation for all of them, then a host copy into fresh arrays (copy_threads: through torch's
        multi-threaded copy, for the large label maps of predict_instances_big); returns (arrays, bytes)"""
        pinned = []
        for i, t in enumerate(tensors):
            if t is None:
                pinned.append(None); continue
            p = self._pinned('out%d' % i, t.shape, t.dtype)
            p.copy_(t, non_blocking=True)
            pinned.append(p)
        torch.cuda.current_stream().synchronize()
        if copy_threads and len(tensors) == 1 and tensors[0] is not None and tensors[0].numel() >= (1 << 24) and tensors[0].is_contiguous():
            # one large map (predict_instances_big): D2H in chunks, the host copy of chunk i overlaps the transfer of chunk i+1
            import os
            t = tensors[0]
            p = self._pinned('out0', t.shape, t.dtype)
            out = torch.empty(t.shape, dtype=t.dtype)
            src, pin, dst = t.reshape(-1), p.reshape(-1), out.reshape(-1)
            n, k = t.numel(), 8
            step = -(-n // k)
            evs = []
            for i in range(k):
                a, b = i * step, min(n, (i + 1) * step)
                pin[a:b].copy_(src[a:b], non_blocking=True)
                ev = torch.cuda.Event(); ev.record(); evs.append((ev, a, b))
            nt = torch.get_num_threads()
            want = max(1, min(16, (os.cpu_count() or 1) // max(1, int(os.environ.get("LOCAL_WORLD_SIZE", "1")))))
            try:
                if want > nt: torch.set_num_threads(want)
                for ev, a, b in evs:
                    ev.synchronize()
                    dst[a:b].copy_(pin[a:b])
            finally:
                if want > nt: torch.set_num_threads(nt)
            return [out.numpy()], t.numel() * t.element_size()

        def host_copy(p):
            if copy_threads and p.numel() >= (1 << 22):
                # torchrun starts every rank with OMP_NUM_THREADS=1: give this one large copy its threads back
                import os
                nt = torch.get_num_threads()
                want = max(1, min(16, (os.cpu_count() or 1) // max(1, int(os.environ.get("LOCAL_WORLD_SIZE", "1")))))
                try:
                    if want > nt: torch.set_num_threads(want)
                    out = torch.empty(p.shape, dtype=p.dtype)
                    out.copy_(p)
                finally:
                    if want > nt: torch.set_num_threads(nt)
                return out.numpy()
            return p.numpy().copy()
        return [None if p is None else host_copy(p) for p in pinned], sum(0 if p is None else p.numel() * p.element_size() for p in pinned)

    def predict_direct_device(self, x_dev, n_tiles=None):
        """x_dev [1,...,C] float32 device -> (prob [...], dist [..., R]) device tensors (padded, /grid).
        n_tiles (axes_net order, channel entry 1): run the network tile by tile (base.py:446-529)."""
        if n_tiles is not None and int(np.prod(n_tiles)) > 1:
            prob, dist = self._predict_tiled_device(x_dev, tuple(int(t) for i, t in enumerate(n_tiles) if i != len(n_tiles) - 1))
        else:
            prob, dist = self.net.forward(x_dev)
            prob, dist = prob[0], dist[0]
            pc = getattr(self.net, 'prob_class', None)
            self._last_class = None if pc is None else pc[0]      # multi-class models: [..., n_classes+1] softmax map
        self._last = (prob, dist)
        return prob, dist

    def _predict_tiled_device(self, x_dev, n_tiles_sp):
        """The padded input is split into n_tiles blocks per spatial axis (block borders on multiples of
        pool^depth*grid); every block is extended by the network's receptive-field radius (_axes_tile_overlap, as
        the reference does), pushed through the network, and the block's own region of the prob/dist maps is kept.
        Same maps as the single pass up to float summation order (small tiles may select another conv kernel
        variant): only zero padding further than the receptive field away differs."""
        sp_axes = self.config.axes.replace('C', '')
        sp = tuple(int(v) for v in x_dev.shape[1:-1])
        nd = len(sp)
        div = self._axes_div_by(sp_axes)
        grid = tuple(self.config.grid)
        ov = tuple(int(-(-o // d) * d) for o, d in zip(self._axes_tile_overlap(sp_axes), div))
        R = self.config.n_rays
        prob = torch.empty(tuple(s // g for s, g in zip(sp, grid)), dtype=torch.float32, device=x_dev.device)
        dist = torch.empty(prob.shape + (R,), dtype=torch.float32, device=x_dev.device)
        pclass = None
        if self._is_multiclass():
            pclass = torch.empty(prob.shape + (self.config.n_classes + 1,), dtype=torch.float32, device=x_dev.device)
        cuts = []
        for s, d, n in zip(sp, div, n_tiles_sp):
            units = s // d
            n = max(1, min(int(n), units))
            b = [round(i * units / n) * d for i in range(n + 1)]
            cuts.append([(b[i], b[i + 1]) for i in range(n) if b[i + 1] > b[i]])
        import itertools
        for block in itertools.product(*cuts):
            ext = tuple((max(0, a0 - o), min(s, a1 + o)) for (a0, a1), o, s in zip(block, ov, sp))
            xt = x_dev[(slice(None),) + tuple(slice(e0, e1) for e0, e1 in ext) + (slice(None),)].contiguous()
            p, d = self.net.forward(xt)
            src = tuple(slice((a0 - e0) // g, (a1 - e0) // g) for (a0, a1), (e0, e1), g in zip(block, ext, grid))
            dst = tuple(slice(a0 // g, a1 // g) for (a0, a1), g in zip(block, grid))
            prob[dst] = p[0][src]
            dist[dst] = d[0][src]
            if pclass is not None:
                pclass[dst] = self.net.prob_class[0][src]
        self._last_class = pclass
        return prob, dist

    def _last_maps(self):
        """(tests) padded prob / dist maps of the most recent forward pass, as numpy"""
        return self._last[0].cpu().numpy(), self._last[1].cpu().numpy()

    # ------------------------------------------------------------------ predict (dense)
    def predict(self, img, axes=None, normalizer=None, n_tiles=None, show_tile_progress=True, **predict_kwargs):
        """Dense prediction: returns (prob, dist) numpy arrays (base.py:446-529)."""
        return tuple(m.cpu().numpy() for m in self._predict_device(img, axes=axes, normalizer=normalizer, n_tiles=n_tiles))

    def _predict_device(self, img, axes=None, normalizer=None, n_tiles=None):
        """predict() with the cropped maps left in HBM: (prob, dist[, prob_class]) contiguous device tensors"""
        L.require_cuda()
        x, axes, axes_net, axes_net_div_by, _permute_axes, resizer, n_tiles, grid, grid_dict, channel = \
            self._predict_setup(img, axes, normalizer, n_tiles)
        prob_d, dist_d = self.predict_direct_device(self._to_device(x), n_tiles)
        sp_axes = axes_net.replace('C', '')
        crop = resizer.crop_slices(sp_axes, tuple(prob_d.shape))
        prob = prob_d[crop].contiguous()
        dist = dist_d[crop + (slice(None),)].contiguous()
        dist = torch.clamp_min(dist, 1e-3)                  # np.maximum(1e-3, dist), base.py:517
        if self._is_multiclass():                           # (prob, dist, prob_class), base.py:476-477,524-527
            return prob, dist, self._last_class[crop + (slice(None),)].contiguous()
        return prob, dist

    # ------------------------------------------------------------------ predict_sparse
    def _predict_sparse_device(self, img, prob_thresh=None, axes=None, normalizer=None, n_tiles=None, b=2, _zoom=None):
        """device-resident sparse prediction (base.py:541-633): returns dict of device tensors
        prob[n], dist[n,R], points_f32[n,nd] (for the NMS kernels), sorted by score."""
        L.require_cuda()
        x, axes, axes_net, axes_net_div_by, _permute_axes, resizer, n_tiles, grid, grid_dict, channel = \
            self._predict_setup(img, axes, normalizer, n_tiles, _zoom=_zoom)
        sp_axes = axes_net.replace('C', '')
        bounds = resizer.point_bounds(sp_axes)
        return self._candidates_from_device_input(self._to_device(x), bounds, prob_thresh=prob_thresh, b=b, n_tiles=n_tiles)

    def _candidates_from_device_input(self, x_dev, bounds, prob_thresh=None, b=2, n_tiles=None):
        """x_dev: padded, normalized input [1,...,C] float32 already in HBM; bounds = un-padded spatial
        extent (filter_points).  Network -> threshold/border mask -> score sort -> gather."""
        lib = L.require_cuda()
        if prob_thresh is None:
            prob_thresh = self.thresholds.prob
        grid = tuple(self.config.grid)
        self._mark('net_begin')
        sparse_store = None
        if self._use_sparse_forward(x_dev, n_tiles):
            # large volumes: features + heads slab by slab, only the dist rows above the threshold are kept (SURVEY H7)
            try:
                prob_d, store_d, slot_d = self.net.forward_candidates(x_dev, np.float32(prob_thresh))
                prob_d, dist_d, sparse_store = prob_d[0], None, (store_d, slot_d)
                self._last, self._last_class = (prob_d, None), None
            except L.StarDistB200Error as e:
                if 'fp16 overflow' not in str(e):
                    raise
        if sparse_store is None:
            prob_d, dist_d = self.predict_direct_device(x_dev, n_tiles)
        self._mark('net_end')
        cand = self._candidates_from_maps(prob_d, dist_d, bounds, np.float32(prob_thresh), b=b, sparse_store=sparse_store)
        self._mark('cand_end')
        if self._is_multiclass():                           # prob_class[inds] of the candidates, base.py:595-614
            pc = self._last_class
            cand['prob_class'] = pc.reshape(-1, pc.shape[-1]).index_select(0, cand['index'].long())
        return cand

    def _candidates_from_maps(self, prob_d, dist_d, bounds, prob_thresh, b=2, sparse_store=None):
        """device prob [...] / dist [..., R] maps (or the sparse candidate store) -> candidates with prob > prob_thresh
        (float32) outside the border b and inside bounds (un-padded extent, image pixels): dict of device tensors prob[n],
        dist[n, R], points_f32[n, nd] (index * grid), index[n] (flat map index), sorted by score (csrc/candidates.cu)."""
        lib = L.require_cuda()
        grid = tuple(self.config.grid)
        nd = self.config.n_dim
        R = self.config.n_rays
        shape = tuple(int(s) for s in prob_d.shape)
        valid = tuple(int(-(-bd // g)) for bd, g in zip(bounds, grid))     # idx*g < bound  <=>  idx < ceil(bound/g)
        if b is not None and np.isscalar(b):
            bs = ((int(b), int(b)),) * nd
        elif b is None:
            bs = ((0, 0),) * nd
        else:
            bs = tuple((max(0, int(lo)), max(0, int(hi))) for lo, hi in b)
        npix = int(np.prod(shape))
        sidx = torch.empty(npix, dtype=torch.int32, device=prob_d.device)
        sprob = torch.empty(npix, dtype=torch.float32, device=prob_d.device)
        import ctypes
        cnt = ctypes.c_int(0)
        L.check(lib.sdb_threshold_sort(L.ptr(prob_d), nd, L.iarr(shape), L.iarr(valid), L.iarr([s[0] for s in bs]),
                                      L.iarr([s[1] for s in bs]), float(prob_thresh), L.ptr(sidx), L.ptr(sprob),
                                      npix, ctypes.byref(cnt), L.stream_ptr()))
        n = int(cnt.value)
        self._last_n_cand = n
        sidx, sprob = sidx[:n], sprob[:n]
        dist_s = torch.empty((n, R), dtype=torch.float32, device=prob_d.device)
        pts_f = torch.empty((n, nd), dtype=torch.float32, device=prob_d.device)
        if sparse_store is not None:
            L.check(lib.sdb_gather_candidates_slots(L.ptr(sparse_store[0]), L.ptr(sparse_store[1]), L.ptr(sidx), n, R, nd, L.iarr(shape), L.iarr(grid),
                                                   L.ptr(dist_s), L.ptr(pts_f), L.stream_ptr()))
        else:
            L.check(lib.sdb_gather_candidates(L.ptr(dist_d), L.ptr(sidx), n, R, nd, L.iarr(shape), L.iarr(grid),
                                             L.ptr(dist_s), L.ptr(pts_f), L.stream_ptr()))
        return dict(prob=sprob, dist=dist_s, points_f32=pts_f, n=n, index=sidx)

    def _use_sparse_forward(self, x_dev, n_tiles):
        """slab-wise sparse forward (UNetDevice3DTC.forward_candidates): STARDIST_B200_SPARSE_FORWARD = 1 / 0 / auto
        (default: volumes of 2^24 voxels and more, where features + dense dist would take tens of GB)"""
        import os
        mode = os.environ.get("STARDIST_B200_SPARSE_FORWARD", "auto")
        if mode == "0" or not hasattr(self.net, 'forward_candidates') or self._is_multiclass():
            return False
        if n_tiles is not None and int(np.prod(n_tiles)) > 1:
            return False
        if tuple(self.config.grid) != (1,) * self.config.n_dim or x_dev.shape[0] != 1:
            return False
        return mode == "1" or int(np.prod(x_dev.shape[1:-1])) >= (1 << 24)

    def predict_instances_device(self, x_dev, img_shape, prob_thresh=None, nms_thresh=None, return_labels=True, **nms_kwargs):
        """predict_instances for an input that is already resident in HBM (padded, normalized,
        [1,...,C] float32).  Used by bench.py's device-resident timing and by predict_instances_big."""
        cand = self._candidates_from_device_input(x_dev, tuple(img_shape), prob_thresh=prob_thresh)
        return self._instances_from_candidates_device(tuple(img_shape), cand, nms_thresh=nms_thresh,
                                                      return_labels=return_labels, **nms_kwargs)

    def predict_sparse(self, img, prob_thresh=None, axes=None, normalizer=None, n_tiles=None, show_tile_progress=True, b=2, **predict_kwargs):
        """Sparse version of model.predict(): (prob, dist, points) flat lists (base.py:541-642).
        Candidate order is score-descending (stable), see csrc/candidates.cu."""
        r = self._predict_sparse_device(img, prob_thresh=prob_thresh, axes=axes, normalizer=normalizer, n_tiles=n_tiles, b=b)
        prob = r['prob'].cpu().numpy()
        dist = r['dist'].cpu().numpy()
        points = r['points_f32'].cpu().numpy().astype(np.int64)
        return prob, dist, points

    # ------------------------------------------------------------------ predict_instances
    def predict_instances(self, img, axes=None, normalizer=None, sparse=True, prob_thresh=None, nms_thresh=None,
                          scale=None, n_tiles=None, show_tile_progress=True, verbose=False, return_labels=True,
                          predict_kwargs=None, nms_kwargs=None, overlap_label=None, return_predict=False, _device_labels=False):
        """Predict instance segmentation from input image (base.py:645-790).

        Returns (labels, dict(coord|dist, points, prob, ...)) [, (prob, dist) when return_predict]."""
        L.require_cuda()
        if predict_kwargs is None:
            predict_kwargs = {}
        if nms_kwargs is None:
            nms_kwargs = {}
        if return_predict and sparse:
            sparse = False
            warnings.warn("Setting sparse to False because return_predict is True")
        nms_kwargs.setdefault("verbose", verbose)
        _axes = self._normalize_axes(img, axes)
        _axes_net = self.config.axes
        _permute_axes = self._make_permute_axes(_axes, _axes_net)
        _shape_inst = tuple(s for s, a in zip(_permute_axes(img).shape, _axes_net) if a != 'C')
        if scale is not None:
            from scipy import ndimage as ndi
            if isinstance(scale, numbers.Number):
                scale = tuple(scale if a in 'XYZ' else 1 for a in _axes)
            scale = tuple(scale)
            len(scale) == len(_axes) or _raise(ValueError(f"scale {scale} must be of length {len(_axes)}, i.e. one value for each of the axes {_axes}"))
            for s, a in zip(scale, _axes):
                s > 0 or _raise(ValueError("scale values must be greater than 0"))
                (s in (1, None) or a in 'XYZ') or warnings.warn(f"replacing scale value {s} for non-spatial axis {a} with 1")
            scale = tuple(s if a in 'XYZ' else 1 for s, a in zip(scale, _axes))
            verbose and print(f"scaling image by factors {scale} for axes {_axes}")
            if not sparse:
                img = ndi.zoom(img, scale, order=1)
        scale_dict = None if scale is None else dict(zip(_axes, scale))
        if sparse:
            # the zoom (ndi.zoom(img, scale, order=1), base.py:735) runs in HBM when the input qualifies (_device_prep_plan)
            cand = self._predict_sparse_device(img, prob_thresh=prob_thresh, axes=axes, normalizer=normalizer, n_tiles=n_tiles, _zoom=scale)
            if _device_labels:
                nms_kwargs = dict(nms_kwargs, device_labels=True)
            res = self._instances_from_candidates_device(_shape_inst, cand, nms_thresh=nms_thresh, scale=scale_dict,
                                                         return_labels=return_labels, overlap_label=overlap_label, **nms_kwargs)
            return res
        else:
            pred = self.predict(img, axes=axes, normalizer=normalizer, n_tiles=n_tiles)
            prob, dist = pred[0], pred[1]
            res = self._instances_from_prediction(_shape_inst, prob, dist, points=None, prob_class=(pred[2] if len(pred) > 2 else None),
                                                  prob_thresh=prob_thresh, nms_thresh=nms_thresh, scale=scale_dict,
                                                  return_labels=return_labels, overlap_label=overlap_label, **nms_kwargs)
            if return_predict:
                return res, tuple(pred)
            return res

    # ------------------------------------------------------------------ predict_instances_big
    def predict_instances_big(self, img, axes, block_size, min_overlap, context=None,
                              labels_out=None, labels_out_dtype=np.int32, show_progress=True, group=None, **kwargs):
        """Predict instance segmentation from very large input images (base.py:838-983).

        The image is covered by overlapping blocks (stardist_b200.big.BlockND.cover); every block is an
        independent predict_instances call, objects are assigned to exactly one block
        (filter_objects), label ids get a running offset in block-id order and later blocks overwrite
        earlier ones inside overlaps.  Assumption (as in the reference): every object is smaller than
        `min_overlap`, and min_overlap + 2*context < block_size.

        With an initialised torch.distributed process group (one rank per GPU) the blocks are sharded
        round-robin over the ranks and assembled on rank 0 (stardist_b200/parallel_big.py); the result
        on rank 0 is identical to the single-process result."""
        from ..big import _grid_divisible, BlockND, OBJECT_KEYS
        from ..matching import relabel_sequential
        from .. import parallel_big
        n = img.ndim
        axes = axes_check_and_normalize(axes, length=n)
        grid = self._axes_div_by(axes)
        axes_out = self.config.axes.replace('C', '')
        shape_dict = dict(zip(axes, img.shape))
        shape_out = tuple(shape_dict[a] for a in axes_out)
        if context is None:
            context = self._axes_tile_overlap(axes)
        if np.isscalar(block_size): block_size = n * [block_size]
        if np.isscalar(min_overlap): min_overlap = n * [min_overlap]
        if np.isscalar(context): context = n * [context]
        block_size, min_overlap, context = list(block_size), list(min_overlap), list(context)
        assert n == len(block_size) == len(min_overlap) == len(context)
        if 'C' in axes:
            i = axes_dict(axes)['C']
            block_size[i] = img.shape[i]
            min_overlap[i] = context[i] = 0
        block_size = tuple(_grid_divisible(g, v, name='block_size', verbose=False) for v, g, a in zip(block_size, grid, axes))
        min_overlap = tuple(_grid_divisible(g, v, name='min_overlap', verbose=False) for v, g, a in zip(min_overlap, grid, axes))
        context = tuple(_grid_divisible(g, v, name='context', verbose=False) for v, g, a in zip(context, grid, axes))
        if show_progress:
            print(f'effective: block_size={block_size}, min_overlap={min_overlap}, context={context}', flush=True)
        blocks = BlockND.cover(img.shape, axes, block_size, min_overlap, context, grid)
        want_labels = not (np.isscalar(labels_out) and bool(labels_out) is False)
        if want_labels and labels_out is not None:
            labels_out.shape == shape_out or _raise(ValueError(f"'labels_out' must have shape {shape_out} (axes {axes_out})."))
        kwargs_override = dict(axes=axes, overlap_label=None, return_labels=True, return_predict=False)
        for k, v in kwargs_override.items():
            if k in kwargs and show_progress: print(f"changing '{k}' from {kwargs[k]} to {v}", flush=True)
            kwargs[k] = v
        kwargs.pop('show_tile_progress', None)

        def process(block):
            labels, polys = self.predict_instances(block.read(img, axes=axes), **kwargs)
            labels = block.crop_context(labels, axes=axes_out)
            labels, polys = block.filter_objects(labels, polys, axes=axes_out)
            return labels, polys

        rank, world = parallel_big.rank_world(group)
        if StarDistBase._big_on_device(img, axes, shape_out, want_labels, kwargs, group) and hasattr(self, '_process_block_device'):
            # device-resident pipeline: label tiles stay in HBM from the painting kernel to the assembled map
            def process_device(block):
                return self._process_block_device(block, img, axes, axes_out, kwargs)
            labels_d, polys_all = parallel_big.run_sharded_device(blocks, process_device, shape_out, axes_out, want_labels, group=group)
            if rank != 0:
                return None, None
            if not want_labels:
                return None, polys_all
            import os, time
            t0 = time.perf_counter()
            (lab_np,), nbytes = self._to_host([labels_d], copy_threads=True)
            if os.environ.get("STARDIST_B200_BIG_TIMING") == "1":
                print("[big rank 0] %-22s %.1f ms" % ("label map D2H + copy", 1e3 * (time.perf_counter() - t0)), flush=True)
            self._stats['d2h_bytes'] = self._stats.get('d2h_bytes', 0) + nbytes
            if labels_out is None:
                labels_out = lab_np if lab_np.dtype == np.dtype(labels_out_dtype) else lab_np.astype(labels_out_dtype)
            else:
                labels_out[...] = lab_np
            return labels_out, polys_all
        if world > 1:
            return parallel_big.run_sharded(blocks, process, shape_out, axes_out, labels_out if want_labels else False,
                                            labels_out_dtype, group=group)
        if want_labels and labels_out is None:
            labels_out = np.zeros(shape_out, dtype=labels_out_dtype)
        polys_all = {}
        label_offset = 1
        for block in blocks:
            labels, polys = process(block)
            labels = relabel_sequential(labels, label_offset)[0]
            if want_labels:
                block.write(labels_out, labels, axes=axes_out)
            for k, v in polys.items():
                polys_all.setdefault(k, []).append(v)
            label_offset += len(polys['prob'])
            del labels
        polys_all = {k: (np.concatenate(v) if k in OBJECT_KEYS else v[0]) for k, v in polys_all.items()}
        return (labels_out if want_labels else None), polys_all

    @staticmethod
    def _big_on_device(img, axes, shape_out, want_labels, kwargs, group):
        """the device-resident block pipeline applies to the default (sparse) predict_instances arguments, a CUDA device,
        a NCCL (or no) process group and an assembled label map that fits next to the per-block working set"""
        import os
        if os.environ.get("STARDIST_B200_BIG", "device") != "device" or not torch.cuda.is_available():
            return False
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized() and dist.get_backend(group) != "nccl":
            return False
        if kwargs.get('sparse', True) is False or kwargs.get('scale') is not None or kwargs.get('return_labels') is False:
            return False
        free, _ = torch.cuda.mem_get_info()
        return int(np.prod(shape_out)) * 4 * 2 < 0.5 * free

    def _process_block_device(self, block, img, axes, axes_out, kwargs):
        """One block of predict_instances_big without leaving HBM: predict_instances (label image kept on the device) ->
        crop_context -> filter_objects (per-label bounding boxes by sdb_label_bbox, the responsibility rule of
        big.py:89-122 vectorised on the small box table, foreign objects removed and ids compacted by sdb_label_remap).
        Returns (tile int32 device tensor with ids 1..n_kept in ascending order of the original ids, polys dict (host,
        global coordinates), n_kept) -- the same objects BlockND.filter_objects + relabel_sequential keep."""
        import ctypes
        from ..big import OBJECT_KEYS, COORD_KEYS
        lib = L.require_cuda()
        lab_d, polys = self.predict_instances(block.read(img, axes=axes), _device_labels=True, **kwargs)
        nd = lab_d.dim()
        tile = lab_d[block.slice_crop_context(axes_out)].contiguous()
        nk = len(polys['prob'])
        dev = tile.device
        bbox_d = torch.empty((nk + 1) * 6 + 1, dtype=torch.int32, device=dev)
        L.check(lib.sdb_label_bbox(L.ptr(tile), nd, L.iarr(tile.shape), nk, L.ptr(bbox_d), L.ptr(bbox_d[(nk + 1) * 6:]), L.stream_ptr()))
        bb = bbox_d.cpu().numpy()
        if bb[-1]:
            raise L.StarDistB200Error("predict_instances_big: label outside [0, n_objects] in a block")
        bb = bb[:-1].reshape(nk + 1, 6)[1:]
        bmin, bmax = bb[:, 3 - nd:3], bb[:, 6 - nd:6] + 1
        present = bmax[:, -1] > bmin[:, -1]
        ids = np.nonzero(present)[0]                       # object index = label - 1
        mine, invisible = block.responsible_many(bmin[ids], bmax[ids], axes_out)
        if invisible.any():                                # big.py:377-381
            i = int(np.nonzero(invisible)[0][0])
            shape_object = tuple(int(b - a) for a, b in zip(bmin[ids[i]], bmax[ids[i]]))
            shape_min_overlap = tuple(t.min_overlap for t in block.blocks_for_axes(axes_out))
            raise RuntimeError(f"Found object of shape {shape_object}, which violates the assumption of being smaller than 'min_overlap' {shape_min_overlap}. Increase 'min_overlap' to avoid this problem.")
        ind = ids[mine]
        lut = np.zeros(nk + 1, np.int32)
        lut[ind + 1] = np.arange(1, len(ind) + 1, dtype=np.int32)
        lut_d = torch.from_numpy(lut).to(dev, non_blocking=True)
        L.check(lib.sdb_label_remap(L.ptr(tile), tile.numel(), L.ptr(lut_d), L.stream_ptr()))
        out = {k: (v[ind] if k in OBJECT_KEYS else v) for k, v in polys.items()}
        for k in COORD_KEYS:
            if k in out:
                out[k] = block.translate_coordinates(out[k], axes=axes_out)
        return tile, out, len(ind)

    # ------------------------------------------------------------------ threshold optimisation
    def optimize_thresholds(self, X_val, Y_val, nms_threshs=[0.3, 0.4, 0.5], iou_threshs=[0.3, 0.5, 0.7], predict_kwargs=None,
                            optimize_kwargs=None, save_to_json=True):
        """Optimize the two thresholds (probability, NMS overlap) of predict_instances (base.py:986-1043).

        For every value of nms_threshs, utils.optimize_threshold finds the prob_thresh with the best matching performance on
        (X_val, Y_val), averaged over iou_threshs; the best pair becomes self.thresholds and, with save_to_json and a model
        folder, <logdir>/thresholds.json.  X_val must be normalized.  predict_kwargs go to predict (default n_tiles:
        _guess_n_tiles); optimize_kwargs to utils.optimize_threshold.  The predicted maps stay in HBM for the search."""
        from ..utils import optimize_threshold
        import sys
        if predict_kwargs is None:
            predict_kwargs = {}
        if optimize_kwargs is None:
            optimize_kwargs = {}

        def _predict_kwargs(x):
            if 'n_tiles' in predict_kwargs:
                return predict_kwargs
            return {**predict_kwargs, 'n_tiles': self._guess_n_tiles(x), 'show_tile_progress': False}

        def _predict(x, axes=None, normalizer=None, n_tiles=None, show_tile_progress=True, **kw):
            # predict()'s signature (other keywords are accepted and ignored, as there); only (prob, dist) of a multi-class model
            return self._predict_device(x, axes=axes, normalizer=normalizer, n_tiles=n_tiles)[:2]
        Yhat_val = [_predict(x, **_predict_kwargs(x)) for x in X_val]
        opt_prob_thresh, opt_measure, opt_nms_thresh = None, -np.inf, None
        for _opt_nms_thresh in nms_threshs:
            _opt_prob_thresh, _opt_measure = optimize_threshold(Y_val, Yhat_val, model=self, nms_thresh=_opt_nms_thresh,
                                                                iou_threshs=iou_threshs, **optimize_kwargs)
            if _opt_measure > opt_measure:
                opt_prob_thresh, opt_measure, opt_nms_thresh = _opt_prob_thresh, _opt_measure, _opt_nms_thresh
        opt_threshs = dict(prob=opt_prob_thresh, nms=opt_nms_thresh)
        self.thresholds = opt_threshs
        print(end='', file=sys.stderr, flush=True)
        print("Using optimized values: prob_thresh={prob:g}, nms_thresh={nms:g}.".format(prob=self.thresholds.prob, nms=self.thresholds.nms))
        if save_to_json and self.logdir is not None:
            print("Saving to 'thresholds.json'.")
            with open(self.logdir / 'thresholds.json', 'w') as f:
                json.dump({k: float(v) for k, v in opt_threshs.items()}, f)
        return opt_threshs

    def _guess_n_tiles(self, img):
        """tiles per image axis so that a tile holds about one training batch of patches (base.py:1046-1055)"""
        axes = self._normalize_axes(img, axes=None)
        shape = list(img.shape)
        if 'C' in axes:
            del shape[axes_dict(axes)['C']]
        b = self.config.train_batch_size ** (1.0 / self.config.n_dim)
        n_tiles = [int(np.ceil(s / (p * b))) for s, p in zip(shape, self.config.train_patch_size)]
        if 'C' in axes:
            n_tiles.insert(axes_dict(axes)['C'], 1)
        return tuple(n_tiles)

    # ------------------------------------------------------------------ misc
    def _compute_receptive_field(self, img_size=None):
        """base.py:1068-1098: empirical receptive field from the response to a unit impulse"""
        from scipy.ndimage import zoom
        if img_size is None:
            img_size = tuple(g * (128 if self.config.n_dim == 2 else 64) for g in self.config.grid)
        if np.isscalar(img_size):
            img_size = (img_size,) * self.config.n_dim
        img_size = tuple(img_size)
        assert all(_is_power_of_2(s) for s in img_size)
        mid = tuple(s // 2 for s in img_size)
        x = np.zeros((1,) + img_size + (self.config.n_channel_in,), dtype=np.float32)
        z = np.zeros_like(x)
        x[(0,) + mid + (slice(None),)] = 1
        dev = self.net.device
        y = self.net.forward(torch.from_numpy(x).to(dev))[0][0].cpu().numpy()
        y0 = self.net.forward(torch.from_numpy(z).to(dev))[0][0].cpu().numpy()
        grid = tuple((np.array(x.shape[1:-1]) / np.array(y.shape)).astype(int))
        assert grid == tuple(self.config.grid)
        y = zoom(y, grid, order=0)
        y0 = zoom(y0, grid, order=0)
        ind = np.where(np.abs(y - y0) > 0)
        if any(len(i) == 0 for i in ind):
            untrained = type(self)(self.config, name=None, basedir=None)
            return untrained._compute_receptive_field(img_size=img_size)
        return [(m - np.min(i), np.max(i) - m) for (m, i) in zip(mid, ind)]

    def _axes_tile_overlap(self, query_axes):
        query_axes = axes_check_and_normalize(query_axes)
        try:
            self._tile_overlap
        except AttributeError:
            self._tile_overlap = self._compute_receptive_field()
        overlap = dict(zip(self.config.axes.replace('C', ''), tuple(max(rf) for rf in self._tile_overlap)))
        return tuple(overlap.get(a, 0) for a in query_axes)


def load_weights_npz(path):
    z = np.load(path)
    names = sorted(set(k.rsplit('/', 1)[0] for k in z.files))
    return {n: (z[n + '/kernel'], z[n + '/bias']) for n in names}
