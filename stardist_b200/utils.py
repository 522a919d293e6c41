"""Host-side helpers that the prediction path needs.

Reference: stardist/utils.py:54-77 (_is_power_of_2, _normalize_grid); csbdeep.utils
(axes_check_and_normalize, axes_dict, normalize -- csbdeep is an un-vendored dependency of the
reference, setup.py:140; behaviour restated from its documented semantics).
"""
import numpy as np
from collections.abc import Iterable


def _raise(e):
    raise e


def _is_power_of_2(i):
    assert i > 0
    e = np.log2(i)
    return e == int(e)


def _normalize_grid(grid, n):
    # stardist/utils.py:60-77
    try:
        grid = tuple(grid)
        (len(grid) == n and all(map(np.isscalar, grid)) and all(map(_is_power_of_2, grid))) or _raise(TypeError())
        return tuple(int(g) for g in grid)
    except (TypeError, AssertionError):
        raise ValueError("grid = {grid} must be a list/tuple of length {n} with values that are power of 2".format(grid=grid, n=n))


def axes_check_and_normalize(axes, length=None, disallowed=None, return_allowed=False):
    """S(ample), T(ime), C(hannel), Z, Y, X"""
    allowed = 'STCZYX'
    axes is not None or _raise(ValueError('axis cannot be None.'))
    axes = str(axes).upper()
    for a in axes:
        a in allowed or _raise(ValueError("invalid axis '%s', must be one of %s." % (a, list(allowed))))
        (disallowed is None or a not in disallowed) or _raise(ValueError("disallowed axis '%s'." % a))
        axes.count(a) == 1 or _raise(ValueError("axis '%s' occurs more than once." % a))
    (length is None or len(axes) == length) or _raise(ValueError('axes (%s) must be of length %d.' % (axes, length)))
    return (axes, allowed) if return_allowed else axes


def axes_dict(axes):
    axes, allowed = axes_check_and_normalize(axes, return_allowed=True)
    return {a: None if axes.find(a) == -1 else axes.find(a) for a in allowed}


def move_image_axes(x, fr, to, adjust_singletons=False):
    fr = axes_check_and_normalize(fr, length=x.ndim)
    to = axes_check_and_normalize(to)
    fr_initial, x_shape_initial = fr, x.shape
    adjust_singletons = bool(adjust_singletons)
    if adjust_singletons:
        # remove axes not present in 'to'
        slices = [slice(None) for _ in x.shape]
        for i, a in enumerate(fr):
            if (a not in to) and (x.shape[i] == 1):
                slices[i] = 0
                fr = fr.replace(a, '')
        x = x[tuple(slices)]
        # add dummy axes present in 'to'
        for i, a in enumerate(to):
            if a not in fr:
                x = np.expand_dims(x, -1)
                fr += a
    if set(fr) != set(to):
        _adjusted = '(adjusted to %s and %s) ' % (x.shape, fr) if adjust_singletons else ''
        raise ValueError('image with shape %s and axes %s %snot compatible with target axes %s.'
                         % (x_shape_initial, fr_initial, _adjusted, to))
    ax_from, ax_to = axes_dict(fr), axes_dict(to)
    if fr == to:
        return x
    return np.moveaxis(x, [ax_from[a] for a in fr], [ax_to[a] for a in fr])


def normalize(x, pmin=3, pmax=99.8, axis=None, clip=False, eps=1e-20, dtype=np.float32):
    """Percentile-based image normalization (csbdeep.utils.normalize)."""
    mi = np.percentile(x, pmin, axis=axis, keepdims=True)
    ma = np.percentile(x, pmax, axis=axis, keepdims=True)
    return normalize_mi_ma(x, mi, ma, clip=clip, eps=eps, dtype=dtype)


def normalize_mi_ma(x, mi, ma, clip=False, eps=1e-20, dtype=np.float32):
    if dtype is not None:
        x = x.astype(dtype, copy=False)
        mi = dtype(mi) if np.isscalar(mi) else mi.astype(dtype, copy=False)
        ma = dtype(ma) if np.isscalar(ma) else ma.astype(dtype, copy=False)
        eps = dtype(eps)
    x = (x - mi) / (ma - mi + eps)
    if clip:
        x = np.clip(x, 0, 1)
    return x


def _is_floatarray(x):
    return isinstance(x.dtype.type(0), np.floating)


def optimize_threshold(Y, Yhat, model, nms_thresh, measure='accuracy', iou_threshs=[0.3, 0.5, 0.7], bracket=None, tol=1e-2, maxiter=20, verbose=1):
    """Tune prob_thresh for a fixed nms_thresh to maximise `measure` of matching_dataset averaged over iou_threshs
    (stardist/utils.py:271-307): a golden-section search over prob_thresh in `bracket` (default: half the largest prob to
    the largest).  Y: ground-truth label images, Yhat: (prob, dist) per image as `model.predict` returns them (numpy arrays;
    device tensors are used in place).  Returns (prob_thresh, value).

    Same search and values as the reference; each value comes from the threshold engine (stardist_b200/optimize.py), which
    runs the NMS, label painting and overlap table once per image and restricts them to each probe."""
    import datetime
    from scipy.optimize import minimize_scalar
    from . import optimize as E
    np.isscalar(nms_thresh) or _raise(ValueError("nms_thresh must be a scalar"))
    iou_threshs = [iou_threshs] if np.isscalar(iou_threshs) else iou_threshs
    values = dict()

    if bracket is None:
        max_prob = max([(np.float32(prob.max().item()) if hasattr(prob, 'is_cuda') else np.max(prob)) for prob, dist in Yhat])
        bracket = max_prob / 2, max_prob
    tables = [E.image_tables(model, y, prob, dist, nms_thresh, t_floor=min(bracket)) for y, (prob, dist) in zip(Y, Yhat)]

    def fn(thr):
        prob_thresh = np.clip(thr, *bracket)
        value = values.get(prob_thresh)
        if value is None:
            stats = E.dataset_matching(tables, prob_thresh, iou_threshs)
            values[prob_thresh] = value = np.mean([s._asdict()[measure] for s in stats])
        if verbose > 1:
            print("{now}   thresh: {prob_thresh:f}   {measure}: {value:f}".format(
                now=datetime.datetime.now().strftime('%H:%M:%S'), prob_thresh=prob_thresh, measure=measure, value=value), flush=True)
        return -value

    opt = minimize_scalar(fn, method='golden', bracket=bracket, tol=tol, options={'maxiter': maxiter})
    verbose > 1 and print('\n', opt, flush=True)
    return opt.x, -opt.fun


def edt_prob(lbl_img, anisotropy=None):
    """Perform EDT on each labeled object and normalize. (stardist/utils.py:71-125)

    Equal to the reference's scipy variant bit for bit: one multi-label exact distance transform of the whole map on the
    device (stardist_b200/labelprep.py, csrc/labelprep.cu) instead of one scipy call per object."""
    from .labelprep import edt_prob as _edt_prob
    return _edt_prob(lbl_img, anisotropy=anisotropy)


def fill_label_holes(lbl_img, **kwargs):
    """Fill small holes in label image. (stardist/utils.py:137-153)

    All labels at once on the device (stardist_b200/labelprep.py); kwargs as binary_fill_holes takes them, with `structure`
    one of generate_binary_structure(ndim, c)."""
    from .labelprep import fill_label_holes as _fill_label_holes
    return _fill_label_holes(lbl_img, **kwargs)


def calculate_extents(lbl, func=np.median):
    """ Aggregate bounding box sizes of objects in label images. (stardist/utils.py:180-193)

    The bounding boxes come from sdb_region_stats on the device, one per label in ascending label order, as regionprops
    lists them."""
    if (isinstance(lbl, np.ndarray) and lbl.ndim == 4) or (not isinstance(lbl, np.ndarray) and isinstance(lbl, Iterable)):
        return func(np.stack([calculate_extents(_lbl, func) for _lbl in lbl], axis=0), axis=0)

    n = lbl.ndim
    n in (2, 3) or _raise(ValueError("label image should be 2- or 3-dimensional (or pass a list of these)"))

    from .geometry.distances import label_map_to_device, region_stats_device
    seq, n_labels, _ = label_map_to_device(lbl)
    if n_labels == 0:
        return np.zeros(n)
    _, _, bmin, bmax = region_stats_device(seq, n_labels)
    extents = (bmax.to(dtype=bmin.dtype) - bmin + 1).cpu().numpy().astype(np.int64)
    return func(extents, axis=0)


def grid_divisible_patch_size(patch_size, grid, warn=True):
    # stardist/utils.py:397-403
    import warnings
    patch_size, grid = tuple(patch_size), tuple(grid)
    assert len(patch_size) == len(grid)
    patch_size_divisible = tuple(int(np.ceil(sh / g) * g) for sh, g in zip(patch_size, grid))
    if patch_size != patch_size_divisible and warn:
        warnings.warn(f"increasing patch_size from {patch_size} to {patch_size_divisible}, since it was not evenly divisible by grid {grid}")
    return patch_size_divisible


def _invert_dict(d):
    """ return  v-> [k_1,k_2,k_3....] for k,v in d"""
    from collections import defaultdict
    res = defaultdict(list)
    for k, v in d.items():
        res[v].append(k)
    return res


_INT32_MAX = int(np.iinfo(np.int32).max)


def _class_code(cls, n_classes):
    """the class-map code of one class id (stardist/utils.py:365-372): -1 for None, else the id in 0..n_classes"""
    if cls is None:
        return -1
    if np.issubdtype(type(cls), np.integer) and 0 <= cls <= n_classes:
        return int(cls)
    raise ValueError(f"Wrong class id '{cls}' (for n_classes={n_classes})")


def mask_to_categorical(y, n_classes, classes, return_cls_dict=False):
    """generates a multi-channel categorical class map (stardist/utils.py:318-380)

    y: integer label array (labels below 2^31), or a contiguous CUDA int32 tensor; n_classes: number of object classes
    (without background); classes: dict {label -> class_id} with class_id 0 (background), 1..n_classes or None (ignored
    object: -1 in the object channels), or a single integer / None broadcast to every label of y.

    Returns the probability map float32 y.shape + (n_classes + 1,) (first channel is background), as numpy for numpy input
    and as a CUDA tensor for a CUDA tensor, and with return_cls_dict also the inverted dict {class_id -> [labels]}.
    The labels of y are found on the device (sdb_stack_labels), only their id list comes back to be checked against the
    dict, and one pass writes the map (sdb_label_class_map).  A dict's class ids are checked before the device is used, so a
    dict with both a wrong class id and a missing label reports the class id."""
    import torch
    from . import _lib as L
    from .matching import _check_label_array, stack_labels_device
    is_tensor = isinstance(y, torch.Tensor)
    if is_tensor:
        if not (y.is_cuda and y.dtype == torch.int32 and y.is_contiguous()):
            raise ValueError("mask_to_categorical expects a contiguous CUDA int32 tensor (or a numpy label array)")
    else:
        _check_label_array(y, 'y')
        if np.iinfo(y.dtype).max > _INT32_MAX and y.size and int(y.max()) > _INT32_MAX:
            raise ValueError("mask_to_categorical: labels must be below 2^31")
    if not (np.issubdtype(type(n_classes), np.integer) and n_classes >= 1):
        raise ValueError(f"n_classes is '{n_classes}' but should be a positive integer")
    broadcast = np.issubdtype(type(classes), np.integer) or classes is None
    if not (broadcast or isinstance(classes, dict)):
        raise ValueError("classes should be dict, single scalar, or None!")
    if not broadcast:
        for cls in _invert_dict(classes):
            _class_code(cls, n_classes)

    lib = L.require_cuda()
    shape = tuple(y.shape)
    d_y = y if is_tensor else torch.from_numpy(np.ascontiguousarray(y, dtype=np.int32)).cuda()
    try:
        ids, _ = stack_labels_device(d_y.reshape(1, -1))
    except ValueError:
        raise ValueError("y must be an array of non-negative integers.")
    y_labels = ids.tolist()
    if broadcast:
        classes = dict((k, classes) for k in y_labels)
    if not set(y_labels).issubset(set(classes.keys())):
        raise ValueError(f"all gt labels should be present in class dict provided \ngt_labels found\n{set(y_labels)}\nclass dict labels provided\n{set(classes.keys())}")
    cls_dict = _invert_dict(classes)
    for cls in cls_dict:
        _class_code(cls, n_classes)

    codes = np.array([_class_code(classes[k], n_classes) for k in y_labels], np.int32)
    d_keys = torch.from_numpy(np.ascontiguousarray(ids, np.int32)).cuda()
    d_codes = torch.from_numpy(codes).cuda()
    out = torch.empty(shape + (n_classes + 1,), dtype=torch.float32, device=d_y.device)
    L.check(lib.sdb_label_class_map(L.ptr(d_y), d_y.numel(), L.ptr(d_keys), L.ptr(d_codes), len(y_labels), int(n_classes),
                                    L.ptr(out), L.stream_ptr()))
    y_mask = out if is_tensor else out.cpu().numpy()
    return (y_mask, cls_dict) if return_cls_dict else y_mask


def _mask_compact_device(mask, nonzero, lo, hi, prob=None):
    """The set elements of the box [lo, hi) of a mask (numpy array or CUDA tensor of bool / integers, at most 4-D), in C order,
    compacted on the device (sdb_mask_compact_count / _write): a tuple of int32 host coordinate arrays, one per axis, and the
    float32 values of `prob` (a CUDA float32 tensor of the mask's shape, or None) at them.  nonzero: an element is set when it
    is non-zero (np.where), else when its low bit is (numpy's mask & 1)."""
    import ctypes, torch
    from . import _lib as L
    lib = L.require_cuda()
    if isinstance(mask, torch.Tensor):
        d_m = mask.contiguous()
        elem = d_m.element_size()
    else:
        m = np.ascontiguousarray(mask)
        elem = m.itemsize
        d_m = torch.from_numpy(m.view(np.uint8).reshape(-1)).cuda()
    ndim, shape = len(lo), tuple(int(s) for s in mask.shape)
    rows = int(np.prod([max(0, h - l) for l, h in zip(lo[:-1], hi[:-1])], dtype=np.int64))
    pre = torch.empty(rows + 1, dtype=torch.int64, device='cuda')
    args = (L.ptr(d_m), elem, int(bool(nonzero)), ndim, L.larr(shape), L.larr(lo), L.larr(hi))
    h_n = ctypes.c_longlong(0)
    L.check(lib.sdb_mask_compact_count(*args, L.ptr(pre), ctypes.byref(h_n), L.stream_ptr()))
    n = int(h_n.value)
    coords = torch.empty((ndim, n), dtype=torch.int32, device='cuda')
    w = torch.empty(n, dtype=torch.float32, device='cuda') if prob is not None else None
    L.check(lib.sdb_mask_compact_write(*args, L.ptr(pre), n, L.ptr(coords), L.ptr(prob), L.ptr(w), L.stream_ptr()))
    return tuple(coords.cpu().numpy()), (None if w is None else w.cpu().numpy())


def sample_points(n_samples, mask, prob=None, b=2):
    """sample points to draw some of the associated polygons (stardist/utils.py:156-177)

    Candidates are the set pixels of `mask & 1` (a 2-D bool or integer mask) at least `b` pixels inside the border (every
    pixel for b None or 0), in C order; they are drawn with np.random.choice(n, n_samples, replace=True), weighted by `prob`
    at the candidates when it is given.  Returns int64 [n_samples, 2] (y, x).

    The candidates are compacted on the device, which also gathers `prob` there when it is a CUDA float32 tensor (a numpy
    `prob` is read on the host at the candidates); the mask may be a numpy array or a CUDA bool / integer tensor, e.g. from a
    device-resident predict.  The draw makes the reference's numpy calls on the candidates, so points and np.random's state
    are the reference's.  Deliberate difference: a mask that is not 2-D raises ValueError."""
    import torch
    is_tensor = isinstance(mask, torch.Tensor)
    use_border = b is not None and b > 0
    if is_tensor:
        if not mask.is_cuda or mask.dtype.is_floating_point or mask.dtype.is_complex:
            raise TypeError("sample_points: a tensor mask must be a CUDA bool or integer tensor")
    else:
        mask = np.asanyarray(mask)
        if not (mask.dtype == bool or np.issubdtype(mask.dtype, np.integer)):
            empty = np.zeros(0, mask.dtype)
            empty & (empty if use_border else True)                         # numpy's own TypeError
    if mask.ndim != 2:
        raise ValueError("sample_points: mask must be 2-dimensional (it has %d dimensions)" % mask.ndim)
    shape = tuple(int(s) for s in mask.shape)
    if use_border:
        box = [slice(b, -b).indices(s)[:2] for s in shape]                  # mask_b[b:-b, b:-b] = True
    else:
        box = [(0, s) for s in shape]
    lo, hi = [l for l, _ in box], [max(l, h) for l, h in box]
    d_prob = prob if isinstance(prob, torch.Tensor) else None
    if d_prob is not None and not (d_prob.is_cuda and d_prob.dtype == torch.float32 and tuple(d_prob.shape) == shape):
        raise ValueError("sample_points: a tensor prob must be a CUDA float32 tensor of the mask's shape")
    points, w = _mask_compact_device(mask, False, lo, hi, None if d_prob is None else d_prob.contiguous())
    points = tuple(p.astype(np.intp) for p in points)

    if prob is not None:
        # weighted sampling via prob
        w = (w if d_prob is not None else prob[points[0], points[1]]).astype(np.float64)
        w /= np.sum(w)
        ind = np.random.choice(len(points[0]), n_samples, replace=True, p=w)
    else:
        ind = np.random.choice(len(points[0]), n_samples, replace=True)

    points = points[0][ind], points[1][ind]
    points = np.stack(points, axis=-1)
    return points

