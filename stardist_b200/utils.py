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
