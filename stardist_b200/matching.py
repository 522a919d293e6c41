"""relabel_sequential (stardist/matching.py:319-406; itself taken from scikit-image) -- host-side
integer bookkeeping used by StarDist3D._instances_from_prediction (model3d.py:645) and
predict_instances_big (base.py:959)."""
import os
import numpy as np

from .utils import _raise


def relabel_sequential(label_field, offset=1):
    """Relabel arbitrary labels to {`offset`, ... `offset` + number_of_labels}.
    Returns (relabeled, forward_map, inverse_map); label 0 is background and never remapped."""
    offset = int(offset)
    if offset <= 0:
        raise ValueError("Offset must be strictly positive.")
    if np.min(label_field) < 0:
        raise ValueError("Cannot relabel array that contains negative values.")
    max_label = int(label_field.max())
    if not np.issubdtype(label_field.dtype, np.integer):
        new_type = np.min_scalar_type(max_label)
        label_field = label_field.astype(new_type)
    labels = np.unique(label_field)
    labels0 = labels[labels != 0]
    new_max_label = offset - 1 + len(labels0)
    new_labels0 = np.arange(offset, new_max_label + 1)
    output_type = label_field.dtype
    required_type = np.min_scalar_type(new_max_label)
    if np.dtype(required_type).itemsize > np.dtype(label_field.dtype).itemsize:
        output_type = required_type
    forward_map = np.zeros(max_label + 1, dtype=output_type)
    forward_map[labels0] = new_labels0
    inverse_map = np.zeros(new_max_label + 1, dtype=output_type)
    inverse_map[offset:] = labels0
    relabeled = forward_map[label_field]
    return relabeled, forward_map, inverse_map


def relabel_sequential_device(label_field, offset=1, max_label=None):
    """relabel_sequential (stardist/matching.py:319-406) on a device int32 label map, IN PLACE (sdb_relabel_sequential).
    Returns (label_field, forward_map[max_label + 1] device int32, n_labels).  `max_label`: an upper bound of the values
    (default: computed on the device).  No CPU fallback: raises without the CUDA library."""
    import ctypes, torch
    from . import _lib as L
    lib = L.require_cuda()
    if not (isinstance(label_field, torch.Tensor) and label_field.is_cuda and label_field.dtype == torch.int32 and label_field.is_contiguous()):
        raise ValueError("relabel_sequential_device expects a contiguous CUDA int32 tensor")
    if int(offset) <= 0:
        raise ValueError("Offset must be strictly positive.")
    if max_label is None:
        max_label = int(label_field.max()) if label_field.numel() else 0
    fwd = torch.empty(int(max_label) + 3, dtype=torch.int32, device=label_field.device)
    cnt = ctypes.c_int(0)
    rc = lib.sdb_relabel_sequential(L.ptr(label_field), label_field.numel(), int(max_label), int(offset), L.ptr(fwd), ctypes.byref(cnt), L.stream_ptr())
    if rc != 0:
        msg = L.load().sdb_last_error().decode('utf-8', 'replace')
        if 'negative' in msg:
            raise ValueError("Cannot relabel array that contains negative values.")
        L.check(rc)
    return label_field, fwd[:int(max_label) + 1], int(cnt.value)




def label_overlap_device(a, b, capacity=1 << 16):
    """Sparse label-overlap table of two device int32 label maps of the same shape (sdb_label_overlap): every distinct pair
    (a[i], b[i]), background 0 included, sorted by (a, b).  Returns (pairs [m, 2] int32, counts [m] int64), device tensors.
    `capacity`: first guess of the number of pairs; when it is too small the call is repeated once with the bound the
    kernel reports.  Negative labels raise ValueError.  No CPU fallback: raises without the CUDA library."""
    import ctypes, torch
    from . import _lib as L
    lib = L.require_cuda()
    for t in (a, b):
        if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == torch.int32 and t.is_contiguous()):
            raise ValueError("label_overlap_device expects contiguous CUDA int32 tensors")
    if a.shape != b.shape:
        raise ValueError("x and y must have the same shape")
    n = a.numel()
    cap = max(1, min(int(capacity), max(n, 1)))
    for attempt in range(2):
        pairs = torch.empty((cap, 2), dtype=torch.int32, device=a.device)
        counts = torch.empty(cap, dtype=torch.int64, device=a.device)
        m = ctypes.c_longlong(0)
        rc = lib.sdb_label_overlap(L.ptr(a), L.ptr(b), n, L.ptr(pairs), L.ptr(counts), cap, ctypes.byref(m), L.stream_ptr())
        if rc != 0:
            if 'negative' in L.load().sdb_last_error().decode('utf-8', 'replace'):
                raise ValueError("label maps must be arrays of non-negative integers.")
            L.check(rc)
        if m.value <= cap:
            return pairs[:m.value], counts[:m.value]
        cap = int(m.value)
    raise L.StarDistB200Error("label_overlap: %d pairs do not fit the reported bound %d" % (m.value, cap))


# ---------------------------------------------------------------------------------------------------------
# Detection metrics (stardist/matching.py:13-314).  Host-side evaluation: pairs ground-truth and predicted objects by an
# optimal assignment on the IoU (or IoT / IoP) matrix and counts tp / fp / fn at one or several thresholds.
MATCHING_CRITERIA = ('iou', 'iot', 'iop')
_DATASET_KEYS = frozenset(('fp', 'tp', 'fn', 'precision', 'recall', 'accuracy', 'f1', 'criterion', 'thresh', 'n_true', 'n_pred',
                           'mean_true_score', 'mean_matched_score', 'panoptic_quality'))


def label_are_sequential(y):
    """True if y has only the labels 1..max (and 0)"""
    labels = np.unique(y)
    return (set(labels) - {0}) == set(range(1, 1 + labels.max()))


def _check_label_array(y, name=None, check_sequential=False):
    err = ValueError("{label} must be an array of {integers}.".format(
        label='labels' if name is None else name, integers=('sequential ' if check_sequential else '') + 'non-negative integers'))
    if not (isinstance(y, np.ndarray) and np.issubdtype(y.dtype, np.integer)):
        raise err
    if len(y) == 0:
        return True
    if check_sequential:
        label_are_sequential(y) or _raise(err)
    else:
        y.min() >= 0 or _raise(err)
    return True


def label_overlap(x, y, check=True):
    """overlap[i, j] = number of pixels with label i in x and j in y, shape (1 + x.max(), 1 + y.max()), dtype np.uint
    (stardist/matching.py:38-52).  With check, both must be arrays of sequential non-negative integers of one shape."""
    if check:
        _check_label_array(x, 'x', True)
        _check_label_array(y, 'y', True)
        x.shape == y.shape or _raise(ValueError("x and y must have the same shape"))
    return _overlap_matrix(x, y).astype(np.uint)


def _overlap_matrix(a, b):
    """counts[i, j] = number of pixels with label i in a and j in b (labels already sequential, 0 = background)"""
    na, nb = int(a.max()) + 1, int(b.max()) + 1
    flat = a.ravel().astype(np.int64) * nb + b.ravel().astype(np.int64)
    return np.bincount(flat, minlength=na * nb).reshape(na, nb)


def _ratio(num, den):
    out = np.zeros(np.broadcast(num, den).shape, np.float32)
    np.divide(num, den, out=out, where=np.abs(den) > 1e-10)
    return out


def intersection_over_union(overlap):
    """overlap / (n_pixels_true + n_pixels_pred - overlap) as float32, 0 where the denominator is 0; an all-zero overlap
    is returned as it is (stardist/matching.py:65-72)"""
    _check_label_array(overlap, 'overlap')
    if np.sum(overlap) == 0:
        return overlap
    n_pixels_pred = np.sum(overlap, axis=0, keepdims=True)
    n_pixels_true = np.sum(overlap, axis=1, keepdims=True)
    return _ratio(overlap, n_pixels_pred + n_pixels_true - overlap)


def intersection_over_true(overlap):
    """overlap / n_pixels_true (row sums) as float32 (stardist/matching.py:77-82)"""
    _check_label_array(overlap, 'overlap')
    if np.sum(overlap) == 0:
        return overlap
    return _ratio(overlap, np.sum(overlap, axis=1, keepdims=True))


def intersection_over_pred(overlap):
    """overlap / n_pixels_pred (column sums) as float32 (stardist/matching.py:87-92)"""
    _check_label_array(overlap, 'overlap')
    if np.sum(overlap) == 0:
        return overlap
    return _ratio(overlap, np.sum(overlap, axis=0, keepdims=True))


_CRITERION_FUNCTIONS = dict(iou=intersection_over_union, iot=intersection_over_true, iop=intersection_over_pred)


def _criterion_scores(overlap, criterion):
    criterion in _CRITERION_FUNCTIONS or _raise(ValueError("Matching criterion '%s' not supported." % criterion))
    return _CRITERION_FUNCTIONS[criterion](overlap)


def matching_from_overlap(overlap, thresh=0.5, criterion='iou', report_matches=False, map_rev_true=None, map_rev_pred=None):
    """The metrics of `matching` from the overlap matrix of two sequentially labelled images (row / column 0 = background):
    one Matching for a scalar `thresh`, a tuple of them for a sequence (stardist/matching.py:155-230).  `map_rev_true` /
    `map_rev_pred` map sequential ids back to the original ones for `report_matches` (default: identity)."""
    from collections import namedtuple
    from scipy.optimize import linear_sum_assignment
    criterion in MATCHING_CRITERIA or _raise(ValueError("Matching criterion '%s' not supported." % criterion))
    if thresh is None:
        thresh = 0
    single = np.isscalar(thresh)
    threshs = (float(thresh),) if single else tuple(map(float, thresh))
    scores = _criterion_scores(overlap, criterion)[1:, 1:]
    n_true, n_pred = scores.shape
    n_matched = min(n_true, n_pred)
    rev_t = (lambda i: int(i)) if map_rev_true is None else (lambda i: int(map_rev_true[i]))
    rev_p = (lambda j: int(j)) if map_rev_pred is None else (lambda j: int(map_rev_pred[j]))

    def _single(thr):
        tp, sum_matched = 0, 0.0
        if n_matched > 0:
            # maximise the number of pairs above the threshold, ties broken by the summed score (:185-190)
            costs = -(scores >= thr).astype(float) - scores / (2 * n_matched)
            ti, pi = linear_sum_assignment(costs)
            ok = scores[ti, pi] >= thr
            tp = np.count_nonzero(ok)                      # numpy integer scalar, as in the reference: float32 / np.int64 -> float64 below
            sum_matched = np.sum(scores[ti, pi][ok])       # stays float32 like the reference's (matching.py:190): the means below are float32 quotients
        fp, fn = n_pred - tp, n_true - tp
        div = lambda a, b: (a / b) if np.abs(b) > 1e-10 else 0.0       # _safe_divide on scalars (matching.py:55-58)
        # scalar types follow the reference's expressions (matching.py:180-196) so that the float results are the same numbers:
        # sum (float32) / n_true (int) stays float32, / tp (numpy int) and / (tp + fp/2 + fn/2) are float64 quotients
        fields = dict(criterion=criterion, thresh=thr, fp=fp, tp=tp, fn=fn,
                      precision=(tp / (tp + fp) if tp > 0 else 0), recall=(tp / (tp + fn) if tp > 0 else 0),
                      accuracy=(tp / (tp + fp + fn) if tp > 0 else 0), f1=((2 * tp) / (2 * tp + fp + fn) if tp > 0 else 0),
                      n_true=n_true, n_pred=n_pred, mean_true_score=div(sum_matched, n_true),
                      mean_matched_score=div(sum_matched, tp), panoptic_quality=div(sum_matched, tp + fp / 2 + fn / 2))
        if bool(report_matches):
            if n_matched > 0:                              # matching.py:208-219: every assigned pair, also those below thr
                fields.update(matched_pairs=tuple((rev_t(i), rev_p(j)) for i, j in zip(1 + ti, 1 + pi)),
                              matched_scores=tuple(scores[ti, pi]), matched_tps=tuple(map(int, np.flatnonzero(ok))))
            else:
                fields.update(matched_pairs=(), matched_scores=(), matched_tps=())
        return namedtuple('Matching', fields.keys())(*fields.values())

    return _single(threshs[0]) if single else tuple(map(_single, threshs))


def matching(y_true, y_pred, thresh=0.5, criterion='iou', report_matches=False):
    """Matching(criterion, thresh, fp, tp, fn, precision, recall, accuracy, f1, n_true, n_pred, mean_true_score,
    mean_matched_score, panoptic_quality) between two label images (stardist/matching.py:109-232).  `thresh` may be a
    sequence: then a tuple with one Matching per value.  report_matches adds matched_pairs (original ids), matched_scores
    and matched_tps."""
    for name, y in (('y_true', y_true), ('y_pred', y_pred)):
        if not (isinstance(y, np.ndarray) and np.issubdtype(y.dtype, np.integer) and (y.size == 0 or y.min() >= 0)):
            raise ValueError("%s must be an array of non-negative integers." % name)
    if y_true.shape != y_pred.shape:
        raise ValueError("y_true and y_pred have different shapes")
    criterion in MATCHING_CRITERIA or _raise(ValueError("Matching criterion '%s' not supported." % criterion))
    yt, _, rev_t = relabel_sequential(y_true)
    yp, _, rev_p = relabel_sequential(y_pred)
    return matching_from_overlap(_overlap_matrix(yt, yp), thresh, criterion, report_matches, rev_t, rev_p)


def accumulate_matching(stats_all, thresh, criterion='iou', by_image=False):
    """DatasetMatching per threshold from per-image results (stardist/matching.py:270-314): stats_all holds, per image, the
    tuple of Matching results for the thresholds `thresh` (a sequence).  Counts are summed; with by_image the ratios are
    averaged over images, otherwise recomputed from the summed counts (mean_true_score accumulates as v * n_true)."""
    from collections import namedtuple
    n_images = len(stats_all)
    accumulate = [{} for _ in thresh]
    for stats in stats_all:
        for acc, s in zip(accumulate, stats):
            for k, v in s._asdict().items():
                if k == 'mean_true_score' and not bool(by_image):
                    acc[k] = acc.setdefault(k, 0) + v * s.n_true          # -> "sum_matched_score"
                else:
                    try:
                        acc[k] = acc.setdefault(k, 0) + v
                    except TypeError:
                        pass
    div = lambda a, b: (a / b) if np.abs(b) > 1e-10 else 0.0
    for thr, acc in zip(thresh, accumulate):
        set(acc.keys()) == _DATASET_KEYS or _raise(ValueError("unexpected keys"))
        acc['criterion'] = criterion
        acc['thresh'] = thr
        acc['by_image'] = bool(by_image)
        if bool(by_image):
            for k in ('precision', 'recall', 'accuracy', 'f1', 'mean_true_score', 'mean_matched_score', 'panoptic_quality'):
                acc[k] /= n_images
        else:
            tp, fp, fn, n_true = acc['tp'], acc['fp'], acc['fn'], acc['n_true']
            sum_matched_score = acc['mean_true_score']
            acc.update(precision=(tp / (tp + fp) if tp > 0 else 0), recall=(tp / (tp + fn) if tp > 0 else 0),
                       accuracy=(tp / (tp + fp + fn) if tp > 0 else 0), f1=((2 * tp) / (2 * tp + fp + fn) if tp > 0 else 0),
                       mean_true_score=div(sum_matched_score, n_true), mean_matched_score=div(sum_matched_score, tp),
                       panoptic_quality=div(sum_matched_score, tp + fp / 2 + fn / 2))
    return tuple(namedtuple('DatasetMatching', acc.keys())(*acc.values()) for acc in accumulate)


def matching_dataset(y_true, y_pred, thresh=0.5, criterion='iou', by_image=False, show_progress=True, parallel=False):
    """matching metrics for lists of images, see `matching` (stardist/matching.py:234-240).  show_progress and parallel are
    accepted for compatibility; the images are evaluated in order."""
    len(y_true) == len(y_pred) or _raise(ValueError("y_true and y_pred must have the same length."))
    return matching_dataset_lazy(tuple(zip(y_true, y_pred)), thresh=thresh, criterion=criterion, by_image=by_image,
                                 show_progress=show_progress, parallel=parallel)


def matching_dataset_lazy(y_gen, thresh=0.5, criterion='iou', by_image=False, show_progress=True, parallel=False):
    """matching_dataset over an iterable of (y_true, y_pred) pairs (stardist/matching.py:244-314): one DatasetMatching for a
    scalar thresh, a tuple for a sequence."""
    single = np.isscalar(thresh)
    threshs = (thresh,) if single else tuple(thresh)
    stats_all = tuple(matching(y_t, y_p, thresh=threshs, criterion=criterion, report_matches=False) for y_t, y_p in y_gen)
    acc = accumulate_matching(stats_all, threshs, criterion=criterion, by_image=by_image)
    return acc[0] if single else acc


# ---------------------------------------------------------------------------------------------------------
# group_matching_labels (stardist/matching.py:409-472): objects of consecutive frames are linked greedily, frame i + 1 against
# the grouped frame i.  Grouping only renames the objects of frame i (one-to-one), so the overlap of the original frames i,
# i + 1 on their compacted ids is the overlap `matching` builds, up to the order of its rows: `matching` relabels the grouped
# frame sequentially, i.e. rows in ascending order of the grouped ids, and linear_sum_assignment breaks ties by that order.
# _group_chain therefore re-orders each pair's rows by the grouped ids before the assignment.  The overlap tables come from
# the device (sdb_stack_overlap) or from numpy; _group_chain serves both.
_INT32_MAX = int(np.iinfo(np.int32).max)


def _compact_labels(y):
    """(ids, compacted): the sorted non-zero labels of y, and y with each label replaced by 1 + its index in ids (0 stays 0),
    as int32 -- the numbering of relabel_sequential, without its dense forward map of max(y) + 1 entries"""
    u, inv = np.unique(y, return_inverse=True)
    inv = inv.reshape(y.shape).astype(np.int32)
    if u.size and u[0] == 0:
        return u[1:], inv
    return u, inv + 1


def _group_chain(ids, overlap, thresh, criterion):
    """Grouped ids of every object of every frame.  ids[f]: the sorted non-zero labels of frame f; overlap(p): the dense
    int64 overlap of frames p and p + 1 on their compacted ids, (1 + len(ids[p])) x (1 + len(ids[p + 1])).  Returns luts:
    luts[f][k] is the grouped id of the label ids[f][k]; frame 0 keeps its labels."""
    luts = [np.asarray(ids[0], np.int64)]
    next_id = int(luts[0].max()) + 1 if luts[0].size else 1                       # ys_grouped[0].max() + 1
    for p in range(len(ids) - 1):
        g = luts[p]
        order = np.argsort(g)                                                        # grouped ids are distinct
        rows = np.concatenate(([0], 1 + order))
        res = matching_from_overlap(overlap(p)[rows], thresh, criterion, report_matches=True,
                                    map_rev_true=np.concatenate(([0], g[order])))
        lut = np.full(len(ids[p + 1]), -1, np.int64)
        for k in res.matched_tps:
            gid, j = res.matched_pairs[k]
            lut[j - 1] = gid
        new = np.flatnonzero(lut < 0)                                               # ascending label order, as regionprops
        if new.size and next_id + new.size - 1 > _INT32_MAX:
            raise ValueError("group_matching_labels: more than 2^31 - 1 label ids are needed (the result is int32)")
        lut[new] = next_id + np.arange(new.size)
        next_id += int(new.size)
        luts.append(lut)
    return luts


def _check_group_input(ys, criterion):
    """the checks of stardist/matching.py:441-450, then labels below 2^31 and a supported criterion"""
    len(ys) > 1 or _raise(ValueError("'ys' must have 2 or more entries"))
    if isinstance(ys, np.ndarray):
        _check_label_array(ys, 'ys')
        ys.ndim > 1 or _raise(ValueError("'ys' must be at least 2-dimensional"))
    else:
        all(_check_label_array(y, 'ys') for y in ys) or _raise(ValueError("'ys' must be a list of label images"))
        all(y.shape == ys[0].shape for y in ys) or _raise(ValueError("all label images must have the same shape"))
    for y in ((ys,) if isinstance(ys, np.ndarray) else ys):
        if np.iinfo(y.dtype).max > _INT32_MAX and y.size and int(y.max()) > _INT32_MAX:
            raise ValueError("group_matching_labels: labels must be below 2^31 (the result is int32)")
    criterion in MATCHING_CRITERIA or _raise(ValueError("Matching criterion '%s' not supported." % criterion))


def _device_ready():
    import torch
    from . import _lib as L
    return torch.cuda.is_available() and os.path.exists(L.LIB_PATH)


def group_matching_labels(ys, thresh=1e-10, criterion='iou'):
    """Group matching objects of consecutive label images (e.g. the frames of a time-lapse) under one id
    (stardist/matching.py:409-472).  Frame i + 1 is matched against the grouped frame i with `matching` (`thresh`,
    `criterion`); its matched objects take the id of their partner, the others new ids in ascending order of their label,
    counting up from ys[0].max() + 1.

    ys: an integer array [T, ...] or a list / tuple of equally shaped integer label images, T >= 2, labels in [0, 2^31);
    returns an np.int32 array [T, ...] whose frame 0 is ys[0].  A contiguous CUDA int32 tensor [T, ...] is also accepted
    and gives a CUDA int32 tensor; only the per-frame id lists and per-pair overlap tables then leave the device.
    With the CUDA library the overlaps and the relabelling run on the device, otherwise in numpy; the result is the same."""
    import torch
    if isinstance(ys, torch.Tensor):
        len(ys) > 1 or _raise(ValueError("'ys' must have 2 or more entries"))
        ys.ndim > 1 or _raise(ValueError("'ys' must be at least 2-dimensional"))
        if not (ys.is_cuda and ys.dtype == torch.int32 and ys.is_contiguous()):
            raise ValueError("group_matching_labels expects a contiguous CUDA int32 tensor (or numpy label arrays)")
        criterion in MATCHING_CRITERIA or _raise(ValueError("Matching criterion '%s' not supported." % criterion))
        return _group_device(ys, thresh, criterion)
    _check_group_input(ys, criterion)
    if _device_ready():
        stack = torch.from_numpy(np.ascontiguousarray(np.stack([np.asarray(y, np.int32) for y in ys]))).cuda()
        return _group_device(stack, thresh, criterion).cpu().numpy()
    return _group_host(ys, thresh, criterion)


def _group_host(ys, thresh, criterion):
    """group_matching_labels on the host: the overlaps from numpy (_overlap_matrix on compacted frames)"""
    ids, comp = zip(*(_compact_labels(np.asarray(y, np.int32)) for y in ys))
    luts = _group_chain(ids, lambda p: _overlap_matrix(comp[p], comp[p + 1]), thresh, criterion)
    out = np.empty((len(ys),) + comp[0].shape, np.int32)
    out[0] = ys[0]
    for f in range(1, len(ys)):
        out[f] = np.concatenate(([0], luts[f]))[comp[f]]
    return out


def _table_device(call, capacity):
    """(keys, counts) host int64 arrays of one sdb_stack_* table call under the capacity protocol of label_overlap_device,
    or None when the table needs more than 2^28 entries"""
    import ctypes, torch
    from . import _lib as L
    cap = max(1, min(int(capacity), 1 << 28))
    for attempt in range(2):
        keys = torch.empty(cap, dtype=torch.int64, device='cuda')
        counts = torch.empty(cap, dtype=torch.int64, device='cuda')
        m = ctypes.c_longlong(0)
        rc = call(L.ptr(keys), L.ptr(counts), cap, ctypes.byref(m))
        if rc != 0:
            if 'negative' in L.load().sdb_last_error().decode('utf-8', 'replace'):
                raise ValueError("ys must be an array of non-negative integers.")
            L.check(rc)
        if m.value <= cap:
            return keys[:m.value].cpu().numpy(), counts[:m.value].cpu().numpy()
        if m.value > (1 << 28):
            return None
        cap = int(m.value)
    raise L.StarDistB200Error("stack table: %d keys do not fit the reported bound %d" % (m.value, cap))


def stack_labels_device(stack, capacity=1 << 16):
    """The sorted non-zero labels of every frame of a contiguous CUDA int32 stack [T, ...] (sdb_stack_labels).  Returns
    host arrays (ids int32, offsets int64 [T + 1]): the labels of frame f are ids[offsets[f]:offsets[f + 1]].  Negative
    labels raise ValueError."""
    from . import _lib as L
    lib = L.require_cuda()
    T = int(stack.shape[0]); S = stack.numel() // max(T, 1)
    tab = _table_device(lambda k, c, cap, m: lib.sdb_stack_labels(L.ptr(stack), T, S, k, c, cap, m, L.stream_ptr()), capacity)
    if tab is None:
        raise L.StarDistB200Error("stack_labels: more than 2^28 distinct (frame, label) pairs")
    keys = tab[0]
    frame, lab = keys >> 32, (keys & 0xffffffff).astype(np.int32)
    frame, lab = frame[lab != 0], lab[lab != 0]
    return lab, np.searchsorted(frame, np.arange(T + 1)).astype(np.int64)


def stack_overlap_device(stack, ids, offsets, capacity=None, pairs_per_chunk=None):
    """Overlap tables of every consecutive frame pair of a contiguous CUDA int32 stack [T, ...] on ids compacted per frame
    (sdb_stack_overlap), in one pass over the stack per chunk of pairs.  `ids`, `offsets`: as stack_labels_device returns
    them.  Returns a list of T - 1 tuples (a, b, counts) of host int64 arrays, sorted by (a, b), with 0 for the background and
    k + 1 for the label ids[offsets[f] + k].  The key holds the pair index in the bits the compacted ids leave free; pairs
    are processed in chunks that fit there, or that `pairs_per_chunk` bounds.  `capacity`: first guess of the number of
    keys per chunk (default: from the object counts); a short guess costs one repeated call."""
    import torch
    from . import _lib as L
    lib = L.require_cuda()
    T = int(stack.shape[0]); S = stack.numel() // max(T, 1)
    n_obj = np.diff(offsets)
    w = max(1, int(n_obj.max()).bit_length() if n_obj.size else 1)
    chunk = min(max(T - 1, 1), 1 << min(63 - 2 * w, 40))
    if pairs_per_chunk is not None:
        chunk = max(1, min(chunk, int(pairs_per_chunk)))
    ids_d = torch.from_numpy(np.ascontiguousarray(ids, np.int32)).cuda()
    off_d = torch.from_numpy(np.ascontiguousarray(offsets, np.int64)).cuda()
    mask = (1 << w) - 1
    tables, p = [], 0
    while p < T - 1:
        k = min(chunk, T - 1 - p)
        cap = capacity if capacity is not None else 2 * int(n_obj[p:p + k + 1].sum() + n_obj[p + 1:p + k + 1].sum() + 2 * k)
        tab = _table_device(lambda kd, cd, c, m: lib.sdb_stack_overlap(L.ptr(stack), S, p, k, L.ptr(ids_d), L.ptr(off_d), w, kd, cd,
                                                                       c, m, L.stream_ptr()), cap)
        if tab is None:
            if k == 1:
                raise L.StarDistB200Error("stack_overlap: more than 2^28 distinct pairs in one frame pair")
            chunk = (k + 1) // 2
            continue
        keys, counts = tab
        g = keys >> (2 * w)
        cuts = np.searchsorted(g, np.arange(k + 1))
        for q in range(k):
            kk = keys[cuts[q]:cuts[q + 1]]
            tables.append(((kk >> w) & mask, kk & mask, counts[cuts[q]:cuts[q + 1]]))
        p += k
    return tables


def _group_device(stack, thresh, criterion):
    """group_matching_labels of a contiguous CUDA int32 stack: per-frame ids and overlap tables on the device, the chaining
    on the host, the grouped stack written by one pass (sdb_stack_group_remap)"""
    import torch
    from . import _lib as L
    lib = L.require_cuda()
    T = int(stack.shape[0]); S = stack.numel() // T
    ids, offsets = stack_labels_device(stack)
    tables = stack_overlap_device(stack, ids, offsets)
    per_frame = [ids[offsets[f]:offsets[f + 1]] for f in range(T)]

    def overlap(p):
        a, b, c = tables[p]
        m = np.zeros((1 + len(per_frame[p]), 1 + len(per_frame[p + 1])), np.int64)
        m[a, b] = c
        return m

    luts = _group_chain(per_frame, overlap, thresh, criterion)
    lut_d = torch.from_numpy(np.concatenate(luts).astype(np.int32)).cuda()
    ids_d = torch.from_numpy(np.ascontiguousarray(ids, np.int32)).cuda()
    off_d = torch.from_numpy(offsets).cuda()
    out = torch.empty_like(stack)
    L.check(lib.sdb_stack_group_remap(L.ptr(stack), T, S, L.ptr(ids_d), L.ptr(off_d), L.ptr(lut_d), L.ptr(out), L.stream_ptr()))
    return out
