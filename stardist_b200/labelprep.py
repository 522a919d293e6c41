"""edt_prob and fill_label_holes on the device (csrc/labelprep.cu).

Both work on a sequential relabelling of the map: negative labels become 0 (they are never an object, and like background
they count as "another label"), the positive labels become 1..n in ascending order.  The order is kept, so the largest new
id of a pixel is the new id of its largest original label, and fill_label_holes maps its result back through the inverse.
"""
import warnings
import numpy as np
from . import _lib as L

# the relabelling keeps a forward map with one int32 entry per label value (sdb_relabel_sequential)
_MAX_LABEL = 2 ** 30 - 1
_DEVICE_DTYPES = ("int8", "uint8", "int16", "uint16", "int32", "int64")


def _sampling(anisotropy, ndim):
    """float64 [ndim] sampling of scipy's distance_transform_edt (a scalar is broadcast), or None"""
    if anisotropy is None:
        return None
    s = np.asarray(anisotropy, dtype=np.float64)
    if s.ndim == 0:
        s = np.full(ndim, float(s))
    if s.shape != (ndim,):
        raise ValueError("anisotropy must be a scalar or have one value per image axis (%d), got %s" % (ndim, anisotropy))
    if not np.all(np.isfinite(s) & (s > 0)):
        raise ValueError("anisotropy values must be positive and finite, got %s" % (anisotropy,))
    return np.ascontiguousarray(s)


def _connectivity(kwargs, ndim):
    """the c of a structure generate_binary_structure(ndim, c) passed to binary_fill_holes (default 1)"""
    unknown = set(kwargs) - {"structure", "output", "origin", "axes"}
    if unknown:
        raise TypeError("binary_fill_holes() got an unexpected keyword argument '%s'" % sorted(unknown)[0])
    if kwargs.get("output") is not None:
        raise NotImplementedError("fill_label_holes: 'output' is not supported")
    if kwargs.get("axes") is not None:
        raise NotImplementedError("fill_label_holes: 'axes' is not supported")
    if np.any(np.asarray(kwargs.get("origin", 0)) != 0):
        raise NotImplementedError("fill_label_holes: only origin 0 is supported")
    structure = kwargs.get("structure")
    if structure is None:
        return 1
    st = np.asarray(structure, dtype=bool)
    if st.ndim != ndim:
        raise ValueError("structure and input must have the same dimensionality")
    if st.shape == (3,) * ndim:
        dist = np.abs(np.indices((3,) * ndim) - 1).sum(axis=0)
        for c in range(1, ndim + 1):
            if np.array_equal(st, dist <= c):
                return c
    raise NotImplementedError("fill_label_holes: structure must be generate_binary_structure(%d, c) for some c in 1..%d" % (ndim, ndim))


def _check_device_labels(lbl, what):
    import torch
    if not (isinstance(lbl, torch.Tensor) and lbl.is_cuda):
        raise ValueError("%s: expected a CUDA label tensor" % what)
    if str(lbl.dtype).replace("torch.", "") not in _DEVICE_DTYPES:
        raise ValueError("%s: label tensor must have an integer dtype among %s, got %s" % (what, ", ".join(_DEVICE_DTYPES), lbl.dtype))
    if lbl.dim() not in (2, 3):
        raise ValueError("%s: label image should be 2- or 3-dimensional, got %d dimensions" % (what, lbl.dim()))


def _relabel(lbl):
    """(sequential CUDA int32 map, n_labels, original labels in ascending order as CUDA int64, raw min, raw max); reads the
    minimum and maximum back (one synchronisation) and raises ValueError for labels above 2^30 - 1 before any launch"""
    import torch
    from .matching import relabel_sequential_device
    t = lbl.to(torch.int64 if lbl.dtype == torch.int64 else torch.int32)
    lo, hi = (int(v) for v in torch.stack([t.min().to(torch.int64), t.max().to(torch.int64)]).cpu())
    if hi > _MAX_LABEL:
        raise ValueError("labels above 2^30 - 1 are not supported")
    t = t.clamp_min(0).to(torch.int32).contiguous()
    seq, fwd, n = relabel_sequential_device(t, max_label=max(hi, 0))
    return seq, n, torch.nonzero(fwd > 0).flatten(), lo, hi


def edt_prob_device(lbl, anisotropy=None):
    """edt_prob of a CUDA integer label map [H, W] / [D, H, W] -> CUDA float32 of the same shape (sdb_edt_prob).  The result
    stays on the device; the map's minimum and maximum and the label count are read back on the way."""
    import torch
    _check_device_labels(lbl, "edt_prob")
    s = _sampling(anisotropy, lbl.dim())
    if lbl.numel() == 0:
        raise ValueError("zero-size array to reduction operation minimum which has no identity")
    lib = L.require_cuda()
    seq, n, _, lo, hi = _relabel(lbl)
    constant = lo == hi and hi > 0
    if constant:
        warnings.warn("EDT of constant label image is ill-defined. (Assuming background around it.)")
    out = torch.empty(lbl.shape, dtype=torch.float32, device=lbl.device)
    L.check(lib.sdb_edt_prob(L.ptr(seq), seq.dim(), L.iarr(seq.shape), n, L.ptr(s), int(constant), L.ptr(out), L.stream_ptr()))
    return out


def fill_label_holes_device(lbl, **kwargs):
    """fill_label_holes of a CUDA integer label map [H, W] / [D, H, W] -> CUDA tensor of the same shape and dtype
    (sdb_fill_label_holes).  kwargs as binary_fill_holes takes them: `structure` = generate_binary_structure(ndim, c),
    c = 1..ndim (default: c = 1); `origin` 0; `output` None."""
    import torch
    _check_device_labels(lbl, "fill_label_holes")
    conn = _connectivity(kwargs, lbl.dim())
    if lbl.numel() == 0:
        return torch.zeros_like(lbl)
    lib = L.require_cuda()
    seq, n, labels, _, _ = _relabel(lbl)
    out = torch.empty(seq.shape, dtype=torch.int32, device=seq.device)
    L.check(lib.sdb_fill_label_holes(L.ptr(seq), seq.dim(), L.iarr(seq.shape), n, conn, L.ptr(out), L.stream_ptr()))
    lut = torch.zeros(n + 1, dtype=torch.int64, device=seq.device)
    lut[1:] = labels
    return lut[out.to(torch.int64)].to(lbl.dtype)


def _check_host_labels(lbl_img, what):
    if not (isinstance(lbl_img, np.ndarray) and np.issubdtype(lbl_img.dtype, np.integer)):
        raise ValueError("%s: lbl_img must be a numpy array of integers" % what)
    if lbl_img.ndim not in (2, 3):
        raise ValueError("%s: label image should be 2- or 3-dimensional, got %d dimensions" % (what, lbl_img.ndim))
    if lbl_img.size and lbl_img.dtype.itemsize >= 4 and int(lbl_img.max()) > _MAX_LABEL:
        raise ValueError("labels above 2^30 - 1 are not supported")


def _to_device(lbl_img):
    """numpy integer label map -> CUDA int32 tensor with the same positive labels (values below -1 become -1: every
    negative label is treated alike)"""
    import torch
    if lbl_img.dtype.itemsize >= 4 and np.issubdtype(lbl_img.dtype, np.signedinteger):
        lbl_img = np.maximum(lbl_img, -1)
    L.require_cuda()
    return torch.from_numpy(np.ascontiguousarray(lbl_img, dtype=np.int32)).to("cuda")


def edt_prob(lbl_img, anisotropy=None):
    """Perform EDT on each labeled object and normalize.  (stardist/utils.py:71-125, the scipy variant)"""
    _check_host_labels(lbl_img, "edt_prob")
    _sampling(anisotropy, lbl_img.ndim)
    if lbl_img.size == 0:
        raise ValueError("zero-size array to reduction operation minimum which has no identity")
    return edt_prob_device(_to_device(lbl_img), anisotropy).cpu().numpy()


def fill_label_holes(lbl_img, **kwargs):
    """Fill small holes in label image.  (stardist/utils.py:137-153)"""
    _check_host_labels(lbl_img, "fill_label_holes")
    _connectivity(kwargs, lbl_img.ndim)
    if lbl_img.size == 0:
        return np.zeros_like(lbl_img)
    return fill_label_holes_device(_to_device(lbl_img), **kwargs).cpu().numpy().astype(lbl_img.dtype, copy=False)
