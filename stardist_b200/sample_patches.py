"""Patch sampling (stardist/sample_patches.py): sample_patches draws random crops of equally shaped arrays, get_valid_inds
lists the crop centres a patch filter allows.

The draw is the reference's on the host (csbdeep's `choice`, restated in models/data.py, so np.random and `random` advance
as they do there); the crops are copied by one device gather per array (sdb_gather_patches), element words copied as they
are, so values cannot change.  A filter's mask is compacted on the device (sdb_mask_compact_*).  Numpy arrays come back as
numpy, CUDA tensors as CUDA tensors.  Arrays and masks may have at most 4 dimensions (ValueError above)."""
import numpy as np

from .utils import _raise

_WORDS = (1, 2, 4, 8, 16)


def _crop_shapes(rand_inds, patch_size, shape):
    """start and clipped extent of every drawn crop: numpy's slicing of
    data[tuple(slice(_r-(_p//2),_r+_p-(_p//2)) for _r,_p in zip(r,patch_size))] (sample_patches.py:31), computed on the
    same scalars"""
    starts, extents = [], []
    for r in zip(*rand_inds):
        st, ex = [], []
        for _r, _p, s in zip(r, patch_size, shape):
            a, b, _ = slice(_r - (_p // 2), _r + _p - (_p // 2)).indices(s)
            st.append(a); ex.append(max(0, b - a))
        starts.append(st); extents.append(tuple(ex))
    return starts, extents


def _gather(data, starts, extent):
    """the crops of `data` at `starts` [n][ndim] with shape `extent`, stacked: numpy for numpy, a CUDA tensor for one"""
    import torch
    from . import _lib as L
    lib = L.require_cuda()
    n = len(starts)
    if isinstance(data, torch.Tensor):
        src = data.contiguous()
        out = torch.empty((n,) + tuple(extent), dtype=src.dtype, device=src.device)
        elem, shape, ext, st = src.element_size(), tuple(src.shape), tuple(extent), np.asarray(starts, np.int64)
    else:
        a = np.ascontiguousarray(data)
        elem, shape, ext, st = a.itemsize, a.shape, tuple(extent), np.asarray(starts, np.int64).reshape(n, a.ndim)
        if elem not in _WORDS:                                   # any other element type: its bytes, one more axis
            shape, ext, elem = shape + (elem,), ext + (elem,), 1
            st = np.concatenate([st, np.zeros((n, 1), np.int64)], axis=1)
        src = torch.from_numpy(a.view(np.uint8).reshape(-1)).cuda()
        out = torch.empty(n * int(np.prod(ext, dtype=np.int64)) * elem, dtype=torch.uint8, device='cuda')
    if len(shape) > 4:
        raise ValueError("sample_patches: arrays with more than 4 dimensions (counting the bytes of an element that is not "
                         "1, 2, 4, 8 or 16 bytes wide) are not supported")
    d_st = torch.from_numpy(np.ascontiguousarray(st, np.int64)).cuda()
    L.check(lib.sdb_gather_patches(L.ptr(src), elem, len(shape), L.larr(shape), L.larr(ext), L.ptr(d_st), n, L.ptr(out),
                                   L.stream_ptr()))
    if isinstance(data, torch.Tensor):
        return out
    return out.cpu().numpy().view(a.dtype).reshape((n,) + tuple(extent))


def sample_patches(datas, patch_size, n_samples, valid_inds=None, verbose=False):
    """optimized version of csbdeep.data.sample_patches_from_multiple_stacks (stardist/sample_patches.py:7-35)

    datas: equally shaped numpy arrays or CUDA tensors (any element type); returns one stack of n_samples patches per array.
    Without valid_inds the centres are those of the reference, np.meshgrid (default 'xy' indexing) of
    arange(p//2, s-p//2+1) per axis; for odd p that range includes centres whose crops numpy clips at the far border.  As in
    the reference, clipped crops are returned when all drawn crops have one shape, and np.stack's ValueError is raised
    otherwise."""
    from .models.data import choice

    len(patch_size) == datas[0].ndim or _raise(ValueError())

    if not all((a.shape == datas[0].shape for a in datas)):
        raise ValueError("all input shapes must be the same: %s" % (" / ".join(str(a.shape) for a in datas)))

    if not all((0 < s <= d for s, d in zip(patch_size, datas[0].shape))):
        raise ValueError("patch_size %s negative or larger than data shape %s along some dimensions" % (str(patch_size), str(datas[0].shape)))

    shape = tuple(int(s) for s in datas[0].shape)
    if valid_inds is None:
        # the reference's meshgrid without building it: its raveled position -> one index per axis ('xy' swaps axes 0 and 1)
        ranges = tuple(np.arange(p // 2, s - p // 2 + 1) for s, p in zip(shape, patch_size))
        lens = tuple(len(r) for r in ranges)
        n_valid = int(np.prod(lens, dtype=np.int64))
        grid_shape = (lens[1], lens[0]) + lens[2:] if len(lens) > 1 else lens
    else:
        n_valid = len(valid_inds[0])

    if n_valid == 0:
        raise ValueError("no regions to sample from!")

    idx = choice(range(n_valid), n_samples, replace=(n_valid < n_samples))
    if valid_inds is None:
        u = np.unravel_index(np.asarray(idx, np.int64), grid_shape)
        u = (u[1], u[0]) + tuple(u[2:]) if len(lens) > 1 else u
        rand_inds = [r[k] for r, k in zip(ranges, u)]
    else:
        rand_inds = [v[idx] for v in valid_inds]

    starts, extents = _crop_shapes(rand_inds, patch_size, shape)
    if len(set(extents)) != 1:
        np.stack([np.empty(e, np.uint8) for e in extents])                 # np.stack's own ValueError
    return [_gather(data, starts, extents[0]) for data in datas]


def get_valid_inds(img, patch_size, patch_filter=None):
    """
    Returns all indices of an image that
    - can be used as center points for sampling patches of a given patch_size, and
    - are part of the boolean mask given by the function patch_filter (if provided)

    img: np.ndarray
    patch_size: tuple of ints
        the width of patches per img dimension,
    patch_filter: None or callable
        a function with signature patch_filter(img, patch_size) returning a boolean mask (numpy, or a CUDA bool / uint8
        tensor), compacted on the device

    (stardist/sample_patches.py:38-66): uint32 index arrays, one per axis.
    """
    import torch

    len(patch_size) == img.ndim or _raise(ValueError())

    if not all((0 < s <= d for s, d in zip(patch_size, img.shape))):
        raise ValueError("patch_size %s negative or larger than image shape %s along some dimensions" % (str(patch_size), str(img.shape)))

    if patch_filter is None:
        # only cut border indices (which is faster)
        valid_inds = tuple(np.arange(p // 2, s - p + p // 2 + 1).astype(np.uint32) for p, s in zip(patch_size, img.shape))
        return tuple(s.ravel() for s in np.meshgrid(*valid_inds, indexing='ij'))

    patch_mask = patch_filter(img, patch_size)
    if isinstance(patch_mask, torch.Tensor):
        if not (patch_mask.is_cuda and patch_mask.dtype in (torch.bool, torch.uint8)):
            raise ValueError("get_valid_inds: a tensor patch mask must be a CUDA bool or uint8 tensor")
    else:
        patch_mask = np.asarray(patch_mask)
        if patch_mask.dtype != bool:
            patch_mask = patch_mask.astype(bool)                             # np.where's truth value of any dtype
    if patch_mask.ndim != len(patch_size):
        raise ValueError("get_valid_inds: patch_filter returned a %d-dimensional mask for a %d-dimensional image"
                         % (patch_mask.ndim, len(patch_size)))
    if patch_mask.ndim > 4:
        raise ValueError("get_valid_inds: masks with more than 4 dimensions are not supported")
    # the border slices (p // 2, s - p + p // 2 + 1), as numpy clips them to the mask
    box = [slice(p // 2, s - p + p // 2 + 1).indices(int(m))[:2] for p, s, m in zip(patch_size, img.shape, patch_mask.shape)]
    from .utils import _mask_compact_device
    coords, _ = _mask_compact_device(patch_mask, True, [a for a, _ in box], [max(a, b) for a, b in box])
    return tuple(c.astype(np.uint32) for c in coords)
