"""numpy restatement of edt_prob and fill_label_holes from their whole-image definitions (the contract of csrc/labelprep.cu).

edt_prob: a pixel p of label l > 0 has d2(p) = min over pixels q of the image with a label != l (background, negative and
other labels alike) of sum_a ((q_a - p_a) * s_a)^2, summed in float64 in axis order 0, 1, ...; positions outside the image
do not count, except for a constant image with a positive label, where those just outside it do.  prob(p) =
float32(sqrt(d2(p)) / (sqrt(max of d2 over label l) + 1e-10)); every other pixel is 0.

fill_label_holes: for a label i > 0, let B be its bounding box grown by one pixel on every side that does not touch the image
border.  A hole of i is a pixel of B with a label != i that no path of label-!=-i pixels of B (under
generate_binary_structure(ndim, c)) joins to the boundary of B.  out(p) = the largest i such that p has label i or is a hole
of i, 0 where there is none, in the input's dtype.

`edt_prob_brute` evaluates the minimum over all pixels (small maps only).  `edt_prob_boxes` gets the same d2 per object from
scipy's exact distance transform of the object's mask in its grown box (pixels farther than the box's outer layer are never
the nearest); the CPU tests pin it to the brute force, and it serves the sizes the brute force cannot reach."""
import numpy as np
from scipy import ndimage as ndi


def _constant(lbl):
    return lbl.size > 0 and lbl.min() == lbl.max() and lbl.flat[0] > 0


def _sampling(anisotropy, ndim):
    if anisotropy is None:
        return np.ones(ndim)
    s = np.asarray(anisotropy, np.float64)
    return np.full(ndim, float(s)) if s.ndim == 0 else s


def _normalise(lbl, d2):
    prob = np.zeros(lbl.shape, np.float32)
    for l in np.unique(lbl[lbl > 0]):
        m = lbl == l
        d = np.sqrt(d2[m])
        prob[m] = d / (np.sqrt(d2[m].max()) + 1e-10)
    return prob


def edt_prob_brute(lbl, anisotropy=None):
    lbl = np.asarray(lbl)
    nd, s = lbl.ndim, _sampling(anisotropy, lbl.ndim)
    coords = np.indices(lbl.shape).reshape(nd, -1).T
    flat = lbl.ravel()
    d2 = np.zeros(flat.shape)
    black = _constant(lbl)
    for l in np.unique(flat[flat > 0]):
        P = coords[flat == l]
        Q = coords[flat != l]
        best = np.full(len(P), np.inf)
        for q0 in range(0, len(Q), 256):
            q = Q[q0:q0 + 256]
            dd = np.zeros((len(P), len(q)))
            for a in range(nd):
                t = (q[None, :, a] - P[:, None, a]).astype(np.float64) * s[a]
                dd = dd + t * t
            best = np.minimum(best, dd.min(axis=1)) if len(q) else best
        if black:
            for a in range(nd):
                for e in (-1, lbl.shape[a]):
                    t = (e - P[:, a]).astype(np.float64) * s[a]
                    dd = np.zeros(len(P))
                    for b in range(nd):
                        dd = dd + (t * t if b == a else 0.0)
                    best = np.minimum(best, dd)
        d2[flat == l] = best
    return _normalise(lbl, d2.reshape(lbl.shape))


def grown_boxes(lbl):
    """[(label, grown box slices)] for every positive label, ascending"""
    labels = np.unique(lbl[lbl > 0])
    seq = np.where(lbl > 0, np.searchsorted(labels, lbl) + 1, 0)
    return [(labels[k], tuple(slice(max(x.start - 1, 0), min(x.stop + 1, n)) for x, n in zip(sl, lbl.shape)))
            for k, sl in enumerate(ndi.find_objects(seq))]


def edt_prob_boxes(lbl, anisotropy=None):
    lbl = np.asarray(lbl)
    s = _sampling(anisotropy, lbl.ndim)
    black = _constant(lbl)
    work = np.pad(lbl, 1) if black else lbl
    prob = np.zeros(work.shape, np.float32)
    for l, box in grown_boxes(work):
        mask = work[box] == l
        d = ndi.distance_transform_edt(mask, sampling=s)[mask]
        prob[box][mask] = d / (d.max() + 1e-10)
    return prob[(slice(1, -1),) * lbl.ndim] if black else prob


def fill_label_holes_def(lbl, connectivity=1):
    lbl = np.asarray(lbl)
    st = ndi.generate_binary_structure(lbl.ndim, connectivity)
    out = np.zeros(lbl.shape, np.int64)
    for l, box in grown_boxes(lbl):
        other = lbl[box] != l
        cc, _ = ndi.label(other, st)
        edge = np.zeros(other.shape, bool)
        for a in range(other.ndim):
            idx = [slice(None)] * other.ndim
            idx[a] = 0; edge[tuple(idx)] = True
            idx[a] = -1; edge[tuple(idx)] = True
        reach = np.unique(cc[edge & other])
        filled = ~other | (other & ~np.isin(cc, reach))
        view = out[box]
        view[filled] = np.maximum(view[filled], int(l))
    return out.astype(lbl.dtype)


def random_labels(rng, shape, density=0.02, drop=0.05, negative=False):
    """seeded label map: grown seeds in a random order, touching objects, holes punched by background pixels"""
    seeds = rng.random(shape) < density
    m, n = ndi.label(seeds)
    lab = ndi.grey_dilation(m, size=(5,) * len(shape))
    lab[rng.random(shape) < drop] = 0
    perm = np.r_[0, rng.permutation(max(n, 1))[:n] + 1]
    lab = perm[lab].astype(np.int32)
    if negative:
        lab[rng.random(shape) < 0.05] = -1
    return lab
