"""Threshold engine of optimize_threshold / StarDistBase.optimize_thresholds (stardist/utils.py:271-307, models/base.py:986-1043).

The reference evaluates every probe threshold t of its golden-section search from scratch: _instances_from_prediction (NMS and
label painting) and matching_dataset per image.  For one image and nms_thresh, all probes t >= t_floor share one computation:

1. candidates are ordered by descending score, so those with prob > t are a prefix of those with prob > t_floor;
2. greedy NMS decides a candidate from its pair decisions with earlier candidates only, so the survivors at t are the first
   k(t) survivors at t_floor;
3. each pixel shows the covering polygon that is first in paint priority (prob, ties by list index), and ids are
   survivor index + 1, so the label map at t is where(L_floor <= k(t), L_floor, 0).

Hence the overlap table of ground truth g against survivor r is computed once per (image, nms_thresh) on the device
(ImageTables), and a probe only restricts its columns to r <= k(t) (probe_overlap).  k(t) counts survivors with
float64(prob) > t, the comparison the reference makes (a float32 map against a float64 threshold); the device selection at the
floor uses a float32 threshold at or below t_floor, a superset.  The per-probe matrix is the one `matching` builds from the
label images, so the assignment and the accumulation are the reference's (matching.matching_from_overlap, accumulate_matching).
"""
import numpy as np
import torch

from . import _lib as L
from .matching import matching_from_overlap, accumulate_matching, relabel_sequential_device, label_overlap_device


def float32_at_or_below(t):
    """largest float32 f with f <= t: `prob > f` (float32) selects a superset of `float64(prob) > t`"""
    f = np.float32(t)
    if float(f) > float(t):
        f = np.nextafter(f, np.float32(-np.inf))
    return f


class ImageTables:
    """Everything a probe needs of one (image, nms_thresh): ground-truth row totals (row 0 = background), the survivors'
    scores (descending, float64), each survivor's painted area and the sparse overlap entries (g, r, count) with r >= 1."""

    def __init__(self, n_true, row_total, surv_prob, area, g, r, count):
        self.n_true, self.row_total, self.surv_prob = int(n_true), row_total, surv_prob
        self.area, self.g, self.r, self.count = area, g, r, count

    @classmethod
    def from_pairs(cls, n_true, surv_prob, pairs, counts):
        """pairs [m, 2] (ground truth id 0..n_true, survivor id 0..n_surv) and their counts, host arrays"""
        surv_prob = np.asarray(surv_prob, np.float32).astype(np.float64)
        g, r, c = pairs[:, 0].astype(np.int64), pairs[:, 1].astype(np.int64), np.asarray(counts, np.int64)
        row_total = np.zeros(n_true + 1, np.int64)
        np.add.at(row_total, g, c)
        area = np.zeros(len(surv_prob) + 1, np.int64)
        np.add.at(area, r, c)
        fg = r >= 1
        return cls(n_true, row_total, surv_prob, area[1:], g[fg], r[fg], c[fg])

    def probe_overlap(self, t):
        """overlap matrix (n_true + 1) x (n_kept + 1) of `matching` at prob_thresh t: the survivors with float64(prob) > t that
        painted a pixel, in ascending id order; column 0 takes whatever the kept columns do not"""
        k = int(np.count_nonzero(self.surv_prob > t))
        col = np.zeros(k + 1, np.int64)
        col[1:] = np.cumsum(self.area[:k] > 0)
        m = np.zeros((self.n_true + 1, int(col[-1]) + 1), np.int64)
        sel = self.r <= k
        m[self.g[sel], col[self.r[sel]]] = self.count[sel]
        m[:, 0] = self.row_total - m[:, 1:].sum(axis=1)
        return m


def dataset_matching(tables, t, iou_threshs, criterion='iou'):
    """matching_dataset(Y, Y_instances(t), thresh=iou_threshs) from the per-image tables"""
    stats_all = tuple(matching_from_overlap(tab.probe_overlap(t), tuple(iou_threshs), criterion) for tab in tables)
    return accumulate_matching(stats_all, tuple(iou_threshs), criterion=criterion, by_image=False)


def _as_device(a, dtype, dev):
    if isinstance(a, torch.Tensor):
        return a.to(device=dev, dtype=dtype).contiguous()
    return torch.from_numpy(np.ascontiguousarray(a)).to(device=dev, dtype=dtype).contiguous()


def _survivors_and_labels_2d(model, img_shape, cand, nms_thresh):
    """the dense 2-D path of _instances_from_prediction on device candidates: labels painted with ids = survivor index + 1"""
    lab_d, res = model._instances_from_candidates_device(img_shape, cand, nms_thresh=nms_thresh, device_labels=True)
    return res['prob'], lab_d


def _survivors_and_labels_3d(model, img_shape, cand, nms_thresh):
    """the dense 3-D path of _instances_from_prediction (nms.py non_maximum_suppression_3d_inds: the NMS runs in the order
    np.argsort(prob, kind='stable')[::-1] of the candidate list, survivors stay in list order; polyhedron_to_label paints
    them first-cover-wins in the same order of their scores, ids = survivor index + 1) -- without relabel_sequential, which
    `matching` repeats anyway.  Every tensor handed to the library is bound to a name until the stream has used it: a
    temporary freed right after its pointer is taken goes back to the caching allocator and the next allocation reuses it."""
    from .rays3d import rays_from_json
    from .nms import _argsort_desc
    lib = L.require_cuda()
    rays = rays_from_json(model.config.rays_json)
    n, R, dev = cand['n'], model.config.n_rays, cand['dist'].device
    lab_d = torch.zeros(tuple(int(s) for s in img_shape), dtype=torch.int32, device=dev)
    if n == 0:
        return np.zeros(0, np.float32), lab_d
    verts_d = torch.from_numpy(np.ascontiguousarray(rays.vertices, np.float32)).to(dev)
    faces_d = torch.from_numpy(np.ascontiguousarray(rays.faces, np.int32)).to(dev)
    prob_h = cand['prob'].cpu().numpy()
    order = torch.from_numpy(np.ascontiguousarray(_argsort_desc(prob_h))).to(dev)
    dist_o = cand['dist'].index_select(0, order).contiguous()
    pts_o = cand['points_f32'].index_select(0, order).contiguous()
    keep_o = torch.zeros(n, dtype=torch.uint8, device=dev)
    L.check(lib.sdb_nms3d(L.ptr(dist_o), L.ptr(pts_o), L.ptr(verts_d), L.ptr(faces_d), n, R, int(faces_d.shape[0]),
                          float(np.float32(nms_thresh)), 1, 1, 0, L.ptr(keep_o), L.stream_ptr()))
    keep = torch.empty_like(keep_o)
    keep[order] = keep_o
    sel = torch.nonzero(keep, as_tuple=False).flatten()
    nk = int(sel.numel())
    probi = prob_h[sel.cpu().numpy()]
    if nk == 0:
        return probi, lab_d
    paint = np.ascontiguousarray(np.argsort(probi, kind='stable')[::-1])
    paint_d = sel.index_select(0, torch.from_numpy(paint).to(dev))
    ids_d = torch.from_numpy(paint + 1).to(device=dev, dtype=torch.int32)
    dist_p = cand['dist'].index_select(0, paint_d).contiguous()
    pts_p = cand['points_f32'].index_select(0, paint_d).contiguous()
    L.check(lib.sdb_polyhedron_to_label(L.ptr(dist_p), L.ptr(pts_p), L.ptr(verts_d), L.ptr(faces_d), nk, R, int(faces_d.shape[0]),
                                        L.ptr(ids_d), int(img_shape[0]), int(img_shape[1]), int(img_shape[2]), 0, 0, 0,
                                        L.ptr(lab_d), L.stream_ptr()))
    torch.cuda.current_stream().synchronize()
    return probi, lab_d


def image_tables(model, y, prob, dist, nms_thresh, t_floor):
    """ImageTables of one validation image: ground truth y (host label image), prob / dist maps as `predict` returns them
    (host arrays or device tensors), for every probe t >= t_floor"""
    L.require_cuda()
    dev = prob.device if isinstance(prob, torch.Tensor) else torch.device('cuda', torch.cuda.current_device())
    prob_d, dist_d = _as_device(prob, torch.float32, dev), _as_device(dist, torch.float32, dev)
    img_shape = tuple(int(s) for s in np.shape(y))
    bounds = tuple(int(s) * g for s, g in zip(prob_d.shape, model.config.grid))     # the whole map: predict() already cropped it
    cand = model._candidates_from_maps(prob_d, dist_d, bounds, float32_at_or_below(t_floor), b=2)
    paint = _survivors_and_labels_2d if model.config.n_dim == 2 else _survivors_and_labels_3d
    surv_prob, lab_d = paint(model, img_shape, cand, nms_thresh)
    y = np.asarray(y)
    if not (np.issubdtype(y.dtype, np.integer) and (y.size == 0 or (y.min() >= 0 and y.max() <= np.iinfo(np.int32).max))):
        raise ValueError("y_true must be an array of non-negative integers.")
    gt_d = torch.from_numpy(np.ascontiguousarray(y, np.int32)).to(dev)
    gt_d, _, n_true = relabel_sequential_device(gt_d, max_label=int(y.max()) if y.size else 0)
    pairs, counts = label_overlap_device(gt_d, lab_d.contiguous())
    return ImageTables.from_pairs(n_true, surv_prob, pairs.cpu().numpy(), counts.cpu().numpy())
