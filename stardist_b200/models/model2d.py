"""StarDist2D on the H100 path.

Mirrors stardist/models/model2d.py: Config2D (:123-269, in config.py), StarDist2D._build
(:310-349 -> UNetDevice2D), _instances_from_prediction (:512-563), _axes_div_by (:566-574).
"""
import numpy as np
import torch

from .. import _lib as L
from ..utils import axes_check_and_normalize, _raise
from ..nms import non_maximum_suppression, non_maximum_suppression_sparse
from ..geometry.geom2d import polygons_to_label, dist_to_coord, dist_to_coord_device, paint_order
from .base import StarDistBase
from .config import Config2D
import os
from .unet_device import UNetDevice2D, UNetDevice2DTC


class StarDist2D(StarDistBase):
    """StarDist2D model (prediction and training).

    Parameters
    ----------
    config : :class:`Config2D` or None
        If ``None``, loaded from ``<basedir>/<name>/config.json`` (must exist).
    name : str or None
    basedir : str or None
    """

    def __init__(self, config=Config2D(), name=None, basedir='.', **kwargs):
        super().__init__(config, name=name, basedir=basedir, **kwargs)

    def _build(self):
        self.config.backbone == 'unet' or _raise(NotImplementedError())
        # default: tcgen05 tensor-core path; STARDIST_B200_UNET=simt selects the exact-fp32 CUDA-core
        # kernels (also used automatically for layer shapes the tensor-core kernel does not cover)
        mode = os.environ.get("STARDIST_B200_UNET", "tc").lower()
        if mode != "simt" and UNetDevice2DTC.supported(self.config):
            return UNetDevice2DTC(self.config, self.weights)
        return UNetDevice2D(self.config, self.weights)

    # ------------------------------------------------------------------ numpy-level (reference signature)
    def _instances_from_prediction(self, img_shape, prob, dist, points=None, prob_class=None, prob_thresh=None,
                                   nms_thresh=None, overlap_label=None, return_labels=True, scale=None, **nms_kwargs):
        """
        if points is None     -> dense prediction
        if points is not None -> sparse prediction
        """
        if prob_thresh is None: prob_thresh = self.thresholds.prob
        if nms_thresh is None: nms_thresh = self.thresholds.nms
        if overlap_label is not None: raise NotImplementedError("overlap_label not supported for 2D yet!")
        if points is not None:
            points, probi, disti, indsi = non_maximum_suppression_sparse(dist, prob, points, nms_thresh=nms_thresh, **nms_kwargs)
            if prob_class is not None:
                prob_class = np.asarray(prob_class)[indsi]
        else:
            points, probi, disti = non_maximum_suppression(dist, prob, grid=self.config.grid,
                                                           prob_thresh=prob_thresh, nms_thresh=nms_thresh, **nms_kwargs)
            if prob_class is not None:                      # model2d.py:533-535
                inds = tuple(p // g for p, g in zip(points.T, self.config.grid))
                prob_class = np.asarray(prob_class)[inds]
        if scale is not None:
            if not (isinstance(scale, dict) and 'X' in scale and 'Y' in scale):
                raise ValueError("scale must be a dictionary with entries for 'X' and 'Y'")
            rescale = (1 / scale['Y'], 1 / scale['X'])
            points = points * np.array(rescale).reshape(1, 2)
        else:
            rescale = (1, 1)
        if return_labels:
            labels = polygons_to_label(disti, points, prob=probi, shape=img_shape, scale_dist=rescale)
        else:
            labels = None
        coord = dist_to_coord(disti, points, scale_dist=rescale)
        res_dict = dict(coord=coord, points=points, prob=probi)
        if prob_class is not None:                          # model2d.py:556-560
            prob_class = np.asarray(prob_class)
            res_dict.update(dict(class_prob=prob_class, class_id=np.argmax(prob_class, axis=-1)))
        return labels, res_dict

    # ------------------------------------------------------------------ device-resident (sparse) path
    def _instances_from_candidates_device(self, img_shape, cand, nms_thresh=None, scale=None, return_labels=True,
                                          overlap_label=None, use_bbox=True, use_kdtree=True, verbose=False, device_labels=False):
        """Same result as _instances_from_prediction(points=...) but on tensors that stay in HBM:
        NMS -> survivors -> dist_to_coord -> label painting; one D2H of the results at the end.
        device_labels: return the label image as a device tensor (predict_instances_big keeps it in HBM)."""
        lib = L.require_cuda()
        if nms_thresh is None: nms_thresh = self.thresholds.nms
        if overlap_label is not None: raise NotImplementedError("overlap_label not supported for 2D yet!")
        n, R = cand['n'], self.config.n_rays
        dev = cand['dist'].device
        import ctypes
        nk_c = ctypes.c_int(0)
        sel = torch.empty(max(n, 1), dtype=torch.int32, device=dev)
        if n > 0:
            L.check(lib.sdb_nms2d_survivors(L.ptr(cand['dist']), L.ptr(cand['points_f32']), n, R, float(np.float32(nms_thresh)),
                                           int(use_bbox), int(use_kdtree), int(verbose), L.ptr(None), L.ptr(sel), ctypes.byref(nk_c),
                                           L.stream_ptr()))
        self._mark('nms_end')
        nk = int(nk_c.value)
        sel = sel[:nk]
        disti_d = cand['dist'].index_select(0, sel)
        probi_d = cand['prob'].index_select(0, sel)
        pts_d = cand['points_f32'].index_select(0, sel).to(torch.float64)   # integer pixel centres, exact
        if scale is not None:
            if not (isinstance(scale, dict) and 'X' in scale and 'Y' in scale):
                raise ValueError("scale must be a dictionary with entries for 'X' and 'Y'")
            rescale = (1 / scale['Y'], 1 / scale['X'])
            pts_d = pts_d * torch.tensor(rescale, dtype=torch.float64, device=dev).reshape(1, 2)
        else:
            rescale = (1, 1)
        coord_d = dist_to_coord_device(disti_d, pts_d, rescale)
        labels = None
        if return_labels:
            # paint in ascending stable prob order, id = index + 1 (geom2d.py:191-197); survivors are listed by
            # descending score, so the order is computed on the device (sdb_paint_order_2d)
            rank_d = torch.empty(max(nk, 1), dtype=torch.int32, device=dev)
            ids_d = torch.empty(max(nk, 1), dtype=torch.int32, device=dev)
            L.check(lib.sdb_paint_order_2d(L.ptr(probi_d), nk, L.ptr(rank_d), L.ptr(ids_d), L.stream_ptr()))
            lab_d = torch.empty(tuple(int(s) for s in img_shape), dtype=torch.int32, device=dev)
            L.check(lib.sdb_polygons_to_label_2d(L.ptr(coord_d), L.ptr(rank_d), L.ptr(ids_d), nk, R,
                                                int(img_shape[0]), int(img_shape[1]), L.ptr(lab_d), L.stream_ptr()))
            self._mark('label_end')
        else:
            lab_d = None
        pc_d = cand['prob_class'].index_select(0, sel) if 'prob_class' in cand else None
        (labels, probi, coord, points, prob_class), nbytes = self._to_host([None if device_labels else lab_d, probi_d, coord_d, pts_d, pc_d])
        if device_labels:
            labels = lab_d
        if scale is None:
            points = points.astype(np.int64)
        self._stats['d2h_bytes'] = self._stats.get('d2h_bytes', 0) + nbytes
        res_dict = dict(coord=coord, points=points, prob=probi)
        if prob_class is not None:                          # model2d.py:556-560
            res_dict.update(dict(class_prob=prob_class, class_id=np.argmax(prob_class, axis=-1)))
        return labels, res_dict

    def _axes_div_by(self, query_axes):
        self.config.backbone == 'unet' or _raise(NotImplementedError())
        query_axes = axes_check_and_normalize(query_axes)
        assert len(self.config.unet_pool) == len(self.config.grid)
        div_by = dict(zip(
            self.config.axes.replace('C', ''),
            tuple(p ** self.config.unet_n_depth * g for p, g in zip(self.config.unet_pool, self.config.grid))
        ))
        return tuple(div_by.get(a, 1) for a in query_axes)

    def train(self, X, Y, validation_data, classes='auto', augmenter=None, seed=None, epochs=None, steps_per_epoch=None, workers=1):
        """Train the network on the device (reference signature; see models/train.py and DESIGN.md 4.2).  Returns a
        History whose .history holds loss, prob_loss, dist_loss, val_loss, val_prob_loss, val_dist_loss and lr per epoch.
        `workers` is accepted for compatibility (batches are made on the device); `train_tensorboard` is ignored."""
        from .train import train
        return train(self, X, Y, validation_data, classes=classes, augmenter=augmenter, seed=seed, epochs=epochs,
                     steps_per_epoch=steps_per_epoch, workers=workers)

    @property
    def _config_class(self):
        return Config2D
