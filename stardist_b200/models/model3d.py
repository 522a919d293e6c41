"""StarDist3D on the H100 path.

Mirrors stardist/models/model3d.py: Config3D (:129-311, in config.py), StarDist3D._build_unet
(:360-399 -> UNetDeviceND), _instances_from_prediction (:589-674), _axes_div_by (:677-691).
"""
import ctypes
import numpy as np
import torch

from .. import _lib as L
from ..utils import axes_check_and_normalize, _raise
from ..nms import non_maximum_suppression_3d, non_maximum_suppression_3d_sparse
from ..geometry.geom3d import polyhedron_to_label
from ..rays3d import rays_from_json
from ..matching import relabel_sequential
from .base import StarDistBase
from .config import Config3D
from .unet_device import UNetDeviceND, ResNetDeviceND, UNetDevice3DTC


class StarDist3D(StarDistBase):
    """StarDist3D model (prediction and training)."""

    def __init__(self, config=Config3D(), name=None, basedir='.', **kwargs):
        super().__init__(config, name=name, basedir=basedir, **kwargs)

    def _build(self):
        if self.config.backbone == 'resnet':
            return ResNetDeviceND(self.config, self.weights)
        self.config.backbone == 'unet' or _raise(NotImplementedError(self.config.backbone))
        import os
        if os.environ.get("STARDIST_B200_UNET", "tc") != "simt" and UNetDevice3DTC.supported(self.config):
            return UNetDevice3DTC(self.config, self.weights)      # tensor-core 3x3x3 convolutions
        return UNetDeviceND(self.config, self.weights)

    def _finish_labels(self, labels, overlap_label):
        # map the overlap_label to something positive and back (model3d.py:632-645)
        if overlap_label is not None and overlap_label < 0 and (overlap_label in labels):
            overlap_mask = (labels == overlap_label)
            overlap_label2 = max(set(np.unique(labels)) - {overlap_label}) + 1
            labels[overlap_mask] = overlap_label2
            labels, fwd, bwd = relabel_sequential(labels)
            labels[labels == fwd[overlap_label2]] = overlap_label
        else:
            labels, _, _ = relabel_sequential(labels)
        return labels

    def _instances_from_prediction(self, img_shape, prob, dist, points=None, prob_class=None, prob_thresh=None,
                                   nms_thresh=None, overlap_label=None, return_labels=True, scale=None, **nms_kwargs):
        if prob_thresh is None: prob_thresh = self.thresholds.prob
        if nms_thresh is None: nms_thresh = self.thresholds.nms
        rays = rays_from_json(self.config.rays_json)
        if points is not None and np.issubdtype(np.asarray(points).dtype, np.integer):
            # sparse candidates (model3d.py:601-606): sort on the host like nms.py:313 (stable), then the device-resident
            # path (NMS, label rendering and relabel_sequential without intermediate host copies)
            prob, dist, points = np.asarray(prob), np.asarray(dist), np.asarray(points)
            assert dist.ndim == 2 and prob.ndim == 1 and points.ndim == 2 and dist.shape[-1] == len(rays) \
                and points.shape[-1] == 3 and len(prob) == len(dist) == len(points)
            from ..nms import _argsort_desc
            order = _argsort_desc(prob)
            dev = self.net.device
            up = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a[order], dt)).to(dev)
            cand = dict(n=len(order), prob=up(prob, np.float32), dist=up(dist, np.float32), points_f32=up(points, np.float32))
            if prob_class is not None:
                cand['prob_class'] = up(np.asarray(prob_class), np.float32)
            kw = {k: nms_kwargs[k] for k in ('use_bbox', 'use_kdtree', 'verbose') if k in nms_kwargs}
            return self._instances_from_candidates_device(img_shape, cand, nms_thresh=nms_thresh, scale=scale, return_labels=return_labels,
                                                          overlap_label=overlap_label, **kw)
        if points is not None:
            points, probi, disti, indsi = non_maximum_suppression_3d_sparse(dist, prob, points, rays, nms_thresh=nms_thresh, **nms_kwargs)
            if prob_class is not None:
                prob_class = np.asarray(prob_class)[indsi]
        else:
            points, probi, disti = non_maximum_suppression_3d(dist, prob, rays, grid=self.config.grid,
                                                              prob_thresh=prob_thresh, nms_thresh=nms_thresh, **nms_kwargs)
            if prob_class is not None:                      # model3d.py:612-614
                inds = tuple(p // g for p, g in zip(points.T, self.config.grid))
                prob_class = np.asarray(prob_class)[inds]
        verbose = nms_kwargs.get('verbose', False)
        if scale is not None:
            if not (isinstance(scale, dict) and 'X' in scale and 'Y' in scale and 'Z' in scale):
                raise ValueError("scale must be a dictionary with entries for 'X', 'Y', and 'Z'")
            rescale = (1 / scale['Z'], 1 / scale['Y'], 1 / scale['X'])
            points = points * np.array(rescale).reshape(1, 3)
            rays = rays.copy(scale=rescale)
        if return_labels:
            labels = polyhedron_to_label(disti, points, rays=rays, prob=probi, shape=img_shape, overlap_label=overlap_label, verbose=verbose)
            labels = self._finish_labels(labels, overlap_label)
        else:
            labels = None
        res_dict = dict(dist=disti, points=points, prob=probi, rays=rays, rays_vertices=rays.vertices, rays_faces=rays.faces)
        if prob_class is not None:                          # model3d.py:663-667
            prob_class = np.asarray(prob_class)
            res_dict.update(dict(class_prob=prob_class, class_id=np.argmax(prob_class, axis=-1)))
        return labels, res_dict

    # ------------------------------------------------------------------ device-resident (sparse) path
    def _instances_from_candidates_device(self, img_shape, cand, nms_thresh=None, scale=None, return_labels=True,
                                          overlap_label=None, use_bbox=True, use_kdtree=True, verbose=False, device_labels=False):
        lib = L.require_cuda()
        if nms_thresh is None: nms_thresh = self.thresholds.nms
        rays = rays_from_json(self.config.rays_json)
        n, R = cand['n'], self.config.n_rays
        dev = cand['dist'].device
        verts_d = torch.from_numpy(np.ascontiguousarray(rays.vertices, np.float32)).to(dev)
        faces_d = torch.from_numpy(np.ascontiguousarray(rays.faces, np.int32)).to(dev)
        keep = torch.zeros(n, dtype=torch.uint8, device=dev)
        if n > 0:
            L.check(lib.sdb_nms3d(L.ptr(cand['dist']), L.ptr(cand['points_f32']), L.ptr(verts_d), L.ptr(faces_d), n, R, int(faces_d.shape[0]),
                                 float(np.float32(nms_thresh)), int(use_bbox), int(use_kdtree), int(verbose), L.ptr(keep), L.stream_ptr()))
        self._mark('nms_end')
        sel = torch.nonzero(keep, as_tuple=False).flatten()
        disti_d = cand['dist'].index_select(0, sel).contiguous()
        probi_d = cand['prob'].index_select(0, sel)
        pts_d = cand['points_f32'].index_select(0, sel).contiguous()
        nk = int(sel.numel())
        points = pts_d.cpu().numpy().astype(np.int64)
        if scale is not None:
            if not (isinstance(scale, dict) and 'X' in scale and 'Y' in scale and 'Z' in scale):
                raise ValueError("scale must be a dictionary with entries for 'X', 'Y', and 'Z'")
            rescale = (1 / scale['Z'], 1 / scale['Y'], 1 / scale['X'])
            points = points * np.array(rescale).reshape(1, 3)
            rays = rays.copy(scale=rescale)
            verts_d = torch.from_numpy(np.ascontiguousarray(rays.vertices, np.float32)).to(dev)
            pts_d = torch.from_numpy(np.ascontiguousarray(points, np.float32)).to(dev)
        labels = None
        lab_host = None
        if return_labels:
            if nk == 0:
                labels = np.zeros(tuple(img_shape), np.uint16)      # geom3d.py:128-131
            else:
                # painting order of geom3d.polyhedron_to_label (geom3d.py:176-180): argsort(prob, stable)[::-1] of the survivor
                # list.  The list is already score-descending; only runs of TIED scores come out reversed by that rule
                # (e.g. a saturated sigmoid), and the dense path applies it -- same rule here so sparse == dense.
                probi_h = probi_d.cpu().numpy()
                order = np.argsort(probi_h, kind='stable')[::-1]
                lab_d = torch.empty(tuple(int(s) for s in img_shape), dtype=torch.int32, device=dev)
                if np.array_equal(order, np.arange(nk)):
                    lab_ids = torch.arange(1, nk + 1, dtype=torch.int32, device=dev)
                    dist_paint, pts_paint = disti_d, pts_d
                else:
                    order_d = torch.from_numpy(np.ascontiguousarray(order)).to(dev)
                    lab_ids = (order_d + 1).to(torch.int32)
                    dist_paint, pts_paint = disti_d.index_select(0, order_d).contiguous(), pts_d.index_select(0, order_d).contiguous()
                L.check(lib.sdb_polyhedron_to_label(L.ptr(dist_paint), L.ptr(pts_paint), L.ptr(verts_d), L.ptr(faces_d), nk, R, int(faces_d.shape[0]),
                                                   L.ptr(lab_ids), int(img_shape[0]), int(img_shape[1]), int(img_shape[2]), 0,
                                                   1 if overlap_label is not None else 0, 0 if overlap_label is None else int(overlap_label),
                                                   L.ptr(lab_d), L.stream_ptr()))
                self._mark('label_end')
                if overlap_label is None:
                    # relabel_sequential (model3d.py:645) on the device: ids are 1..nk, polyhedra that painted no voxel drop out
                    fwd = torch.empty(nk + 3, dtype=torch.int32, device=dev)
                    cnt = ctypes.c_int(0)
                    L.check(lib.sdb_relabel_sequential(L.ptr(lab_d), lab_d.numel(), nk, 1, L.ptr(fwd), ctypes.byref(cnt), L.stream_ptr()))
                    lab_host = lab_d
                else:
                    labels = self._finish_labels(lab_d.cpu().numpy(), overlap_label)
        (lab_np, disti, probi), _ = self._to_host([None if device_labels else lab_host, disti_d, probi_d])
        if lab_np is not None:
            labels = lab_np
        if device_labels:
            labels = lab_host if lab_host is not None else (None if labels is None else torch.from_numpy(np.ascontiguousarray(labels, np.int32)).to(dev))
        self._stats['d2h_bytes'] = self._stats.get('d2h_bytes', 0) + disti.nbytes + points.nbytes + probi.nbytes + (0 if (labels is None or device_labels) else labels.nbytes)
        res_dict = dict(dist=disti, points=points, prob=probi, rays=rays, rays_vertices=rays.vertices, rays_faces=rays.faces)
        if 'prob_class' in cand:                            # model3d.py:663-667
            prob_class = cand['prob_class'].index_select(0, sel).cpu().numpy()
            res_dict.update(dict(class_prob=prob_class, class_id=np.argmax(prob_class, axis=-1)))
        return labels, res_dict

    def _axes_div_by(self, query_axes):
        if self.config.backbone == 'resnet':      # model3d.py:686-688
            query_axes = axes_check_and_normalize(query_axes)
            grid_dict = dict(zip(self.config.axes.replace('C', ''), self.config.grid))
            return tuple(grid_dict.get(a, 1) for a in query_axes)
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
        History whose .history holds loss, prob_loss, dist_loss, val_loss, val_prob_loss, val_dist_loss and lr per epoch,
        and prob_class_loss / val_prob_class_loss for multi-class models.
        X, Y and the two of validation_data are lists, tuples or arrays of images, or lazy sequences (len() and
        __getitem__ returning arrays) read batch by batch (models/data.py).  For multi-class models `classes` and the
        optional third entry of validation_data are per-image class ids or label -> class dicts, or 'auto' (n_classes = 1).
        `workers` is accepted for compatibility (batches are made on the device); `train_tensorboard` is ignored."""
        from .train import train
        return train(self, X, Y, validation_data, classes=classes, augmenter=augmenter, seed=seed, epochs=epochs,
                     steps_per_epoch=steps_per_epoch, workers=workers)

    @property
    def _config_class(self):
        return Config3D
