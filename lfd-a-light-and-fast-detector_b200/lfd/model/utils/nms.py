# -*- coding: utf-8 -*-
"""nms / soft_nms / batched_nms / multiclass_nms with the call signatures of lfd/model/utils/nms.py:7-220, backed by
lfd_nms / lfd_multiclass_nms / lfd_multiclass_soft_nms in liblfd_b200.so (threshold, sort, class-offset suppression or Soft-NMS decay on the
device).  CUDA tensors (or numpy arrays with device_id; soft_nms: on the current CUDA device) only -- there is no CPU NMS in lfd_b200.
nms_cfg type 'soft_nms' runs the reference's Soft-NMS loop over all classes of an image in one array, as its batched_nms does.
nms_match is not provided."""
import ctypes as C

import numpy as np
import torch

from ... import _native as nat

__all__ = ['nms', 'soft_nms', 'batched_nms', 'multiclass_nms']


def _native_nms(dets, iou_thr):
    n = int(dets.shape[0])
    d = dets.detach().float().contiguous()
    keep = torch.empty((max(n, 1),), dtype=torch.int64, device=d.device)
    n_keep = torch.zeros((1,), dtype=torch.int32, device=d.device)
    ws = torch.empty(nat.lib().lfd_nms_workspace_bytes(n), dtype=torch.uint8, device=d.device)
    with torch.cuda.device(d.device):
        nat.check(nat.lib().lfd_nms(nat.ptr(d), n, float(iou_thr), nat.ptr(ws), nat.ptr(keep), nat.ptr(n_keep), nat.stream_ptr()))
    return keep[:int(n_keep.item())]


def nms(dets, iou_thr, device_id=None):
    if isinstance(dets, torch.Tensor):
        is_numpy, dets_th = False, dets
    elif isinstance(dets, np.ndarray):
        is_numpy = True
        if device_id is None:
            raise RuntimeError('lfd_b200 has no CPU NMS: pass device_id or a CUDA tensor')
        dets_th = torch.from_numpy(dets).to('cuda:{}'.format(device_id))
    else:
        raise TypeError('dets must be either a Tensor or numpy array, but got {}'.format(type(dets)))
    if dets_th.shape[0] == 0:
        inds = dets_th.new_zeros(0, dtype=torch.long)
    else:
        if not dets_th.is_cuda:
            raise RuntimeError('lfd_b200 has no CPU NMS: move dets to a CUDA device')
        inds = _native_nms(dets_th, iou_thr)
    if is_numpy:
        inds = inds.cpu().numpy()
    return dets[inds, :], inds


def _device_nms(boxes, box_per_class, scores, score_stride, labels_in, n, num_classes, score_thr, iou_thr, class_agnostic, soft=None):
    """lfd_multiclass_nms (soft None) or lfd_multiclass_soft_nms (soft = (method code, sigma, min_score)): candidates (threshold) + class-offset
    NMS in two launches.  -> (dets [k,5], labels [k] int64, rows [k] int64)."""
    dev = boxes.device
    total = n if labels_in is not None else n * num_classes
    cap = max(int(total), 1)
    L = nat.lib()
    ws = torch.empty(max(L.lfd_multiclass_nms_workspace_bytes(cap), 256), dtype=torch.uint8, device=dev)
    dets = torch.empty((cap, 5), dtype=torch.float32, device=dev)
    labels = torch.empty((cap,), dtype=torch.int32, device=dev)
    src = torch.empty((cap,), dtype=torch.int32, device=dev)
    count = torch.zeros((2,), dtype=torch.int32, device=dev)
    args = (nat.ptr(boxes), int(box_per_class), nat.ptr(scores), int(score_stride), nat.ptr(labels_in), int(n), int(num_classes), float(score_thr),
            float(iou_thr), int(bool(class_agnostic)), cap, nat.ptr(ws), nat.ptr(dets), nat.ptr(labels), nat.ptr(src), nat.ptr(count),
            nat.ptr(count[1:]))
    with torch.cuda.device(dev):
        if soft is None:
            nat.check(L.lfd_multiclass_nms(*args, nat.stream_ptr()))
        else:
            nat.check(L.lfd_multiclass_soft_nms(*args, int(soft[0]), float(soft[1]), float(soft[2]), nat.stream_ptr()))
    k = int(count[0].item())
    return dets[:k], labels[:k].long(), torch.div(src[:k].long(), num_classes, rounding_mode='floor')


def soft_nms(dets, iou_thr, method='linear', sigma=0.5, min_score=1e-3):
    """reference :62-116 (nms_cpu.cpp:76-206) on the device.  dets [n,5] x1,y1,x2,y2,score.  -> (new_dets [k,5], inds [k]): the boxes in
    selection order with their decayed scores, and their input rows.  A tensor input gives tensors in its dtype and on its device (int64
    inds); a numpy array gives numpy arrays (dets in its dtype, int64 inds), computed on the current CUDA device.  Computed in fp32; linear
    mode is bit-exact with the reference's CPU loop.  Empty input gives empty results.

    Example:
        >>> dets = np.array([[4., 3., 5., 3., 0.9],
        >>>                  [4., 3., 5., 4., 0.9],
        >>>                  [3., 1., 3., 1., 0.5],
        >>>                  [3., 1., 3., 1., 0.5],
        >>>                  [3., 1., 3., 1., 0.4],
        >>>                  [3., 1., 3., 1., 0.0]], dtype=np.float32)
        >>> new_dets, inds = soft_nms(dets, 0.6, sigma=0.5)
        >>> assert len(inds) == len(new_dets) == 5
    """
    if isinstance(dets, torch.Tensor):
        if not dets.is_cuda:
            raise RuntimeError('lfd_b200 has no CPU Soft-NMS: move dets to a CUDA device')
        is_tensor, dets_t = True, dets
    elif isinstance(dets, np.ndarray):
        is_tensor, dets_t = False, torch.from_numpy(np.ascontiguousarray(dets))
    else:
        raise TypeError('dets must be either a Tensor or numpy array, but got {}'.format(type(dets)))
    if method not in nat.SOFT_NMS_METHODS:
        raise ValueError('Invalid method for SoftNMS: {}'.format(method))
    device = dets_t.device if is_tensor else torch.device('cuda', torch.cuda.current_device())
    d = dets_t.detach().to(device=device, dtype=torch.float32).reshape(-1, 5)
    n = int(d.shape[0])
    if n == 0:
        new_dets, inds = d.new_zeros((0, 5)), torch.zeros((0,), dtype=torch.int64, device=device)
    else:
        labels_in = torch.zeros((n,), dtype=torch.int32, device=device)
        new_dets, _, inds = _device_nms(d[:, :4].contiguous(), 0, d[:, 4].contiguous(), 1, labels_in, n, 1, 0.0, iou_thr, True,
                                        soft=(nat.SOFT_NMS_METHODS[method], sigma, min_score))
    if is_tensor:
        return new_dets.to(dtype=dets.dtype), inds
    return new_dets.cpu().numpy().astype(dets.dtype), inds.cpu().numpy().astype(np.int64)


_SOFT_KEYS = ('iou_thr', 'method', 'sigma', 'min_score')


def _nms_args(nms_cfg, class_agnostic=False):
    """-> (iou_thr, class_agnostic, soft): soft None for type 'nms'; (method code, sigma, min_score) for type 'soft_nms', whose keys are the
    arguments of soft_nms (an unknown key raises TypeError, as the reference's `soft_nms(dets, **nms_cfg)` call does)."""
    cfg = dict(nms_cfg)
    class_agnostic = cfg.pop('class_agnostic', class_agnostic)
    nms_type = cfg.pop('type', 'nms')
    if nms_type == 'soft_nms':
        for k in cfg:
            if k not in _SOFT_KEYS:
                raise TypeError("soft_nms() got an unexpected keyword argument '%s'" % k)
        if 'iou_thr' not in cfg:
            raise TypeError("soft_nms() missing 1 required positional argument: 'iou_thr'")
        method = cfg.get('method', 'linear')
        if method not in nat.SOFT_NMS_METHODS:
            raise ValueError('Invalid method for SoftNMS: {}'.format(method))
        return float(cfg['iou_thr']), class_agnostic, (nat.SOFT_NMS_METHODS[method], float(cfg.get('sigma', 0.5)), float(cfg.get('min_score', 1e-3)))
    if nms_type != 'nms':
        raise NotImplementedError('nms_cfg type must be "nms" or "soft_nms", got %r' % (nms_type,))
    return float(cfg.get('iou_thr', cfg.get('iou_threshold', 0.5))), class_agnostic, None


def batched_nms(bboxes, scores, inds, nms_cfg, class_agnostic=False):
    """reference :119-158: NMS that never suppresses across different `inds` (class labels).  -> (dets [k,5], keep [k]) with keep indexing the
    inputs, score-descending (type 'soft_nms': in selection order, with the decayed scores).  One native call: the label * (max coordinate + 1)
    offsets live inside the NMS kernel."""
    iou_thr, class_agnostic, soft = _nms_args(nms_cfg, class_agnostic)
    if not bboxes.is_cuda:
        raise RuntimeError('lfd_b200 has no CPU NMS: move the boxes to a CUDA device')
    n = int(bboxes.shape[0])
    if n == 0:
        return torch.cat([bboxes, scores[:, None]], -1), inds.new_zeros(0, dtype=torch.long)
    labels_in = inds.to(torch.int32).contiguous()
    num_classes = int(labels_in.max().item()) + 1
    dets, _, rows = _device_nms(bboxes.detach().float().contiguous(), 0, scores.detach().float().contiguous(), 1, labels_in, n, num_classes,
                                0.0, iou_thr, class_agnostic, soft)
    return dets.to(bboxes.dtype), rows


def multiclass_nms(multi_bboxes, multi_scores, score_thr, nms_cfg, max_num=-1, score_factors=None):
    """reference :161-220: per-class score threshold (strict >) + class-aware NMS or Soft-NMS.  multi_bboxes [n,4] or [n,C*4], multi_scores
    [n,C+1] (background last).  -> (dets [k,5], labels [k]); max_num applies after the (Soft-)NMS."""
    iou_thr, class_agnostic, soft = _nms_args(nms_cfg)
    if not multi_bboxes.is_cuda:
        raise RuntimeError('lfd_b200 has no CPU NMS: move the boxes to a CUDA device')
    n, num_classes = int(multi_scores.shape[0]), int(multi_scores.shape[1]) - 1
    scores = multi_scores.detach().float()
    if score_factors is not None:
        scores = torch.cat([scores[:, :-1] * score_factors[:, None], scores[:, -1:]], 1)
    scores = scores.contiguous()
    if n == 0:
        return multi_bboxes.new_zeros((0, 5)), multi_bboxes.new_zeros((0,), dtype=torch.long)
    dets, labels, _ = _device_nms(multi_bboxes.detach().float().contiguous(), int(multi_bboxes.shape[1] > 4), scores, num_classes + 1, None, n, num_classes,
                                  score_thr, iou_thr, class_agnostic, soft)
    if max_num > 0:
        dets, labels = dets[:max_num], labels[:max_num]
    return dets.to(multi_bboxes.dtype), labels
