# -*- coding: utf-8 -*-
"""LFD -- drop-in for the reference detector class (lfd/model/lfd.py:15-655) on H100.

Same constructor kwargs, state_dict keys and public methods (`forward`, `get_loss`, `get_results`,
`predict_for_single_image`, `generate_point_coordinates`, `annotation_to_target`, `distance2bbox`,
`head_indexes_to_feature_map_sizes`); all device work is done by liblfd_b200.so:

    forward                   -> lfd_plan_forward      (whole net = one layer plan, CUDA-graph replayed)
    get_results / predict_*   -> lfd_postprocess       (sigmoid|softmax + decode + class-aware NMS on device)
    annotation_to_target      -> lfd_assign_targets    (label assignment on device)
    get_loss                  -> lfd_assign_targets + lfd_detection_loss (loss + gradients w.r.t. the outputs)

There is no CPU path: modules and inputs must live on a CUDA (sm_90) device.
`predict_for_single_image_with_tensorrt` (reference :657-800) is out of scope (TensorRT is not part of the
H100 path) and raises.
"""
import ctypes as C

import numpy
from collections.abc import Mapping

import torch
import torch.nn as nn

from .. import _native as nat
from .._engine import InferencePlan, PostPlan

__all__ = ['LFD']


class _DetectionLossFn(torch.autograd.Function):
    """loss value with precomputed d loss / d (cls, reg) from lfd_detection_loss."""

    @staticmethod
    def forward(ctx, cls, reg, loss, grad_cls, grad_reg):
        ctx.save_for_backward(grad_cls, grad_reg)
        return loss.clone()

    @staticmethod
    def backward(ctx, g):
        grad_cls, grad_reg = ctx.saved_tensors
        return grad_cls * g, grad_reg * g, None, None, None


class LossValues(Mapping):
    """`loss_values` of get_loss: the reference returns python floats (three `.item()` calls = three device synchronisations between the
    loss and `loss.backward()`).  Here the three numbers travel to a pinned host buffer with an asynchronous copy and become floats on first
    access -- the training loop can enqueue the backward pass and the optimizer step before anything waits for the device."""
    _names = ('loss', 'classification_loss', 'regression_loss')

    def __init__(self, device_values):
        self._host = torch.empty(3, dtype=torch.float32).pin_memory() if device_values.is_cuda else None
        self._event = None
        self._vals = None
        if self._host is None:
            self._vals = [float(v) for v in device_values.tolist()]
        else:
            self._host.copy_(device_values, non_blocking=True)
            self._event = torch.cuda.Event()
            self._event.record(torch.cuda.current_stream(device_values.device))

    def _values(self):
        if self._vals is None:
            self._event.synchronize()
            self._vals = [float(v) for v in self._host.tolist()]
        return self._vals

    def __getitem__(self, key):
        return self._values()[self._names.index(key)] if key in self._names else self._missing(key)

    @staticmethod
    def _missing(key):
        raise KeyError(key)

    def __iter__(self):
        return iter(self._names)

    def __len__(self):
        return 3

    def __repr__(self):
        return repr(dict(zip(self._names, self._values())))


class LFD(nn.Module):

    def __init__(self, backbone=None, neck=None, head=None, num_classes=80,
                 regression_ranges=((0, 64), (64, 128), (128, 256), (256, 512), (512, 1024)),
                 gray_range_factors=(0.9, 1.1), range_assign_mode='dist', point_strides=(8, 16, 32, 64, 128),
                 classification_loss_func=None, regression_loss_func=None, distance_to_bbox_mode='exp',
                 enable_classification_weight=False, enable_regression_weight=False,
                 classification_threshold=0.05, nms_threshold=0.4):
        super(LFD, self).__init__()
        assert len(regression_ranges) == len(point_strides)
        assert range_assign_mode in ['longer', 'shorter', 'dist']
        assert distance_to_bbox_mode in ['exp', 'sigmoid']
        self._backbone, self._neck, self._head = backbone, neck, head
        self._num_classes = num_classes
        self._regression_ranges = regression_ranges
        self._range_assign_mode = range_assign_mode
        if range_assign_mode in ['shorter']:
            assert type(regression_loss_func).__name__ in ['IoULoss', 'GIoULoss', 'DIoULoss', 'CIoULoss']
            assert distance_to_bbox_mode == 'exp'
        self._gray_range_factors = (min(gray_range_factors), max(gray_range_factors))
        self._gray_ranges = [(int(lo * self._gray_range_factors[0]), int(up * self._gray_range_factors[1]))
                             for (lo, up) in regression_ranges]
        self._num_heads = len(point_strides)
        self._point_strides = point_strides
        if classification_loss_func is not None:
            assert type(classification_loss_func).__name__ in ['BCEWithLogitsLoss', 'FocalLoss', 'CrossEntropyLoss', 'QualityFocalLoss']
        self._classification_loss_func = classification_loss_func
        self._regression_loss_type = 'union'
        if regression_loss_func is not None:
            assert type(regression_loss_func).__name__ in ['SmoothL1Loss', 'MSELoss', 'IoULoss', 'GIoULoss', 'DIoULoss', 'CIoULoss']
            self._regression_loss_type = 'independent' if type(regression_loss_func).__name__ in ['SmoothL1Loss', 'MSELoss'] else 'union'
        self._regression_loss_func = regression_loss_func
        self._distance_to_bbox_mode = distance_to_bbox_mode
        self._enable_classification_weight = enable_classification_weight
        self._enable_regression_weight = enable_regression_weight
        self._classification_threshold = classification_threshold
        self._nms_cfg = dict(type='nms', iou_thr=nms_threshold)
        self._head_indexes_to_feature_map_sizes = dict()
        # native state (not part of the state_dict)
        self._plans = {}
        self._post_plans = {}
        self._train_plans = {}
        self._plan_fingerprint = None
        self.conv_impl = nat.CONV_UMMA
        self.act_dtype = 'bf16'                # 16-bit storage type of the inference plan: 'bf16' or 'fp16' (lfd/_engine.py)
        self.use_cuda_graph = True
        self.max_detections_per_image = 8192   # candidate / output capacity of the device post-process

    @property
    def head_indexes_to_feature_map_sizes(self):
        return self._head_indexes_to_feature_map_sizes

    # ------------------------------------------------------------------ forward
    def _fingerprint(self):
        return tuple((t.data_ptr(), t._version) for t in list(self.parameters()) + list(self.buffers()))

    def train_plan_for(self, n, h, w, device):
        """The native training plan (forward + backward op lists) for one input shape (built on first use)."""
        from .._train import TrainPlan, flat_parameters
        flat_parameters(self)
        # BatchNorm modules in eval mode (norm_eval, frozen stages) normalise with their running statistics, and frozen parameters
        # (requires_grad False) get no gradient ops and may form a prefix on the inference kernels: both are part of the plan
        key = (n, h, w, str(device), tuple(m.training for m in self.modules() if isinstance(m, nn.BatchNorm2d)),
               tuple(p.requires_grad for p in self.parameters()))
        if key not in self._train_plans:
            self._train_plans[key] = TrainPlan(self, n, h, w, device)
            self._train_plans[key].use_graph = bool(getattr(self, 'use_cuda_graph_training', False))
        return self._train_plans[key]

    def invalidate_plans(self):
        self._plans = {}
        self._plan_fingerprint = None

    def inference_plan(self, n, h, w, device):
        fp = self._fingerprint()
        if fp != self._plan_fingerprint:
            self._plans, self._plan_fingerprint = {}, fp
        key = (n, h, w, str(device), self.conv_impl, self.act_dtype)
        if key not in self._plans:
            self._plans[key] = InferencePlan(self, n, h, w, device, self.conv_impl, act_dtype=self.act_dtype)
        return self._plans[key]

    def forward(self, x):
        """x: float32 [N,3,H,W] (reference contract) or uint8 [N,H,W,3] BGR (normalisation fused), on CUDA.
        -> (classification [N,P,C'], regression [N,P,4]) float32."""
        if not x.is_cuda:
            raise RuntimeError('lfd_b200 has no CPU path: move the model and the input to a CUDA (H100) device')
        if self.training:
            # native training step (lfd/_train.py): forward with BatchNorm batch statistics, every intermediate kept for the backward,
            # which loss.backward() triggers through one autograd node
            if x.dtype not in (torch.float32, torch.uint8):
                raise TypeError('training-mode forward takes the float32 NCHW batch of the reference data pipeline (or uint8 NHWC frames)')
            from .._train import train_forward
            return train_forward(self, x.contiguous())
        if x.dtype == torch.uint8:
            n, h, w = x.shape[0], x.shape[1], x.shape[2]
        else:
            x = x.float()
            n, h, w = x.shape[0], x.shape[2], x.shape[3]
        plan = self.inference_plan(n, h, w, x.device)
        cls, reg = plan.forward(x.contiguous(), use_graph=self.use_cuda_graph)
        for i, hw in enumerate(plan.level_sizes):
            self._head_indexes_to_feature_map_sizes[i] = hw
        return cls.clone(), reg.clone()

    # ------------------------------------------------------------------ geometry helpers
    def generate_point_coordinates(self, feature_map_sizes):
        """reference :84-107 (int64, cell origin, row-major)."""
        assert len(feature_map_sizes) == len(self._point_strides)
        out = []
        for i in range(len(self._point_strides)):
            h, w = feature_map_sizes[i]
            s = self._point_strides[i]
            xs = torch.arange(0, w * s, s)
            ys = torch.arange(0, h * s, s)
            ym, xm = torch.meshgrid(ys, xs, indexing='ij')
            out.append(torch.stack((xm.reshape(-1), ym.reshape(-1)), dim=-1))
        return out

    def distance2bbox(self, points, distance, max_shape=None):
        """reference :261-282."""
        x1 = points[:, 0] - distance[:, 0]
        y1 = points[:, 1] - distance[:, 1]
        x2 = points[:, 0] + distance[:, 2]
        y2 = points[:, 1] + distance[:, 3]
        if max_shape is not None:
            x1 = x1.clamp(min=0, max=max_shape[1])
            y1 = y1.clamp(min=0, max=max_shape[0])
            x2 = x2.clamp(min=0, max=max_shape[1])
            y2 = y2.clamp(min=0, max=max_shape[0])
        return torch.stack([x1, y1, x2, y2], -1)

    def _sizes(self):
        if len(self._head_indexes_to_feature_map_sizes) != self._num_heads:
            raise RuntimeError('feature map sizes unknown: call forward() first (as in the reference, lfd.py:532)')
        return [self._head_indexes_to_feature_map_sizes[i] for i in range(self._num_heads)]

    def _levels(self, sizes):
        lv = nat.Levels()
        lv.num_levels = len(sizes)
        off = 0
        for i, (h, w) in enumerate(sizes):
            lv.off[i], lv.w[i], lv.stride[i] = off, w, self._point_strides[i]
            lv.lo[i], lv.hi[i] = float(self._regression_ranges[i][0]), float(self._regression_ranges[i][1])
            lv.glo[i], lv.ghi[i] = float(self._gray_ranges[i][0]), float(self._gray_ranges[i][1])
            off += h * w
        return lv, off

    def _device(self):
        return next(self.parameters()).device

    # ------------------------------------------------------------------ label assignment / loss
    def _assign(self, sizes, gt_bboxes_list, gt_labels_list, device):
        lv, P = self._levels(sizes)
        N = len(gt_bboxes_list)
        for l in gt_labels_list:           # the reference indexes a [P, C] target with the label and raises on a bad one
            l = numpy.asarray(l).reshape(-1)
            if l.size and (int(l.min()) < 0 or int(l.max()) >= self._num_classes):
                raise IndexError('gt label out of range [0, %d): %s' % (self._num_classes, sorted(set(l.tolist()))[:8]))
        gmax = max([int(b.shape[0]) for b in gt_bboxes_list] + [1])
        # boxes | labels | counts of the batch in ONE pinned staging buffer and one asynchronous copy (three pageable `.to(device)` calls
        # would each block the host until the stream -- i.e. the forward pass -- has drained); a small ring of staging buffers, each
        # guarded by the event of its last copy
        n_words = N * gmax * 4 + N * gmax + N
        ring = self.__dict__.setdefault('_ann_ring', [])
        slot = self.__dict__.get('_ann_slot', 0)
        self.__dict__['_ann_slot'] = (slot + 1) % 4
        while len(ring) < 4:
            ring.append([None, None])
        if ring[slot][0] is None or ring[slot][0].numel() < n_words:
            ring[slot] = [torch.empty(max(n_words, 1024), dtype=torch.int32).pin_memory(), None]
        elif ring[slot][1] is not None:
            ring[slot][1].synchronize()
        host = ring[slot][0][:n_words]
        host.zero_()
        hb = host[:N * gmax * 4].view(torch.float32).view(N, gmax, 4)
        hl = host[N * gmax * 4:N * gmax * 5].view(N, gmax)
        hc = host[N * gmax * 5:]
        for i, (b, l) in enumerate(zip(gt_bboxes_list, gt_labels_list)):
            g = int(b.shape[0])
            hc[i] = g
            if g:
                hb[i, :g] = torch.as_tensor(b, dtype=torch.float32).reshape(g, 4)
                hl[i, :g] = torch.as_tensor(l).reshape(g).to(torch.int32)
        dev = torch.empty(n_words, dtype=torch.int32, device=device)
        dev.copy_(host, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(device))
        ring[slot][1] = ev
        boxes = dev[:N * gmax * 4].view(torch.float32).view(N, gmax, 4)
        labels = dev[N * gmax * 4:N * gmax * 5].view(N, gmax)
        counts = dev[N * gmax * 5:]
        C_ = self._num_classes
        cls_t = torch.empty((N, P, C_), dtype=torch.float32, device=device)
        reg_t = torch.empty((N, P, 4), dtype=torch.float32, device=device)
        label = torch.empty((N, P), dtype=torch.int32, device=device)
        counters = torch.empty((2,), dtype=torch.int32, device=device)
        mode = {'dist': nat.ASSIGN_DIST, 'longer': nat.ASSIGN_LONGER, 'shorter': nat.ASSIGN_SHORTER}[self._range_assign_mode]
        with torch.cuda.device(device):
            nat.check(nat.lib().lfd_assign_targets(C.byref(lv), N, P, C_, gmax, mode, int(self._regression_loss_type == 'independent'),
                                                   nat.ptr(boxes), nat.ptr(labels), nat.ptr(counts), nat.ptr(cls_t), nat.ptr(reg_t),
                                                   nat.ptr(label), nat.ptr(counters), nat.stream_ptr()))
        return cls_t, reg_t, label, counters, lv

    def annotation_to_target(self, all_point_coordinates_list, gt_bboxes_list, gt_labels_list, *args):
        """reference :109-153.  Returns (classification targets [N,P,C], regression targets [N,P,4]) on the model's device.
        Regression targets of non-positive points are zero (unspecified in the reference, never read)."""
        sizes = []
        for i, pc in enumerate(all_point_coordinates_list):
            s = self._point_strides[i]
            w = int(pc[:, 0].max().item()) // s + 1
            sizes.append((pc.shape[0] // w, w))
        cls_t, reg_t, _, _, _ = self._assign(sizes, gt_bboxes_list, gt_labels_list, self._device())
        return cls_t, reg_t

    def get_loss(self, predict_outputs, annotation_batch, *args):
        """reference :284-395: FocalLoss | CrossEntropyLoss | BCEWithLogitsLoss | QualityFocalLoss with IoULoss | GIoULoss | DIoULoss | CIoULoss
        (union targets, sigmoid / exp decode) or SmoothL1Loss | MSELoss (independent targets).
        Returns dict(loss=Tensor (differentiable w.r.t. predict_outputs), loss_values=dict of floats)."""
        cls_pred, reg_pred = predict_outputs
        cname = type(self._classification_loss_func).__name__
        rname = type(self._regression_loss_func).__name__
        cls_codes = dict(FocalLoss=nat.CLS_SIGMOID, CrossEntropyLoss=nat.CLS_SOFTMAX, BCEWithLogitsLoss=nat.CLS_BCE, QualityFocalLoss=nat.CLS_QFL)
        reg_codes = dict(IoULoss=nat.REG_IOU, GIoULoss=nat.REG_GIOU, DIoULoss=nat.REG_DIOU, CIoULoss=nat.REG_CIOU, SmoothL1Loss=nat.REG_SMOOTH_L1,
                         MSELoss=nat.REG_MSE)
        if cname not in cls_codes or rname not in reg_codes:
            raise NotImplementedError('native get_loss: unknown loss pair %s + %s' % (cname, rname))
        if self._enable_classification_weight or self._enable_regression_weight:
            raise NotImplementedError('classification / regression weighting is disabled in every shipped config and not implemented')
        device = cls_pred.device
        if not cls_pred.is_cuda:
            raise RuntimeError('lfd_b200 has no CPU path')
        sizes = self._sizes()
        gt_b = [a[0] for a in annotation_batch]
        gt_l = [a[1] for a in annotation_batch]
        cls_t, reg_t, label, counters, lv = self._assign(sizes, gt_b, gt_l, device)
        # Data-parallel training: the reference normalises by the positives of the WHOLE (gathered) batch
        # (reference :323,340,383 run after the DataParallel gather), so the per-rank counters are summed over the process
        # group before the loss kernels use them; per-rank losses / gradients then ADD up to the global-batch values and the
        # gradient all-reduce must sum, not average (`loss_globally_normalised`, read by OptimizerHook).
        self.loss_globally_normalised = False
        if self._data_parallel():
            torch.distributed.all_reduce(counters, op=torch.distributed.ReduceOp.SUM)
            self.loss_globally_normalised = True
        N, P = cls_pred.shape[0], cls_pred.shape[1]
        cls_c = cls_pred.detach().float().contiguous()
        reg_c = reg_pred.detach().float().contiguous()
        need_grad = cls_pred.requires_grad or reg_pred.requires_grad
        grad_cls = torch.empty_like(cls_c) if need_grad else None
        grad_reg = torch.empty_like(reg_c) if need_grad else None
        sums = torch.empty((2,), dtype=torch.float64, device=device)
        lf, rf = self._classification_loss_func, self._regression_loss_func
        lc = nat.LossCfg()
        lc.N, lc.P, lc.C = N, P, self._num_classes
        lc.cls_mode, lc.reg_loss = cls_codes[cname], reg_codes[rname]
        if self._regression_loss_type == 'independent':
            lc.bbox_mode = nat.BBOX_INDEPENDENT
        else:
            lc.bbox_mode = nat.BBOX_SIGMOID if self._distance_to_bbox_mode == 'sigmoid' else nat.BBOX_EXP
        lc.gamma = float(getattr(lf, 'beta', 2.0)) if cname == 'QualityFocalLoss' else float(getattr(lf, 'gamma', 2.0))
        lc.alpha = float(getattr(lf, 'alpha', 0.25))
        lc.reg_eps = float(getattr(rf, 'eps', 1e-6))
        lc.smooth_l1_beta = float(getattr(rf, 'beta', 1.0))
        lc.cls_weight, lc.reg_weight = float(lf.loss_weight), float(rf.loss_weight)
        with torch.cuda.device(device):
            nat.check(nat.lib().lfd_detection_loss(C.byref(lv), C.byref(lc), nat.ptr(cls_c), nat.ptr(reg_c), nat.ptr(cls_t), nat.ptr(reg_t), nat.ptr(label),
                                                   nat.ptr(counters), nat.ptr(grad_cls), nat.ptr(grad_reg), nat.ptr(sums), nat.stream_ptr()))
        n_pos = counters[0].to(torch.float64)
        cls_loss = (lf.loss_weight * sums[0] / (n_pos + 1.0)).float()
        reg_loss = torch.where(n_pos > 0, rf.loss_weight * sums[1] / torch.clamp(n_pos, min=1.0), torch.zeros_like(sums[1])).float()
        total = cls_loss + reg_loss
        if need_grad:
            loss = _DetectionLossFn.apply(cls_pred, reg_pred, total, grad_cls, grad_reg)
        else:
            loss = total
        vals = torch.stack([total, cls_loss, reg_loss])
        if self.loss_globally_normalised:   # logged values = the GLOBAL batch's losses (per-rank sums over the global positive count add up)
            torch.distributed.all_reduce(vals, op=torch.distributed.ReduceOp.SUM)
        return dict(loss=loss, loss_values=LossValues(vals))      # floats on first access (asynchronous D2H), see LossValues

    def _data_parallel(self):
        return self.training and torch.distributed.is_available() and torch.distributed.is_initialized() \
            and torch.distributed.get_world_size() > 1

    def empty_shard_loss(self):
        """A rank whose shard of the batch is empty: joins the two collectives of get_loss (positive counters, logged loss values)
        with zeros and returns loss=None (OptimizerHook then reduces zero gradients)."""
        device = self._device()
        self.loss_globally_normalised = False
        vals = torch.zeros(3, dtype=torch.float32, device=device)
        if self._data_parallel():
            counters = torch.zeros((2,), dtype=torch.int32, device=device)
            torch.distributed.all_reduce(counters, op=torch.distributed.ReduceOp.SUM)
            self.loss_globally_normalised = True
            torch.distributed.all_reduce(vals, op=torch.distributed.ReduceOp.SUM)
        return dict(loss=None, loss_values=LossValues(vals))

    # ------------------------------------------------------------------ post-process
    def _post_cfg(self, N, sizes, score_thr, iou_thr, class_agnostic):
        cfg = nat.PostCfg()
        cfg.N, cfg.C = N, self._num_classes
        is_ce = type(self._classification_loss_func).__name__ == 'CrossEntropyLoss'
        cfg.cls_channels = self._num_classes + 1 if is_ce else self._num_classes
        cfg.cls_mode = nat.CLS_SOFTMAX if is_ce else nat.CLS_SIGMOID
        if self._regression_loss_type == 'independent':
            cfg.bbox_mode = nat.BBOX_INDEPENDENT
        else:
            cfg.bbox_mode = nat.BBOX_SIGMOID if self._distance_to_bbox_mode == 'sigmoid' else nat.BBOX_EXP
        cfg.class_agnostic = int(bool(class_agnostic))
        cfg.num_levels = len(sizes)
        off = 0
        for i, (h, w) in enumerate(sizes):
            cfg.level_off[i], cfg.level_w[i], cfg.level_stride[i] = off, w, self._point_strides[i]
            cfg.level_hi[i] = float(max(self._regression_ranges[i]))
            off += h * w
        cfg.P = off
        cfg.score_thr, cfg.iou_thr = float(score_thr), float(iou_thr)
        cfg.cap = int(self.max_detections_per_image)
        return cfg

    def post_plan(self, n, sizes, device, class_agnostic=False):
        key = (n, tuple(map(tuple, sizes)), int(self.max_detections_per_image), str(device), bool(class_agnostic),
               type(self._classification_loss_func).__name__, self._distance_to_bbox_mode, self._regression_loss_type)
        if key not in self._post_plans:
            self._post_plans[key] = PostPlan(self._post_cfg(n, sizes, self._classification_threshold, self._nms_cfg['iou_thr'],
                                                            class_agnostic), device)
        return self._post_plans[key]

    def detect(self, predict_outputs, heights, widths, scales, score_thr, iou_thr, class_agnostic=False):
        """Device post-process.  -> (dets [N,cap,5] x1,y1,x2,y2,score ; labels [N,cap] ; src [N,cap] ; count [N] ; overflow [1])
        on the device (buffers owned by the cached post-process plan)."""
        cls, reg = predict_outputs
        if not cls.is_cuda:
            raise RuntimeError('lfd_b200 has no CPU path')
        N = cls.shape[0]
        sizes = self._sizes()
        pp = self.post_plan(N, sizes, cls.device, class_agnostic)
        if pp.cfg.P != cls.shape[1]:
            raise ValueError('prediction has %d points but the recorded feature maps give %d' % (cls.shape[1], pp.cfg.P))
        pp.set_meta(widths, heights, scales)
        dets, labels, src, count = pp.run(cls.detach().float().contiguous(), reg.detach().float().contiguous(), score_thr, iou_thr)
        return dets, labels, src, count[:N], count[N:]

    @staticmethod
    def _rows(dets, labels, count, overflow, cap):
        cnt = torch.cat([count, overflow]).tolist()
        if cnt[-1]:
            raise nat.LfdError('more than %d candidates passed the score threshold in one image; raise '
                               'model.max_detections_per_image' % cap)
        results = []
        for i, k in enumerate(cnt[:-1]):
            if k == 0:
                results.append([])
                continue
            d = dets[i, :k].clone()
            # [x1, y1, x2, y2, score] -> [label, score, x1, y1, w, h] with w = x2 - x1 + 1 (reference :423-426)
            d[:, 2] = d[:, 2] - d[:, 0] + 1
            d[:, 3] = d[:, 3] - d[:, 1] + 1
            rows = torch.cat([labels[i, :k, None].to(d), d[:, [4, 0, 1, 2, 3]]], dim=1).tolist()
            results.append([[int(r[0])] + r[1:] for r in rows])
        return results

    def get_results(self, predict_outputs, *args):
        """reference :397-432.  args[0] = meta_batch (dicts with resized_height / resized_width / resize_scale)."""
        meta_batch = args[0]
        dets, labels, _, count, overflow = self.detect(
            predict_outputs, [m['resized_height'] for m in meta_batch], [m['resized_width'] for m in meta_batch],
            [m['resize_scale'] for m in meta_batch], self._classification_threshold, self._nms_cfg['iou_thr'],
            self._nms_cfg.get('class_agnostic', False))
        return self._rows(dets, labels, count, overflow, self.max_detections_per_image)

    def predict_for_single_image(self, image, aug_pipeline, classification_threshold=None, nms_threshold=None,
                                 class_agnostic=False, cuda_device_index=0):
        """reference :544-655.  `aug_pipeline=None` takes the fused path: the uint8 BGR image goes to the device as is and
        `simple_normalize` ((x/255-0.5)/0.5, augmentation_pipeline.py:31-36) happens inside the stem kernel; a callable
        pipeline is applied on the host exactly like the reference does."""
        assert isinstance(image, str) or isinstance(image, numpy.ndarray)
        if isinstance(image, str):
            import cv2
            image = cv2.imread(image, cv2.IMREAD_UNCHANGED)
            assert image is not None, 'image is None, confirm that the path is valid!'
        device = torch.device('cuda', cuda_device_index)
        if aug_pipeline is None:
            if image.dtype != numpy.uint8 or image.ndim != 3 or image.shape[2] != 3:
                raise ValueError('the fused input path expects a uint8 HxWx3 (BGR) image')
            data = torch.from_numpy(numpy.ascontiguousarray(image))[None].to(device)
            height, width = image.shape[0], image.shape[1]
        else:
            from ..data_pipeline.dataset import Sample
            sample = Sample()
            sample['image'] = image
            sample = aug_pipeline(sample)
            batch = sample['image'][None].transpose([0, 3, 1, 2])
            data = torch.from_numpy(numpy.ascontiguousarray(batch)).to(device)
            height, width = data.size(2), data.size(3)
        self.cuda(cuda_device_index)
        self.eval()
        with torch.no_grad():
            outputs = self.forward(data)
        thr = classification_threshold if classification_threshold is not None else self._classification_threshold
        if nms_threshold:
            self._nms_cfg.update({'iou_thr': nms_threshold})
        if class_agnostic:
            self._nms_cfg.update({'class_agnostic': class_agnostic})
        dets, labels, _, count, overflow = self.detect(outputs, [height], [width], [1.0], thr, self._nms_cfg['iou_thr'],
                                                       self._nms_cfg.get('class_agnostic', False))
        return self._rows(dets, labels, count, overflow, self.max_detections_per_image)[0]

    def predict_for_single_image_with_tensorrt(self, *args, **kwargs):
        raise NotImplementedError('the TensorRT deployment path of the reference is out of scope of lfd_b200')
