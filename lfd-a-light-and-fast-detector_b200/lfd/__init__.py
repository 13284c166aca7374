# -*- coding: utf-8 -*-
"""lfd -- H100-native drop-in for the reference `lfd` package (hot path only).

Same module paths, class names, constructor kwargs and state_dict keys as
YonghaoHe/LFD-A-Light-and-Fast-Detector for: lfd.model.backbone.LFDResNet,
lfd.model.neck.SimpleNeck, lfd.model.head.LFDHead, lfd.model.LFD,
lfd.model.losses.{FocalLoss, IoULoss, CrossEntropyLoss}, lfd.model.utils.{nms,
batched_nms, multiclass_nms}, lfd.execution.Executor.  All device work goes
through the C-ABI library liblfd_b200.so (hand-written sm_90a CUDA); there is no
CPU fallback and no second backend.
"""
__version__ = '0.1.0'
