# -*- coding: utf-8 -*-
"""Deployment: export a trained model to a self-contained model file that a C or C++ program runs through liblfd_b200.so alone
(include/lfd_b200.h, lfd_engine_*; examples/lfd_detect.c), without Python or torch.  Takes the place of the reference's
lfd/deployment/tensorrt (build_engine.py serialises an engine, inference.py runs it)."""
import torch

from .._engine import InferencePlan, PostPlan, image_channels

__all__ = ['export_model']


def export_model(model, path, N, H, W, act_dtype='bf16', input_pipeline=None, classification_threshold=None, nms_threshold=None,
                 class_agnostic=False, autotune=True, device=None, create_native=True):
    """Writes the model file of `model` for batches of N frames of up to H x W to `path` and returns (plan, post), the InferencePlan and
    PostPlan it holds.

    The plan is the one predict_for_single_image and StreamingDetector build: the model's act_dtype here given explicitly, its BatchNorm
    folded, the stem fusion and the side-branch schedule of InferencePlan, and the input transform of `input_pipeline` (None: the model's
    own set_input_transform setting) lowered through Compose.device_spec() -- a pipeline the kernels cannot run raises ValueError.  A gray
    model (a 1-channel stem conv) exports a gray plan: its file's op 0 has Cin = 1 and reads 1-channel frames (include/lfd_b200.h).
    autotune: time the side-branch CTA bounds on the device first (InferencePlan.autotune; skipped without use_cuda_graph or a device).
    The post-process is the model's: its classification and NMS thresholds unless given here, its nms_cfg type (greedy or 'soft_nms'
    with its method, sigma and min_score), class_agnostic, and max_detections_per_image as the per-image capacity.
    create_native=False plans on the host only (device 'cpu', no autotune): the file is the same."""
    from ..data_pipeline.augmentation import input_transform_of
    transform = input_transform_of(input_pipeline, channels=image_channels(model)) if input_pipeline is not None else model.input_transform
    if device is None:
        device = next(model.parameters()).device if create_native else torch.device('cpu')
    plan = InferencePlan(model, N, H, W, device, model.conv_impl, create_native=create_native, act_dtype=act_dtype, input_transform=transform)
    if autotune and create_native and getattr(model, 'use_cuda_graph', True):
        plan.autotune()
    thr = classification_threshold if classification_threshold is not None else model._classification_threshold
    iou = nms_threshold if nms_threshold else model._nms_cfg['iou_thr']
    agnostic = bool(class_agnostic or model._nms_cfg.get('class_agnostic', False))
    post = PostPlan(model._post_cfg(N, plan.level_sizes, thr, iou, agnostic), device, model._soft_nms_cfg())
    plan.export(path, post)
    return plan, post
