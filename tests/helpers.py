# -*- coding: utf-8 -*-
import functools
import os

import numpy as np
import torch

import synth
import tl_s
from lfd import _native as nat
from oracle import lfd_oracle as orc

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def load_golden(name):
    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


def build_model(cfg_name):
    """The product's drop-in classes, constructed exactly like the reference config scripts do."""
    from lfd.model.backbone import LFDResNet
    from lfd.model.neck import SimpleNeck
    from lfd.model.head import LFDHead
    from lfd.model.losses import FocalLoss, IoULoss, CrossEntropyLoss
    from lfd.model import LFD
    cfg = orc.CONFIGS[cfg_name]
    bb, hd, lc = cfg['backbone'], cfg['head'], cfg['lfd']
    cls_loss = FocalLoss(use_sigmoid=True, gamma=2.0, alpha=0.25, reduction='mean', loss_weight=1.0) \
        if hd['classification_loss_type'] == 'FocalLoss' else CrossEntropyLoss(reduction='mean', loss_weight=1.0)
    reg_loss = IoULoss(eps=1e-6, reduction='mean', loss_weight=1.0)
    backbone = LFDResNet(block_mode=bb['block_mode'], stem_mode=bb['stem_mode'], body_mode=None, input_channels=3,
                         stem_channels=bb['stem_channels'], body_architecture=bb['body_architecture'],
                         body_channels=bb['body_channels'], out_indices=bb['out_indices'], frozen_stages=-1,
                         activation_cfg=dict(type='ReLU', inplace=True), norm_cfg=dict(type='BatchNorm2d'),
                         init_with_weight_file=None, norm_eval=False)
    neck = SimpleNeck(num_neck_channels=128, num_input_channels_list=backbone.num_output_channels_list,
                      num_input_strides_list=backbone.num_output_strides_list, norm_cfg=dict(type='BatchNorm2d'),
                      activation_cfg=dict(type='ReLU', inplace=True))
    head = LFDHead(num_classes=hd['num_classes'], num_heads=len(neck.num_output_strides_list), num_input_channels=128,
                   num_head_channels=128, num_conv_layers=2, activation_cfg=dict(type='ReLU', inplace=True),
                   norm_cfg=dict(type='GroupNorm', num_groups=16) if hd.get('norm', True) else None,
                   conv_kernel_size=hd.get('conv_kernel_size', 1), share_head_flag=hd['share_head_flag'],
                   merge_path_flag=hd['merge_path_flag'], classification_loss_type=type(cls_loss).__name__,
                   regression_loss_type=type(reg_loss).__name__)
    return LFD(backbone=backbone, neck=neck, head=head, num_classes=lc['num_classes'], regression_ranges=lc['regression_ranges'],
               gray_range_factors=lc['gray_range_factors'], range_assign_mode=lc['range_assign_mode'],
               point_strides=neck.num_output_strides_list, classification_loss_func=cls_loss, regression_loss_func=reg_loss,
               distance_to_bbox_mode=lc['distance_to_bbox_mode'])


def synth_model(cfg_name, cls_bias=-1.0, seed=666):
    model = build_model(cfg_name)
    sd = synth.synth_state_dict(model.state_dict(), seed=seed, cls_bias=cls_bias)
    model.load_state_dict(sd, strict=True)
    model.eval()
    return model, sd


def rel_err(a, b):
    """(max-abs error / max-abs reference, rms error / rms reference)"""
    a, b = a.double(), b.double()
    d = (a - b).abs()
    return float(d.max() / b.abs().max().clamp(min=1e-30)), float(torch.sqrt((d ** 2).mean()) / torch.sqrt((b ** 2).mean()).clamp(min=1e-30))


def rows_to_array(rows):
    return np.asarray(rows, np.float64).reshape(-1, 6)


def assert_same_detections(got_src, want_src, want_scores, what, score_tol=2e-3):
    """Kept (point, class) indices of the CUDA pipeline vs the oracle pipeline, end to end: the kept SET must be identical;
    the order (score descending) must be identical except for swaps between detections whose ORACLE scores differ by less
    than `score_tol` -- two pipelines that agree to 1e-3 on the logits cannot agree on the order of two scores closer than that."""
    got_src, want_src = list(got_src), list(want_src)
    assert sorted(got_src) == sorted(want_src), (what, len(got_src), len(want_src), sorted(set(got_src) ^ set(want_src))[:10])
    score = dict(zip(want_src, [float(v) for v in want_scores]))
    for a, b in zip(got_src[:-1], got_src[1:]):
        assert score[a] >= score[b] - score_tol, (what, 'order', a, b, score[a], score[b])


def _iou_one_to_many(b, bs):
    x1, y1 = np.maximum(b[0], bs[:, 0]), np.maximum(b[1], bs[:, 1])
    x2, y2 = np.minimum(b[2], bs[:, 2]), np.minimum(b[3], bs[:, 3])
    inter = np.clip(x2 - x1, 0, None) * np.clip(y2 - y1, 0, None)
    a = (b[2] - b[0]) * (b[3] - b[1])
    aa = (bs[:, 2] - bs[:, 0]) * (bs[:, 3] - bs[:, 1])
    return inter / np.maximum(a + aa - inter, 1e-12)


def assert_same_detections_up_to_margins(got_src, want_src, scores, boxes, thr, iou_thr, what, num_classes=1, score_tol=3e-3, iou_tol=2e-2,
                                         max_frac=5e-2):
    """End-to-end kept sets of two pipelines whose logits agree to ~1e-3 (CUDA forward + CUDA post-process vs oracle forward +
    oracle post-process): the sets must be identical except for provably borderline decisions.  Every index in the symmetric
    difference must (a) have an oracle score within `score_tol` of the score threshold, or (b) have an IoU within `iou_tol` of
    the NMS threshold against some kept box of its class, or (c) overlap (IoU > iou_thr - iou_tol) another differing index of its
    class (a borderline flip cascading through the greedy sweep); and there may be at most max(4, max_frac * kept) of them.
    (The CUDA post-process on the CUDA outputs is separately required to be EXACTLY the oracle post-process on those outputs.)
    scores: the ORACLE's scores flattened [P*C]; boxes: its decoded boxes [P, 4]; indices are point * C + class."""
    got, want = set(got_src), set(want_src)
    diff = sorted(got ^ want)
    assert len(diff) <= max(4, int(max_frac * len(want))), (what, 'too many differing detections', len(diff), len(want))
    if not diff:
        return 0
    C = int(num_classes)
    boxes, scores = np.asarray(boxes), np.asarray(scores).reshape(-1)
    union = np.asarray(sorted(got | want))
    dset = set(diff)
    for d in diff:
        if abs(float(scores[d]) - thr) < score_tol:
            continue
        same = union[(union % C) == (d % C)]
        ious = _iou_one_to_many(boxes[d // C], boxes[same // C])
        near = np.abs(ious - iou_thr) < iou_tol
        cascade = [int(u) for u, v in zip(same, ious) if int(u) in dset and int(u) != d and v > iou_thr - iou_tol]
        assert bool(near.any()) or cascade, (what, 'detection differs without a borderline decision', d, float(scores[d]))
    return len(diff)


@functools.lru_cache(maxsize=None)
def model_of(name, device='cpu'):
    """The synthetic model of a config, TL_S included, in eval mode on `device` (one instance per name and device)."""
    model = tl_s.synth_model()[0] if name == 'TL_S' else synth_model(name)[0]
    return model.to(device).eval()


def finetune_model(cfg, frozen_stages, cls_bias, seed=666):
    """A synthetic model in training mode with its first `frozen_stages` stages frozen ('all': every stage)."""
    model, _ = synth_model(cfg, cls_bias=cls_bias, seed=seed)
    bb = model._backbone
    bb._frozen_stages = len(bb.stages()) if frozen_stages == 'all' else frozen_stages
    return model.train()                  # LFDResNet.train freezes the stem and stages 0..k-1 (eval mode, requires_grad False)


class ListDataset(object):
    """A dataset of the given samples, indexed 0..n-1."""

    def __init__(self, samples):
        self.samples = dict(enumerate(samples))

    def __len__(self):
        return len(self.samples)

    def __getitem__(self, i):
        return self.samples[i]

    def get_indexes(self):
        return list(self.samples.keys())


def bits(t):
    """The bits of a 16- or 32-bit tensor, as integers of the same width (on its device)."""
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32)


def same_bits(a, b, what):
    bad = bits(a) != bits(b)
    if bool(bad.any()):
        i = tuple(bad.nonzero()[0].tolist())
        raise AssertionError('%s: %d of %d elements differ, first at %s: %r vs %r' % (what, int(bad.sum()), bad.numel(), i, float(a[i]), float(b[i])))


def misaligned(x):
    """A device copy of uint8 x at a base address of 1 (mod 4)."""
    raw = torch.empty(x.numel() + 1, dtype=torch.uint8, device='cuda')
    y = raw[1:].view(x.shape)                        # base address 1 (mod 4): the fused stem's per-pixel loader
    y.copy_(x)
    assert y.data_ptr() % 4 == 1
    return y


def grids_agree(results, what):
    """Results of one op on several grids: entries 0 and 1 (fp32 gradients) bit for bit, every later entry (fp64 sums) to 1e-12."""
    g0 = results[0]
    for r in results[1:]:
        for a, b in zip(g0[:2], r[:2]):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32)), what + ': gradients differ between grids'
        for a, b in zip(g0[2:], r[2:]):   # fp64 sums in another order: the same to ~1e-15
            assert bool(((a - b).abs() <= 1e-12 * a.abs() + 1e-300).all()), (what, a, b)


# ------------------------------------------------------------------------------------------------ probes of whole inference plans
CONV_KINDS = (nat.OP_STEM0, nat.OP_CONV, nat.OP_STEM4)


def conv_outputs(plan):
    """(tensor name, op) of every output of the plan's conv ops (the shortcut outputs included)."""
    return [(op[k], op) for op in plan._ops if op['kind'] in CONV_KINDS for k in ('out', 'out2') if op.get(k) is not None]


def downstream_of_gn(plan):
    """Names of the tensors that depend on a GroupNorm."""
    tainted = set()
    for op in plan._ops:
        if op['kind'] == nat.OP_GN_APPLY or any(op.get(k) in tainted for k in ('inp', 'res')):
            tainted |= {op[k] for k in ('out', 'out2') if op.get(k) is not None}
    return tainted


def close_downstream_of_gn(what, a, b):
    """Results downstream of a GroupNorm, whose statistics come from fp64 atomics that add in another order on another grid: a flipped
    last bit of one group's mean or rstd moves every value of the group, so the number of differing elements depends on the map size and
    the 16-bit type; the largest difference keeps the bound of test_gpu_schedule_invariance.py.  A value read from outside the frame
    would be NaN (or 255-based) instead."""
    assert bool(torch.isfinite(a).all()), what
    d = (a - b).abs()
    assert float(d.max()) <= 2.0 ** -6 * float(b.abs().max()), (what, float(d.max()), int((d > 0).sum()))


def poison(plan):
    """0xff bytes (NaN in every float type, 255 in a uint8 staging) in the plan's workspace, input staging and outputs."""
    plan.workspace.fill_(0xff)
    if plan._stage is not None:
        plan._stage.fill_(0xff)
    for c, r in plan._outputs:
        c.view(torch.uint8).fill_(0xff)
        r.view(torch.uint8).fill_(0xff)


def untouched(plan, call):
    """call() must raise before anything reaches the device: the workspace, the outputs and the staging keep their bytes.
    -> the message of the error"""
    import pytest
    plan.staging(nat.INPUT_U8_NHWC)
    poison(plan)
    torch.cuda.synchronize()
    with pytest.raises((ValueError, nat.LfdError)) as e:
        call()
    torch.cuda.synchronize()
    assert bool((plan.workspace == 0xff).all()) and bool((plan._stage == 0xff).all())
    for c, r in plan._outputs:
        assert bool((c.view(torch.uint8) == 0xff).all()) and bool((r.view(torch.uint8) == 0xff).all())
    return str(e.value)
