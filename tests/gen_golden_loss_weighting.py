# -*- coding: utf-8 -*-
"""Golden vectors for enable_classification_weight / enable_regression_weight, produced by the REFERENCE's own LFD.get_loss
(lfd/model/lfd.py:284-395) + autograd on the CPU (imported from /root/reference, same stubs as tests/gen_golden.py):

    every classification loss (FocalLoss, CrossEntropyLoss, BCEWithLogitsLoss, QualityFocalLoss) x every regression loss (IoULoss,
    GIoULoss, DIoULoss, CIoULoss, SmoothL1Loss, MSELoss) x the four (enable_classification_weight, enable_regression_weight)
    combinations x two batches:
      'mixed'  two images with boxes: 32 positives, 7 gray rows;
      'nopos'  two images without boxes: no positive, weight.sum() == 0.

Each case holds the loss values, or the exception the reference raised (SmoothL1 / MSE with regression weighting on a batch with
positives: the (n, 4) loss times the (n,) weight does not broadcast).  The gradients are stored once per distinct value, to keep the file
small: the gradient w.r.t. the classification output depends only on (classification loss, enable_classification_weight, batch), the one
w.r.t. the regression output only on (regression loss, decode, enable_regression_weight, batch), and is zero outside the positive rows,
of which only the positive rows are kept.  The generator checks both facts on every case before it drops the repeats.

    python tests/gen_golden_loss_weighting.py      ->  tests/golden/loss_weighting.pt   (needs /root/reference; the file is committed)
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [HERE, os.path.dirname(HERE)]
import gen_golden as gg  # noqa: E402
import synth  # noqa: E402
from gen_golden_variants import make_loss  # noqa: E402

CLS = ['FocalLoss', 'CrossEntropyLoss', 'BCEWithLogitsLoss', 'QualityFocalLoss']
REG = ['IoULoss', 'GIoULoss', 'DIoULoss', 'CIoULoss', 'SmoothL1Loss', 'MSELoss']
FLAGS = [(False, False), (True, False), (False, True), (True, True)]
BATCHES = ['mixed', 'nopos']
NUM_CLASSES = 2
RANGES = ((4, 20), (20, 40), (40, 80), (80, 160), (160, 320))     # WIDERFACE-S
STRIDES = (8, 16, 32, 64, 128)
H, W, N = 64, 96, 2


def sizes():
    out = []
    for s in STRIDES:
        out.append(((H + s - 1) // s, (W + s - 1) // s))
    return out


def bbox_mode(ci, ri):
    """The IoU family alternates between the two decodes over the pairs; SmoothL1 / MSE use the 'independent' targets."""
    return 'independent' if REG[ri] in ('SmoothL1Loss', 'MSELoss') else ('sigmoid', 'exp')[(ci + ri) % 2]


def annotations(batch):
    if batch == 'nopos':
        return [(np.zeros((0, 4), np.float32), np.zeros((0,), np.int64)) for _ in range(N)]
    ann = synth.synth_annotations(3, H, W, NUM_CLASSES, seed=13, max_boxes=12)
    return [ann[0], ann[2]]                     # image 1 of synth_annotations is a negative one


def inputs(P):
    """Network outputs shared by the cases: cls [N, P, C] and [N, P, C + 1] (CrossEntropyLoss), reg per decode."""
    g = torch.Generator().manual_seed(4321)
    cls = {c: torch.randn(N, P, c, generator=g) * 1.5 - 1.0 for c in (NUM_CLASSES, NUM_CLASSES + 1)}
    reg = dict(sigmoid=torch.randn(N, P, 4, generator=g), exp=torch.randn(N, P, 4, generator=g) * 0.6 + 2.5,
               independent=torch.randn(N, P, 4, generator=g) * 0.3 + 0.3)
    return cls, reg


def positive_rows(model, ann):
    """Flat (image, point) indices of the positive rows, from the reference's own targets (lfd.py:313-323)."""
    pts = model.generate_point_coordinates(model._head_indexes_to_feature_map_sizes)
    cls_t, _ = model.annotation_to_target(pts, [torch.from_numpy(b) for b, _ in ann], [torch.from_numpy(l) for _, l in ann])
    t = cls_t.reshape(-1, NUM_CLASSES)
    return torch.nonzero((t.min(-1)[0] >= 0) & (t.max(-1)[0] >= 0.001))[:, 0]


def main():
    R = gg.import_reference()
    torch.set_num_threads(8)
    sz = sizes()
    P = sum(h * w for h, w in sz)
    cls_in, reg_in = inputs(P)
    out = dict(num_classes=NUM_CLASSES, ranges=RANGES, strides=STRIDES, H=H, W=W, N=N, sizes=sz, range_assign_mode='dist',
               gray_range_factors=(0.9, 1.1), ann={b: annotations(b) for b in BATCHES}, cls_pred=cls_in, reg_pred=reg_in, cases={},
               grad_cls={}, grad_reg={}, pos_rows={})

    def keep(table, k, grad):
        if k in table:
            assert torch.equal(table[k].view(torch.int32), grad.view(torch.int32)), ('gradient depends on the other loss', k)   # bitwise: NaN too
        else:
            table[k] = grad
    for ci, cname in enumerate(CLS):
        for ri, rname in enumerate(REG):
            bbox = bbox_mode(ci, ri)
            cls_loss, reg_loss = make_loss(R, cname), make_loss(R, rname)
            Cp = NUM_CLASSES + 1 if cname == 'CrossEntropyLoss' else NUM_CLASSES
            for cw, rw in FLAGS:
                model = R['LFD'](backbone=None, neck=None, head=None, num_classes=NUM_CLASSES, regression_ranges=RANGES,
                                 gray_range_factors=(0.9, 1.1), range_assign_mode='dist', point_strides=STRIDES,
                                 classification_loss_func=cls_loss, regression_loss_func=reg_loss,
                                 distance_to_bbox_mode='exp' if bbox == 'exp' else 'sigmoid',
                                 enable_classification_weight=cw, enable_regression_weight=rw)
                for i, s in enumerate(sz):
                    model._head_indexes_to_feature_map_sizes[i] = s
                for batch in BATCHES:
                    cls_pred = cls_in[Cp].clone().requires_grad_(True)
                    reg_pred = reg_in[bbox].clone().requires_grad_(True)
                    key = (cname, rname, cw, rw, batch)
                    try:
                        ld = model.get_loss((cls_pred, reg_pred), out['ann'][batch])
                        ld['loss'].backward()
                    except Exception as e:       # recorded: the reference's own failure is the contract
                        out['cases'][key] = dict(bbox=bbox, error='%s: %s' % (type(e).__name__, e))
                        print('%-18s %-13s cw=%d rw=%d %-6s raises %s' % (cname, rname, cw, rw, batch, out['cases'][key]['error']))
                        continue
                    out['cases'][key] = dict(bbox=bbox, loss_values={k: float(v) for k, v in ld['loss_values'].items()})
                    gr = reg_pred.grad.reshape(-1, 4)
                    pos = out['pos_rows'].setdefault(batch, positive_rows(model, out['ann'][batch]))
                    outside = torch.ones(gr.shape[0], dtype=torch.bool)
                    outside[pos] = False
                    assert bool((gr[outside] == 0).all()), ('regression gradient outside the positives', key)
                    keep(out['grad_cls'], (cname, cw, batch), cls_pred.grad.clone())
                    keep(out['grad_reg'], (rname, bbox, rw, batch), gr[pos].clone())
                    print('%-18s %-13s cw=%d rw=%d %-6s %s' % (cname, rname, cw, rw, batch, out['cases'][key]['loss_values']))
    torch.save(out, os.path.join(HERE, 'golden', 'loss_weighting.pt'))


if __name__ == '__main__':
    main()
