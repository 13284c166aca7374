# -*- coding: utf-8 -*-
"""Generates tests/golden/forward_TL_S.pt by running the REFERENCE's own LFD, built with the arguments of TL_LFD_S.py, on the seeded
synthetic weights and input of tests/synth.py (CPU, fp32).  Run in the build container only; the fixture is committed.  The other
goldens are not touched.

    python tests/gen_golden_tl_s.py

The golden holds what gen_golden.forward_case stores for the other configs -- inputs, cls / reg and the get_results rows -- without
the loss and its gradients, which belong to training.  A QualityFocalLoss head is a sigmoid head at inference, so the thresholds
are those of the focal configs."""
import os
import types

import torch

import gen_golden
import synth
import tl_s


def main():
    R = gen_golden.import_reference()
    # build_ref_model constructs FocalLoss or CrossEntropyLoss from the config; TL_LFD_S.py:80-85 uses QualityFocalLoss
    QFL = R['losses'].QualityFocalLoss
    qfl = lambda **kw: QFL(use_sigmoid=True, beta=2.0, reduction='mean', loss_weight=2.0)  # noqa: E731
    R = dict(R, losses=types.SimpleNamespace(FocalLoss=None, CrossEntropyLoss=qfl, IoULoss=R['losses'].IoULoss))
    torch.set_num_threads(8)
    n, h, w, cls_bias = tl_s.FORWARD_CASE
    cfg = tl_s.TL_S
    model = gen_golden.build_ref_model(R, cfg)
    sd = synth.synth_state_dict(model.state_dict(), seed=666, cls_bias=cls_bias)
    model.load_state_dict(sd, strict=True)
    model.eval()
    x = synth.synth_input(n, h, w)
    with torch.no_grad():
        cls, reg = model(x)
    assert cls.shape[-1] == 1
    sizes = [model.head_indexes_to_feature_map_sizes[i] for i in range(len(model.head_indexes_to_feature_map_sizes))]
    assert sizes == gen_golden.sizes_for(cfg, h, w), (sizes, gen_golden.sizes_for(cfg, h, w))
    meta = [dict(resized_height=h, resized_width=w, resize_scale=1.0) for _ in range(n)]
    meta[-1]['resize_scale'] = 0.75
    results = {}
    for (thr, iou) in ((0.5, 0.3), (0.2, 0.4), (0.05, 0.4)):
        model._classification_threshold = thr
        model._nms_cfg = dict(type='nms', iou_thr=iou)
        with torch.no_grad():
            res = model.get_results((cls, reg), meta)
        results[(thr, iou)] = [torch.tensor(r, dtype=torch.float32).reshape(-1, 6) for r in res]
        print('  TL_S thr=%.3f iou=%.1f: pass=%d kept=%s' % (thr, iou, int((cls.sigmoid() > thr).sum()), [len(r) for r in res]))
    out = os.path.join(gen_golden.HERE, 'golden', 'forward_TL_S.pt')
    torch.save(dict(cfg='TL_S', N=n, H=h, W=w, cls_bias=cls_bias, seed=666, keys=[(k, tuple(v.shape)) for k, v in sd.items()],
                    checksum=synth.state_checksum(sd), sizes=sizes, cls=cls, reg=reg, meta=meta, results=results), out)
    print('forward TL_S: P=%d cls %s -> %s' % (cls.shape[1], tuple(cls.shape), out))


if __name__ == '__main__':
    main()
