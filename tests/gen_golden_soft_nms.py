# -*- coding: utf-8 -*-
"""Generates tests/golden/soft_nms.pt from the REFERENCE's own Soft-NMS: its soft_nms wrapper over the compiled soft_nms_cpu
(oracle/build_ref.py), its multiclass_nms with nms_cfg type 'soft_nms', and LFD.get_results with a Soft-NMS config on the stored forward
outputs of tests/golden/forward_{WIDERFACE_S,TT100K_L}.pt.  Run where the reference sources exist; the fixture is committed.

    python tests/gen_golden_soft_nms.py
"""
import os

import numpy as np
import torch

import gen_golden as G
from oracle import lfd_oracle as orc

HERE = os.path.dirname(os.path.abspath(__file__))
DOC_DETS = np.array([[4., 3., 5., 3., 0.9], [4., 3., 5., 4., 0.9], [3., 1., 3., 1., 0.5], [3., 1., 3., 1., 0.5], [3., 1., 3., 1., 0.4],
                     [3., 1., 3., 1., 0.0]], dtype=np.float32)   # nms.py:79-88
SEEDED_K = (1, 2, 33, 1000, 5000)
SOFT_CFGS = (dict(iou_thr=0.3, method='linear', sigma=0.5, min_score=1e-3), dict(iou_thr=0.3, method='gaussian', sigma=0.5, min_score=1e-3))
MODEL_CASES = {'WIDERFACE_S': 0.05, 'TT100K_L': 0.04}   # cfg -> classification threshold


def random_dets(n, rng, span=200.0):
    d = np.concatenate([rng.uniform(0, span, (n, 2)), rng.uniform(2, 60, (n, 2)), rng.uniform(0.01, 1, (n, 1))], 1).astype(np.float32)
    d[:, 2:4] += d[:, :2]
    return d


def special_dets(rng):
    """Ties, duplicate boxes, zero-area boxes, every score below min_score."""
    ties = np.tile(np.array([[10, 10, 20, 20, 0.5]], np.float32), (40, 1))
    ties[::3, 4] = 0.7
    ties[5:15, :4] += 3
    zero = random_dets(60, rng, 40.0)
    zero[::4, 2] = zero[::4, 0]
    zero[1::5, 3] = zero[1::5, 1]
    below = random_dets(100, rng, 50.0)
    below[:, 4] = rng.uniform(0, 9e-4, 100).astype(np.float32)
    return dict(ties=ties, zero_area=zero, all_below=below)


def main():
    R = G.import_reference()
    soft = R['nms_mod'].soft_nms
    rng = np.random.RandomState(2024)
    out = dict(doc=dict(dets=DOC_DETS), sets={}, multiclass={}, models={})
    for method in ('linear', 'gaussian'):
        nd, inds = soft(DOC_DETS, 0.6, method=method, sigma=0.5)
        out['doc'][method] = (nd, inds)
    sets = {('seeded', k): random_dets(k, rng) for k in SEEDED_K}
    sets.update({(name, 0): d for name, d in special_dets(rng).items()})
    for key, d in sets.items():
        out['sets'][key] = dict(dets=d, results={c['method']: soft(d, c['iou_thr'], c['method'], c['sigma'], c['min_score']) for c in SOFT_CFGS})
        print('soft_nms %s: %s' % (key, {m: len(r[1]) for m, r in out['sets'][key]['results'].items()}))
    # multiclass_nms, 45 classes, boxes shared by the classes of a row
    n, C = 100, 45
    boxes = torch.from_numpy(random_dets(n, rng)[:, :4])
    scores = torch.from_numpy(rng.uniform(0, 1, (n, C + 1)).astype(np.float32) ** 6)
    out['multiclass'] = dict(boxes=boxes, scores=scores, score_thr=0.05, results={})
    for c in SOFT_CFGS:
        dets, labels = R['nms_mod'].multiclass_nms(boxes, scores, 0.05, dict(type='soft_nms', **c))
        out['multiclass']['results'][c['method']] = (dets, labels)
        print('multiclass_nms %s: %d rows' % (c['method'], len(labels)))
    # LFD.get_results with a Soft-NMS config on the stored forward outputs
    for name, thr in MODEL_CASES.items():
        g = torch.load(os.path.join(HERE, 'golden', 'forward_%s.pt' % name), weights_only=False)
        model = G.build_ref_model(R, orc.CONFIGS[name])
        for i, hw in enumerate(g['sizes']):
            model._head_indexes_to_feature_map_sizes[i] = tuple(hw)
        model._classification_threshold = thr
        res = {}
        for c in SOFT_CFGS:
            model._nms_cfg = dict(type='soft_nms', **c)
            with torch.no_grad():
                r = model.get_results((g['cls'], g['reg']), g['meta'])
            res[c['method']] = [torch.tensor(x, dtype=torch.float32).reshape(-1, 6) for x in r]
            print('get_results %s %s: %s rows' % (name, c['method'], [len(x) for x in r]))
        out['models'][name] = dict(score_thr=thr, results=res)
    out['soft_cfgs'] = SOFT_CFGS
    path = os.path.join(HERE, 'golden', 'soft_nms.pt')
    torch.save(out, path)
    print('%s: %d bytes' % (path, os.path.getsize(path)))


if __name__ == '__main__':
    main()
