# -*- coding: utf-8 -*-
"""enable_classification_weight / enable_regression_weight on the CPU:

  * the float64 reference of tests/loss_weighting_ref.py against the goldens of the reference's own get_loss
    (tests/golden/loss_weighting.pt), for every loss pair, flag combination and batch;
  * SmoothL1 / MSE with regression weighting: the reference raises on a batch with positives, LFD.get_loss raises ValueError before
    anything runs;
  * the C ABI rejects malformed switches before it touches a pointer or the device."""
import ctypes as C
import math
import os

import pytest
import torch

import loss_weighting_ref as wref
from loss_weighting_ref import assert_close
from lfd import _native as nat

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = torch.load(os.path.join(HERE, 'golden', 'loss_weighting.pt'), weights_only=False)
KEYS = sorted(GOLDEN['cases'])


def _id(k):
    return '%s-%s-cw%d-rw%d-%s' % (k[0], k[1], k[2], k[3], k[4])


def test_goldens_cover_every_pair_flag_and_batch():
    assert len(KEYS) == 4 * 6 * 4 * 2
    assert sorted(GOLDEN['pos_rows']) == ['mixed', 'nopos'] and GOLDEN['pos_rows']['nopos'].numel() == 0
    # the reference's positive rows, under which the regression gradients are stored, are those of the assignment restatement
    _, _, lab, _, _, _ = wref.golden_targets(GOLDEN, 'mixed', 0)
    assert GOLDEN['pos_rows']['mixed'].tolist() == [i for i, t in enumerate(lab) if 0 <= t < GOLDEN['num_classes']]
    for k in KEYS:
        if 'error' not in GOLDEN['cases'][k]:
            gc, gr = wref.golden_grads(GOLDEN, k)
            assert gc.shape[0] == gr.shape[0] == GOLDEN['N'] * sum(h * w for h, w in GOLDEN['sizes'])
    errors = [k for k in KEYS if 'error' in GOLDEN['cases'][k]]
    # the reference fails exactly for SmoothL1 / MSE with regression weighting on the batch with positives
    assert sorted(errors) == sorted(k for k in KEYS if k[1] in ('SmoothL1Loss', 'MSELoss') and k[3] and k[4] == 'mixed')
    for k in errors:
        assert GOLDEN['cases'][k]['error'].startswith('RuntimeError: The size of tensor a (4) must match the size of tensor b (32)'), k


@pytest.mark.parametrize('key', [k for k in KEYS if 'error' not in GOLDEN['cases'][k]], ids=_id)
def test_float64_reference_matches_the_reference_goldens(key):
    g = GOLDEN['cases'][key]
    r = wref.golden_case_ref(GOLDEN, key)
    if key[4] == 'mixed':
        assert r['n_pos'] == 32 and r['weight_sum'] > 0
    else:
        assert r['n_pos'] == 0 and r['weight_sum'] == 0
    # the goldens are the reference's fp32 evaluation: within the bounds the kernels are held to (tests/test_gpu_loss_post_configs.py,
    # K = 24 classification, 48 regression), doubled for the reference's own roundings
    lv = g['loss_values']
    assert_close(lv['classification_loss'], r['cls_loss'], r['S_cls_loss'], 48, 'classification_loss')
    assert_close(lv['regression_loss'], r['reg_loss'], r['S_reg_loss'], 96, 'regression_loss')
    gc, gr = wref.golden_grads(GOLDEN, key)
    assert_close(gc, r['grad_cls'], r['S_cls'], 48, 'grad_cls')
    assert_close(gr, r['grad_reg'], r['S_reg'], 96, 'grad_reg')
    if key[4] == 'nopos' and key[2]:      # weight.sum() == 0: the reference's classification loss is inf, its regression loss 0
        assert math.isinf(lv['classification_loss']) and lv['regression_loss'] == 0.0
        assert bool((gr == 0).all())


def _loss(name, **kw):
    from lfd.model import losses as L
    return getattr(L, name)(**kw)


@pytest.mark.parametrize('reg', ['SmoothL1Loss', 'MSELoss'])
@pytest.mark.parametrize('cls_w', [False, True])
def test_regression_weighting_with_independent_targets_raises_value_error(reg, cls_w):
    from lfd.model import LFD
    m = LFD(num_classes=2, classification_loss_func=_loss('FocalLoss'), regression_loss_func=_loss(reg), distance_to_bbox_mode='sigmoid',
            enable_classification_weight=cls_w, enable_regression_weight=True)
    with pytest.raises(ValueError, match='does not broadcast'):
        m.get_loss((torch.zeros(1, 4, 2), torch.zeros(1, 4, 4)), [])


def test_weighted_entry_points_are_declared():
    for name in ('lfd_loss_weight_sum_workspace_bytes', 'lfd_loss_weight_sum', 'lfd_detection_loss_weighted'):
        assert name in nat.SYMBOLS


def _cfg(reg_loss=nat.REG_IOU, bbox=nat.BBOX_SIGMOID):
    c = nat.LossCfg()
    c.N, c.P, c.C, c.cls_mode, c.bbox_mode, c.reg_loss = 1, 4, 1, nat.CLS_SIGMOID, bbox, reg_loss
    c.smooth_l1_beta, c.cls_weight, c.reg_weight = 1.0, 1.0, 1.0
    return c


@pytest.mark.parametrize('cw,rw,wsum,reg,msg', [
    (2, 0, 1, nat.REG_IOU, 'must be 0 or 1'), (0, -1, 1, nat.REG_IOU, 'must be 0 or 1'),
    (1, 0, 0, nat.REG_IOU, 'needs weight_sum'), (0, 1, 0, nat.REG_IOU, 'needs weight_sum'),
    (0, 1, 1, nat.REG_SMOOTH_L1, 'does not broadcast'), (1, 1, 1, nat.REG_MSE, 'does not broadcast')])
def test_malformed_switches_are_rejected_before_anything_runs(cw, rw, wsum, reg, msg):
    """Bogus pointers: a call that got past validation would fault or fail on the device check, not return LFD_ERR_INVALID."""
    lib = nat.lib()
    lv = nat.Levels()
    lv.num_levels = 1
    c = _cfg(reg, nat.BBOX_INDEPENDENT if reg >= nat.REG_SMOOTH_L1 else nat.BBOX_SIGMOID)
    p = [C.c_void_p(0x1000 * (i + 1)) for i in range(9)]
    rc = lib.lfd_detection_loss_weighted(C.byref(lv), C.byref(c), *p, cw, rw, C.c_void_p(0x9000 if wsum else 0), C.c_void_p(0))
    assert rc == 1 and msg in lib.lfd_last_error().decode()
