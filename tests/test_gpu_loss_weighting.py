# -*- coding: utf-8 -*-
"""enable_classification_weight / enable_regression_weight on the GPU (lfd_loss_weight_sum + lfd_detection_loss_weighted, LFD.get_loss):

  * per element against the float64 reference of tests/loss_weighting_ref.py and against the reference's goldens
    (tests/golden/loss_weighting.pt), every loss pair x switch combination x batch, under forced grids (max_ctas 1 and 3);
  * on the 10 736-row batches of tests/test_gpu_loss_post_configs.py, where max_ctas 1 and 3 make the grid-stride loops and the
    multi-block weight sum run several passes;
  * get_loss through the public interface, repeated calls bit for bit, one training step against the ATen checker, and two data-parallel
    ranks against one rank on the full batch.
Output buffers are NaN-filled before each launch, so an element a kernel never writes fails the comparison."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import loss_post_ref as ref
import loss_weighting_ref as wref
import synth
import test_gpu_loss_post_configs as lpc
from aten_train_reference import train_forward as aten_train_forward
from helpers import grids_agree, synth_model
from lfd import _native as nat
from loss_weighting_ref import U, assert_close

pytestmark = pytest.mark.gpu
DEV = 'cuda'
GRIDS = [0, 1, 3]
NAN = float('nan')
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = torch.load(os.path.join(ROOT, 'tests', 'golden', 'loss_weighting.pt'), weights_only=False)
KEYS = sorted(k for k, v in GOLDEN['cases'].items() if 'error' not in v)
# SmoothL1 / MSE with regression weighting: the reference only runs on a batch without positives, and LFD.get_loss refuses the combination
# up front (tests/test_loss_weighting_host.py); everything else runs natively
REFUSED = [k for k in KEYS if k[1] in ('SmoothL1Loss', 'MSELoss') and k[3]]
NATIVE_KEYS = [k for k in KEYS if k not in REFUSED]


def run_weighted(cfg_vals, lv, x, reg, q, rt, lab, cw, rw, max_ctas):
    """weight sum + weighted loss on fresh NaN-filled buffers -> grad_cls, grad_reg, sums [2], weight_sum [1] (CPU)."""
    c = nat.LossCfg()
    for k, v in cfg_vals.items():
        setattr(c, k, v)
    c.max_ctas = max_ctas
    lab = np.asarray(lab, np.int32)
    C_ = cfg_vals['C']
    cnt = np.array([int(((lab >= 0) & (lab < C_)).sum()), int((lab >= 0).sum())], np.int32)
    td = [torch.from_numpy(np.ascontiguousarray(a)).to(DEV) for a in (x, reg, q, rt, lab, cnt)]
    gc = torch.full(x.shape, NAN, device=DEV)
    gr = torch.full(reg.shape, NAN, device=DEV)
    sums = torch.full((2,), NAN, dtype=torch.float64, device=DEV)
    wsum = torch.full((1,), NAN, dtype=torch.float64, device=DEV)
    ws = torch.full((int(nat.lib().lfd_loss_weight_sum_workspace_bytes(C.byref(c))) // 8,), NAN, dtype=torch.float64, device=DEV)
    nat.check(nat.lib().lfd_loss_weight_sum(C.byref(c), nat.ptr(td[2]), nat.ptr(td[4]), nat.ptr(ws), nat.ptr(wsum), nat.stream_ptr()))
    nat.check(nat.lib().lfd_detection_loss_weighted(C.byref(lpc._levels_struct(lv)), C.byref(c), *[nat.ptr(t) for t in td], nat.ptr(gc), nat.ptr(gr),
                                                    nat.ptr(sums), int(cw), int(rw), nat.ptr(wsum), nat.stream_ptr()))
    torch.cuda.synchronize()
    return gc.cpu(), gr.cpu(), sums.cpu(), wsum.cpu()


def _id(k):
    return '%s-%s-cw%d-rw%d-%s' % (k[0], k[1], k[2], k[3], k[4])


# ================================================================================================ the goldens, per element
@pytest.mark.parametrize('key', NATIVE_KEYS, ids=_id)
def test_golden_cases_per_element(key):
    cname, rname, cw, rw, batch = key
    case = GOLDEN['cases'][key]
    Cn = GOLDEN['num_classes']
    Cp = Cn + 1 if cname == 'CrossEntropyLoss' else Cn
    lv = wref.golden_level_table(GOLDEN)
    x = GOLDEN['cls_pred'][Cp].reshape(-1, Cp).numpy()
    raw = GOLDEN['reg_pred'][case['bbox']].reshape(-1, 4).numpy()
    ct, rt, lab, _, _, _ = wref.golden_targets(GOLDEN, batch, int(case['bbox'] == 'independent'))
    gamma, alpha, clw = wref.CLS_PARAMS[cname]
    eps, beta, rlw = wref.REG_PARAMS[rname]
    cfg = dict(N=GOLDEN['N'], P=lv['P'], C=Cn, cls_mode=wref.CLS_CODES[cname], bbox_mode=wref.BBOX_CODES[case['bbox']], reg_loss=wref.REG_CODES[rname],
               gamma=gamma, alpha=alpha, reg_eps=eps, smooth_l1_beta=beta, cls_weight=clw, reg_weight=rlw)
    res = [run_weighted(cfg, lv, x, raw, ct, rt, lab, cw, rw, m) for m in GRIDS]
    grids_agree(res, _id(key))
    gc, gr, sums, wsum = res[0]
    r = wref.golden_case_ref(GOLDEN, key)
    assert abs(float(wsum[0]) - r['weight_sum']) <= 1e-12 * r['weight_sum']
    # the loss values as get_loss forms them (lfd/model/lfd.py)
    n_pos = float(r['n_pos'])
    with np.errstate(divide='ignore', invalid='ignore'):
        cls_loss = np.float64(clw) * np.float64(sums[0]) / np.float64(float(wsum[0]) if cw else n_pos + 1.0)
    reg_loss = (rlw * float(sums[1]) / (float(wsum[0]) if rw else n_pos)) if n_pos else 0.0
    # K = 24 classification / 48 regression as in tests/test_gpu_loss_post_configs.py
    assert_close(gc, r['grad_cls'], r['S_cls'], 24, 'grad_cls')
    assert_close(gr, r['grad_reg'], r['S_reg'], 48, 'grad_reg')
    assert_close(float(cls_loss), r['cls_loss'], r['S_cls_loss'], 24, 'classification_loss')
    assert_close(reg_loss, r['reg_loss'], r['S_reg_loss'], 48, 'regression_loss')
    # against the reference's own fp32 evaluation: both within their bounds of the exact value
    lvg = case['loss_values']
    assert_close(float(cls_loss), lvg['classification_loss'], r['S_cls_loss'], 72, 'classification_loss vs golden')
    assert_close(reg_loss, lvg['regression_loss'], r['S_reg_loss'], 144, 'regression_loss vs golden')
    golden_gc, golden_gr = wref.golden_grads(GOLDEN, key)
    assert_close(gc, golden_gc, r['S_cls'], 72, 'grad_cls vs golden')
    assert_close(gr, golden_gr, r['S_reg'], 144, 'grad_reg vs golden')


@pytest.mark.parametrize('key', NATIVE_KEYS[::5], ids=_id)
def test_get_loss_matches_the_golden(key):
    """The public interface: LFD.get_loss with the switches on the golden's outputs and annotations."""
    from lfd.model import LFD
    from lfd.model import losses as L
    cname, rname, cw, rw, batch = key
    case = GOLDEN['cases'][key]
    gamma, alpha, clw = wref.CLS_PARAMS[cname]
    eps, beta, rlw = wref.REG_PARAMS[rname]
    closs = dict(FocalLoss=lambda: L.FocalLoss(gamma=gamma, alpha=alpha, loss_weight=clw), CrossEntropyLoss=lambda: L.CrossEntropyLoss(loss_weight=clw),
                 BCEWithLogitsLoss=lambda: L.BCEWithLogitsLoss(loss_weight=clw), QualityFocalLoss=lambda: L.QualityFocalLoss(beta=gamma, loss_weight=clw))[cname]()
    rloss = L.SmoothL1Loss(beta=beta, loss_weight=rlw) if rname == 'SmoothL1Loss' else L.MSELoss(loss_weight=rlw) if rname == 'MSELoss' else \
        getattr(L, rname)(eps=eps, loss_weight=rlw)
    m = LFD(num_classes=GOLDEN['num_classes'], regression_ranges=GOLDEN['ranges'], gray_range_factors=GOLDEN['gray_range_factors'],
            range_assign_mode='dist', point_strides=GOLDEN['strides'], classification_loss_func=closs, regression_loss_func=rloss,
            distance_to_bbox_mode='exp' if case['bbox'] == 'exp' else 'sigmoid', enable_classification_weight=cw, enable_regression_weight=rw)
    for i, s in enumerate(GOLDEN['sizes']):
        m._head_indexes_to_feature_map_sizes[i] = s
    Cp = GOLDEN['num_classes'] + 1 if cname == 'CrossEntropyLoss' else GOLDEN['num_classes']
    cls = GOLDEN['cls_pred'][Cp].clone().cuda().requires_grad_(True)
    reg = GOLDEN['reg_pred'][case['bbox']].clone().cuda().requires_grad_(True)
    ld = m.get_loss((cls, reg), GOLDEN['ann'][batch])
    ld['loss'].backward()
    assert set(ld['loss_values']) == {'loss', 'classification_loss', 'regression_loss'}
    r = wref.golden_case_ref(GOLDEN, key)
    lvg = case['loss_values']
    assert_close(ld['loss_values']['classification_loss'], lvg['classification_loss'], r['S_cls_loss'], 72, 'classification_loss')
    assert_close(ld['loss_values']['regression_loss'], lvg['regression_loss'], r['S_reg_loss'], 144, 'regression_loss')
    golden_gc, golden_gr = wref.golden_grads(GOLDEN, key)
    assert_close(cls.grad.cpu().reshape(-1, Cp), golden_gc, r['S_cls'], 72, 'grad_cls')
    assert_close(reg.grad.cpu().reshape(-1, 4), golden_gr, r['S_reg'], 144, 'grad_reg')


@pytest.mark.parametrize('cls_mode,reg_kind,bbox', [(0, 0, 0), (1, 3, 1), (2, 1, 0), (3, 2, 1), (0, 4, 2), (1, 5, 2)])
def test_switches_off_are_lfd_detection_loss_bit_for_bit(cls_mode, reg_kind, bbox):
    """lfd_detection_loss_weighted with both switches 0 (and no weight sum) is lfd_detection_loss, byte for byte."""
    case = (cls_mode, 2, 2.0, 0.25, 'mixed')
    x, lab, q, cnt = lpc.cls_inputs(case)
    rows = x.shape[0]
    rng = np.random.RandomState(5)
    raw = rng.randn(rows, 4).astype(np.float32)
    rt = rng.uniform(1, 30, (rows, 4)).astype(np.float32) if bbox < 2 else rng.uniform(0, 1, (rows, 4)).astype(np.float32)
    cfg = dict(N=lpc.LOSS_N, P=rows // lpc.LOSS_N, C=2, cls_mode=cls_mode, bbox_mode=bbox, reg_loss=reg_kind, gamma=2.0, alpha=0.25, reg_eps=1e-6,
               smooth_l1_beta=0.5, cls_weight=1.7, reg_weight=1.3)
    for m in (0, 3):
        a = lpc.run_loss(cfg, lpc.LOSS_LV, x, raw, q, rt, lab, cnt, m)
        c = nat.LossCfg()
        for k, v in cfg.items():
            setattr(c, k, v)
        c.max_ctas = m
        td = [torch.from_numpy(np.ascontiguousarray(t)).to(DEV) for t in (x, raw, q, rt, lab, cnt)]
        gc, gr = torch.full(x.shape, NAN, device=DEV), torch.full(raw.shape, NAN, device=DEV)
        sums = torch.full((2,), NAN, dtype=torch.float64, device=DEV)
        nat.check(nat.lib().lfd_detection_loss_weighted(C.byref(lpc._levels_struct(lpc.LOSS_LV)), C.byref(c), *[nat.ptr(t) for t in td], nat.ptr(gc),
                                                        nat.ptr(gr), nat.ptr(sums), 0, 0, None, nat.stream_ptr()))
        torch.cuda.synchronize()
        assert torch.equal(a[0].view(torch.int32), gc.cpu().view(torch.int32)) and torch.equal(a[1].view(torch.int32), gr.cpu().view(torch.int32))
        assert bool(((a[2] - sums.cpu()).abs() <= 1e-12 * a[2].abs()).all())     # fp64 block sums: atomics in any order


# ================================================================================================ forced grids on 10 736 rows
@pytest.mark.parametrize('mode', range(4))
def test_classification_weighting_under_forced_grids(mode):
    case = (mode, 2, 1.5, 0.5, 'mixed')
    x, lab, q, cnt = lpc.cls_inputs(case)
    rows = x.shape[0]
    reg = np.zeros((rows, 4), np.float32)
    rt = np.ones((rows, 4), np.float32)
    cfg = dict(N=lpc.LOSS_N, P=rows // lpc.LOSS_N, C=2, cls_mode=mode, bbox_mode=0, reg_loss=0, gamma=1.5, alpha=0.5, reg_eps=1e-6, smooth_l1_beta=1.0,
               cls_weight=1.7, reg_weight=1.0)
    res = [run_weighted(cfg, lpc.LOSS_LV, x, reg, q, rt, lab, 1, 0, m) for m in GRIDS]
    grids_agree(res, 'cls mode %d' % mode)
    # the weight sum is deterministic: the same bits on a repeated call
    assert torch.equal(run_weighted(cfg, lpc.LOSS_LV, x, reg, q, rt, lab, 1, 0, 1)[3], res[1][3])
    gc, _, sums, wsum = res[0]
    pos, w = wref.row_weights(q, lab, 2)
    assert int(pos.sum()) == int(cnt[0]) > 1000
    assert abs(float(wsum[0]) - w.sum()) <= 1e-12 * w.sum()
    l, g, sl, sg = ref.cls_ref(mode, x, lab, 2, 1.5, 0.5, q)
    scale = 1.7 / w.sum()
    assert_close(gc, g * scale, sg * scale, 24, 'grad_cls')
    assert abs(float(sums[0]) - float(l.sum())) <= 24 * U * float(sl.sum())


@pytest.mark.parametrize('kind,bbox', [(k, b) for k in range(4) for b in (0, 1)])
def test_regression_weighting_under_forced_grids(kind, bbox):
    raw, t, lab, cnt, pt = lpc.reg_inputs((kind, bbox, 1e-6, 0.125))
    rows = raw.shape[0]
    rng = np.random.RandomState(kind * 2 + bbox)
    q = np.where(lab == 0, rng.uniform(0.001, 1.0, rows), np.where(lab < 0, -1.0, 0.0)).astype(np.float32)[:, None]
    x = np.zeros((rows, 1), np.float32)
    cfg = dict(N=lpc.LOSS_N, P=lpc.LOSS_LV['P'], C=1, cls_mode=0, bbox_mode=bbox, reg_loss=kind, gamma=2.0, alpha=0.25, reg_eps=1e-6,
               smooth_l1_beta=1.0, cls_weight=1.0, reg_weight=1.3)
    res = [run_weighted(cfg, lpc.LOSS_LV, x, raw, q, t, lab, 0, 1, m) for m in GRIDS]
    grids_agree(res, 'reg kind %d bbox %d' % (kind, bbox))
    _, gr, sums, wsum = res[0]
    pos = np.nonzero(lab == 0)[0]
    w = q[pos, 0].astype(np.float64)
    assert abs(float(wsum[0]) - w.sum()) <= 1e-12 * w.sum()
    px, py, hi = np.tile(pt['px'], lpc.LOSS_N)[pos], np.tile(pt['py'], lpc.LOSS_N)[pos], np.tile(pt['hi'], lpc.LOSS_N)[pos]
    l, g, sl, sg = ref.reg_ref(kind, bbox, raw[pos], t[pos], px, py, hi, 1e-6, 0.125)
    f = torch.from_numpy(1.3 * w / w.sum())[:, None]
    assert_close(gr[pos], g * f, sg * f, 48, 'grad_reg')
    assert bool((gr[torch.from_numpy(lab != 0)] == 0).all())
    wl = torch.from_numpy(w) * l
    assert abs(float(sums[1]) - float(wl.sum())) <= 48 * U * float((torch.from_numpy(w) * sl).sum())


# ================================================================================================ model level
def _weighted_model(cfg='WIDERFACE_XS', cw=True, rw=True):
    m, _ = synth_model(cfg, cls_bias=-2.0)
    m._enable_classification_weight, m._enable_regression_weight = cw, rw
    return m.cuda().train()


@pytest.mark.parametrize('cw,rw', [(True, False), (False, True), (True, True)])
def test_repeated_get_loss_is_bit_identical(cw, rw):
    m = _weighted_model(cw=cw, rw=rw)
    n, h, w = 4, 192, 256
    x = synth.synth_input(n, h, w).cuda()
    ann = synth.synth_annotations(n, h, w, 1, seed=3)
    with torch.no_grad():
        cls, reg = m(x)
    outs = []
    for _ in range(2):
        c, r = cls.clone().requires_grad_(True), reg.clone().requires_grad_(True)
        ld = m.get_loss((c, r), ann)
        ld['loss'].backward()
        outs.append((ld['loss'].detach().clone(), [ld['loss_values'][k] for k in ('loss', 'classification_loss', 'regression_loss')], c.grad, r.grad))
    assert torch.equal(outs[0][0], outs[1][0]) and outs[0][1] == outs[1][1]
    assert torch.equal(outs[0][2].view(torch.int32), outs[1][2].view(torch.int32))
    assert torch.equal(outs[0][3].view(torch.int32), outs[1][3].view(torch.int32))
    assert all(np.isfinite(outs[0][1]))


def test_weighted_training_step_matches_aten():
    """One native training step with both switches on against autograd over the ATen evaluation of the same graph (the criteria of
    test_gpu_train.py::test_native_parameter_gradients_end_to_end): losses, whole-model gradient error as small as the bf16 emulation's,
    and the final head convs tightly.  The unweighted step on the same batch gives a different loss: the switches reach the step."""
    models = [_weighted_model() for _ in range(4)]
    models[3]._enable_classification_weight = models[3]._enable_regression_weight = False
    n, h, w = 4, 192, 256
    x = synth.synth_input(n, h, w).cuda()
    ann = synth.synth_annotations(n, h, w, 1, seed=3)
    lv = []
    for i, m in enumerate(models):
        out = m(x) if i in (0, 3) else aten_train_forward(m, x, emulate_bf16=(i == 2))
        ld = m.get_loss(out, ann)
        if i in (1, 2):
            for p in m.parameters():
                p.grad = None
        ld['loss'].backward()
        lv.append(ld['loss_values']['loss'])
    assert abs(lv[0] - lv[1]) < 2e-2 * abs(lv[1]) and abs(lv[0] - lv[2]) < 2e-2 * abs(lv[2]), lv
    assert abs(lv[0] - lv[3]) > 1e-2 * abs(lv[3]), lv
    sq = [0.0, 0.0, 0.0]
    for (name, p), (_, q), (_, r) in zip(*[m.named_parameters() for m in models[:3]]):
        assert p.grad is not None and torch.isfinite(p.grad).all(), name
        g, t, e = p.grad.double(), q.grad.double(), r.grad.double()
        sq[0] += float(((g - t) ** 2).sum()); sq[1] += float(((e - t) ** 2).sum()); sq[2] += float((t ** 2).sum())
        if 'classification_path' in name and name.endswith('weight'):
            assert float((g - t).norm() / t.norm()) < 5e-2, name
    nat_, emu = (sq[0] / sq[2]) ** 0.5, (sq[1] / sq[2]) ** 0.5
    assert nat_ < 1.5 * emu + 0.05, (nat_, emu)


@pytest.mark.parametrize('backend', ['nccl', 'gloo'])
def test_ddp_two_ranks_match_one_rank_on_the_full_batch_weighted(backend):
    """tests/run_train_ddp_weighting.py: 2 ranks, each on half of the batch, with both switches on: the weight sum and the positive
    count summed over the ranks, per-rank losses and gradients adding up == 1 rank on the whole batch.  gloo runs both ranks on one GPU."""
    if backend == 'nccl' and torch.cuda.device_count() < 2:
        pytest.skip('needs 2 GPUs (NCCL)')
    env = dict(os.environ, MASTER_ADDR='127.0.0.1')
    cmd = [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', '2', '--master-addr', '127.0.0.1',
           '--master-port', '29527' if backend == 'nccl' else '29529', os.path.join(ROOT, 'tests', 'run_train_ddp_weighting.py'), backend]
    r = subprocess.run(cmd, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:]
    assert 'DDP_OK' in r.stdout, r.stdout[-3000:]
