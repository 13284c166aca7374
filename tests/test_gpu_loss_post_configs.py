# -*- coding: utf-8 -*-
"""Label assignment, detection losses and post-process (csrc/losses.cu, csrc/postprocess.cu) element by element against the references
of tests/loss_post_ref.py, across their configuration space and under forced small grids (lfd_loss_cfg.max_ctas / lfd_post_cfg.max_ctas
1 and 3) that make the grid-stride loops of cls_loss_kernel, iou_loss_kernel and candidates_flat_kernel run several passes.

  * assignment: bit for bit (every step is one IEEE fp32 operation on both sides);
  * losses: per element |got - ref| <= K * 2^-24 * S with the float64 reference and the magnitude S of the formula (loss_post_ref.R),
    K written next to each assert; loss sums to K * 2^-24 * sum S;
  * post-process: kept (point, class) indices and their order exactly as the oracle's multiclass_nms, on inputs generated with margins
    around every score / IoU decision; explicit-box NMS bit for bit against the float32 oracle.
Every output buffer is filled with NaN before each launch, so an element a kernel never writes fails the comparison."""
import ctypes as C
import zlib

import numpy as np
import pytest
import torch

import loss_post_ref as ref
from helpers import grids_agree
from lfd import _native as nat
from oracle import lfd_oracle as orc

DEV = 'cuda'
GRIDS = [0, 1, 3]
U = 2.0 ** -24
NAN = float('nan')


def _levels_struct(lv):
    s = nat.Levels()
    s.num_levels = lv['num_levels']
    for l in range(lv['num_levels']):
        s.off[l], s.w[l], s.stride[l] = lv['off'][l], lv['w'][l], lv['stride'][l]
        s.lo[l], s.hi[l], s.glo[l], s.ghi[l] = float(lv['lo'][l]), float(lv['hi'][l]), float(lv['glo'][l]), float(lv['ghi'][l])
    return s


# ================================================================================================ level tables
_RANGES = [(4, 20), (20, 40), (40, 80), (80, 160), (160, 320), (320, 640), (640, 1280), (1280, 2560)]
_HW = {1: [(1, 17)], 5: [(13, 17), (7, 9), (4, 5), (2, 3), (1, 207)], 8: [(9, 11), (5, 7), (3, 5), (2, 3), (2, 2), (1, 3), (1, 2), (1, 97)],
       '1b': [(3, 87)]}


def level_specs(key, wide=False):
    """key 1 / '1b' (P = 17 / 261), 5 (P = 517), 8 (P = 261): strides 8 * 2^l, non-power-of-two widths; gray ranges as lfd.py:49-50.
    wide: level 0 takes every size up to 40000 (a very large box on the finest level)."""
    out = []
    for l, (h, w) in enumerate(_HW[key]):
        lo, hi = (4, 40000) if wide and l == 0 else _RANGES[l]
        out.append((h, w, 8 * 2 ** l, lo, hi, int(lo * 0.9), int(hi * 1.1)))
    return out


# ================================================================================================ assignment cases
# (C, assign_mode, independent, level key, per-image gt counts)
ASSIGN_CASES = []
for _i, (_C, _lk) in enumerate([(1, 1), (2, 5), (45, 8), (100, '1b')]):
    for _m in range(3):
        for _ind in (0, 1):
            ASSIGN_CASES.append((_C, _m, _ind, _lk, [(9, 0, 14, 5), (0,), (12, 3), (7, 11, 0, 2)][(_i + _m + _ind) % 4]))


def _assign_id(c):
    return 'C%d_mode%d_ind%d_L%s_G%s' % (c[0], c[1], c[2], c[3], '-'.join(map(str, c[4])))


def assign_inputs(case):
    """-> level table, per-image (boxes [G,4] xywh float32, labels [G]) built on the level grid so that the boundaries occur."""
    C, mode, ind, lk, counts = case
    wide = lk == 1
    lv = ref.level_table(level_specs(lk, wide))
    rng = np.random.RandomState(zlib.crc32(_assign_id(case).encode()))
    pt = ref.point_table(lv)
    imgs = []
    for G in tuple(counts) + ((1,) if wide else ()):     # wide levels: one more image, holding only the very large box
        boxes, labels = [], []
        while len(boxes) < G:
            kind = 4 if G == 1 and wide else len(boxes) % 5
            i = rng.randint(lv['P'])
            l = int(pt['level'][i])
            px, py = int(pt['px'][i]), int(pt['py'][i])
            lo, hi, glo, ghi = (int(lv[k][l]) for k in ('lo', 'hi', 'glo', 'ghi'))
            m = [lo, hi, glo, ghi][rng.randint(4)]
            c = int(rng.randint(C))
            if kind == 0 or kind == 3:      # the measure of this (point, gt) lands exactly on a range end
                if mode == 0:
                    a, b, cc = rng.randint(0, m + 1, 3)
                    bx = (px - m, py - b, m + 1 + a, b + 1 + cc)
                elif mode == 1:
                    w, h = m, int(rng.randint(1, m + 1))
                    w, h = (w, h) if rng.rand() < .5 else (h, w)
                    bx = (px - rng.randint(w), py - rng.randint(h), w, h)
                else:
                    w, h = m, m + int(rng.randint(0, m))
                    w, h = (w, h) if rng.rand() < .5 else (h, w)
                    bx = (px - rng.randint(w), py - rng.randint(h), w, h)
                if kind == 3 and boxes:     # same class as an earlier box: green and gray of one class at shared points
                    c = labels[-1] if rng.rand() < .5 else (labels[-1] + 1) % C
            elif kind == 1:                 # the point on one edge of the box (a zero distance)
                w, h = int(rng.randint(lo, hi + 1)), int(rng.randint(lo, hi + 1))
                e = rng.randint(4)
                x = px if e == 0 else px - w + 1 if e == 2 else px - rng.randint(w)
                y = py if e == 1 else py - h + 1 if e == 3 else py - rng.randint(h)
                bx = (x, y, w, h)
            elif kind == 2:                 # two same-class boxes mirrored about the point: equal scores there
                w, h = int(rng.randint(lo, hi + 1)), int(rng.randint(lo, hi + 1))
                ox, oy = int(rng.randint(0, max(1, w // 3))), int(rng.randint(0, max(1, h // 3)))
                x1, y1 = px - w // 2 - ox, py - h // 2 - oy
                bx = (x1, y1, w, h)
                if len(boxes) + 1 < G:
                    boxes.append(bx)
                    labels.append(c)
                    bx = (2 * px - x1 - w, 2 * py - y1 - h, w, h)
            else:                           # a very large box on the finest level: green score below 0.001 at far points
                bx = (0, 0, 16001, 16001) if wide else (px - 2 * ghi, py - 2 * ghi, 4 * ghi, 4 * ghi)
            boxes.append(bx)
            labels.append(c)
        imgs.append((np.asarray(boxes, np.float32).reshape(-1, 4), np.asarray(labels, np.int64)))
    return lv, imgs


def assign_boundaries(case):
    """Counts of the (point, gt) / point situations the case claims, from the reference's geometry."""
    C, mode, ind, lk, _ = case
    lv, imgs = assign_inputs(case)
    n = dict(lo=0, hi=0, glo=0, ghi=0, edge0=0, edge1=0, edge2=0, edge3=0, tie=0, green_gray_same=0, gray_other=0, low_score=0, empty=0)
    for boxes, labels in imgs:
        if not len(labels):
            n['empty'] += 1
            continue
        g = ref.assign_geometry(lv, mode, boxes)
        pt, hit, ms = g['pt'], g['hit'], g['measure']
        for k in ('lo', 'hi', 'glo', 'ghi'):
            n[k] += int((hit & (ms == pt[k][:, None])).sum())
        for e in range(4):
            n['edge%d' % e] += int((hit & (g['d'][..., e] == 0)).sum())
        sc = np.where(g['green'], g['score'], 0)
        for c in np.unique(labels):
            m = labels == c
            s = sc[:, m]
            top = s.max(-1)
            n['tie'] += int(((s == top[:, None]).sum(-1) > 1)[top > 0].sum())
            n['green_gray_same'] += int((g['green'][:, m].any(-1) & g['gray'][:, m].any(-1)).sum())
            n['gray_other'] += int((g['green'][:, m].any(-1) & g['gray'][:, ~m].any(-1)).sum())
        ct, _, label, _ = ref.assign_ref(lv, C, mode, ind, boxes, labels)
        n['low_score'] += int(((label == C) & (ct.max(-1) > 0)).sum())
    return n


def run_assign(lv, ncls, mode, ind, imgs):
    N = len(imgs)
    gmax = max([len(l) for _, l in imgs] + [1]) + 2                      # padding behind the last gt of every image
    boxes = torch.full((N, gmax, 4), NAN)
    labels = torch.full((N, gmax), 12345, dtype=torch.int32)
    counts = torch.tensor([len(l) for _, l in imgs], dtype=torch.int32)
    for i, (b, l) in enumerate(imgs):
        boxes[i, :len(l)] = torch.from_numpy(b)
        labels[i, :len(l)] = torch.from_numpy(l.astype(np.int32))
    P = lv['P']
    out = [torch.full((N, P, ncls), NAN, device=DEV), torch.full((N, P, 4), NAN, device=DEV), torch.full((N, P), -7, dtype=torch.int32, device=DEV),
           torch.full((2,), -7, dtype=torch.int32, device=DEV)]
    bd, ld, cd = boxes.to(DEV), labels.to(DEV), counts.to(DEV)
    nat.check(nat.lib().lfd_assign_targets(C.byref(_levels_struct(lv)), N, P, ncls, gmax, mode, ind, nat.ptr(bd), nat.ptr(ld), nat.ptr(cd),
                                           *[nat.ptr(t) for t in out], nat.stream_ptr()))
    torch.cuda.synchronize()
    return [t.cpu().numpy() for t in out]


@pytest.mark.gpu
@pytest.mark.parametrize('case', ASSIGN_CASES, ids=_assign_id)
def test_assign_targets_bit_exact(case):
    C, mode, ind, lk, _ = case
    lv, imgs = assign_inputs(case)
    ct, rt, lab, cnt = run_assign(lv, C, mode, ind, imgs)
    npos = nval = 0
    for i, (b, l) in enumerate(imgs):
        wct, wrt, wlab, (p, v) = ref.assign_ref(lv, C, mode, ind, b, l)
        assert np.array_equal(ct[i].view(np.uint32), wct.view(np.uint32)), ('cls_target', i, np.argwhere(ct[i] != wct)[:4])
        assert np.array_equal(rt[i].view(np.uint32), wrt.view(np.uint32)), ('reg_target', i, np.argwhere(rt[i] != wrt)[:4])
        assert np.array_equal(lab[i], wlab), ('label', i, np.argwhere(lab[i] != wlab)[:4])
        npos, nval = npos + p, nval + v
    assert cnt.tolist() == [npos, nval]


# ================================================================================================ detection-loss cases
LOSS_LEVELS = [(23, 29, 8, 4, 20, 3, 22), (13, 17, 16, 20, 40, 18, 44), (7, 9, 32, 40, 80, 36, 88), (4, 5, 64, 80, 160, 72, 176),
               (1, 5, 128, 160, 320, 144, 352)]                           # P = 667 + 221 + 63 + 20 + 5 = 976
LOSS_N = 11                                                               # 10 736 rows
SPECIAL_X = [0.0, 1e-3, -1e-3, 15.0, -15.0, 40.0, -40.0]

# (cls_mode, C, gamma, alpha, batch): batch 'mixed' | 'ignored' (every row label -1) | 'nopos' (labels -1 and C only)
CLS_CASES = [(m, c, g, a, 'mixed') for m in range(4) for c in (1, 2, 45) for g, a in [((0.0, 0.25), (1.5, 0.5), (2.0, 0.25))[(m + c) % 3]]] + \
            [(0, 2, 2.0, 0.25, 'ignored'), (1, 2, 0.0, 0.25, 'nopos'), (3, 45, 2.0, 0.25, 'nopos'), (2, 1, 0.0, 0.5, 'ignored'), (3, 2, 1.5, 0.25, 'mixed')]
# (reg kind, bbox_mode, eps, beta)
REG_CASES = [(k, b, e, 0.125) for k in range(4) for b in (0, 1) for e in ((1e-6, 1e-3) if (k + b) % 2 == 0 else (1e-6,))] + \
            [(4, 2, 1e-6, 0.125), (5, 2, 1e-6, 0.125), (4, 2, 1e-6, 1.0)]


def _cls_id(c):
    return 'mode%d_C%d_g%g_a%g_%s' % c


def _reg_id(c):
    return 'kind%d_bbox%d_eps%g_beta%g' % c


def loss_labels(C, batch, rng, rows):
    if batch == 'ignored':
        return np.full(rows, -1, np.int32)
    lab = rng.choice([-1, C, 0], rows, p=[0.2, 0.5, 0.3]).astype(np.int32)
    if batch == 'nopos':
        return np.where(lab == 0, C, lab).astype(np.int32)
    pos = lab == 0
    lab[pos] = rng.randint(0, C, int(pos.sum()))
    return lab


def cls_inputs(case):
    mode, C_, gamma, alpha, batch = case
    rng = np.random.RandomState(7 + mode * 100 + C_)
    rows = LOSS_N * sum(h * w for h, w, *_ in LOSS_LEVELS)
    Cp = C_ + 1 if mode == 1 else C_
    x = (rng.randn(rows, Cp) * 4).astype(np.float32)
    sel = rng.rand(rows, Cp) < 0.15
    x[sel] = rng.choice(SPECIAL_X, int(sel.sum())).astype(np.float32)
    lab = loss_labels(C_, batch, rng, rows)
    q = np.zeros((rows, C_), np.float32)
    pos = np.nonzero((lab >= 0) & (lab < C_))[0]
    q[pos, lab[pos]] = rng.uniform(0.001, 1.0, pos.size).astype(np.float32)
    other = (rng.rand(rows, C_) < 0.1) & (q == 0)                 # small soft targets of other classes
    q[other] = rng.uniform(0, 0.0009, int(other.sum())).astype(np.float32)
    q[lab < 0, 0] = -1.0
    if mode == 3 and pos.size:                       # QFL: sigmoid(0) == quality exactly (the a == 0 branch), on a few positives
        k = pos[:7]
        x[k, lab[k]] = 0.0
        q[k] = np.where(q[k] > 0.5, 0.4, q[k])
        q[k, lab[k]] = 0.5
    npos = int(pos.size)
    return x, lab, q, np.array([npos, int((lab >= 0).sum())], np.int32)


def run_loss(cfg_vals, lv, x, reg, q, rt, lab, cnt, max_ctas):
    c = nat.LossCfg()
    for k, v in cfg_vals.items():
        setattr(c, k, v)
    c.max_ctas = max_ctas
    td = [torch.from_numpy(np.ascontiguousarray(a)).to(DEV) for a in (x, reg, q, rt, lab, cnt)]
    gc = torch.full(x.shape, NAN, device=DEV)
    gr = torch.full(reg.shape, NAN, device=DEV)
    sums = torch.full((2,), NAN, dtype=torch.float64, device=DEV)
    nat.check(nat.lib().lfd_detection_loss(C.byref(_levels_struct(lv)), C.byref(c), *[nat.ptr(t) for t in td], nat.ptr(gc), nat.ptr(gr), nat.ptr(sums),
                                           nat.stream_ptr()))
    torch.cuda.synchronize()
    return gc.cpu(), gr.cpu(), sums.cpu()


def assert_within(got, want, S, K, what):
    """|got - want| <= K * (2^-24 * S + 2^-126): the second term is fp32 underflow (results below the normal range flush towards 0)."""
    got = torch.as_tensor(got).double()
    err = (got - want).abs()
    tol = K * (U * S + 2.0 ** -126)
    bad = ~(err <= tol)
    if bool(bad.any()):
        i = tuple(torch.nonzero(bad)[0].tolist())
        raise AssertionError('%s: %d / %d elements off; first at %s: got %r want %r (tol %g)' % (what, int(bad.sum()), got.numel(), i, float(got[i]),
                                                                                            float(want[i]), float(tol[i])))


LOSS_LV = ref.level_table(LOSS_LEVELS)


@pytest.mark.gpu
@pytest.mark.parametrize('case', CLS_CASES, ids=_cls_id)
def test_classification_loss_elementwise(case):
    mode, C_, gamma, alpha, batch = case
    x, lab, q, cnt = cls_inputs(case)
    rows = x.shape[0]
    P = rows // LOSS_N
    reg = np.zeros((rows, 4), np.float32)
    rt = np.ones((rows, 4), np.float32)
    cfg = dict(N=LOSS_N, P=P, C=C_, cls_mode=mode, bbox_mode=0, reg_loss=0, gamma=gamma, alpha=alpha, reg_eps=1e-6, smooth_l1_beta=1.0,
               cls_weight=1.7, reg_weight=1.0)
    res = [run_loss(cfg, LOSS_LV, x, reg, q, rt, lab, cnt, m) for m in GRIDS]
    grids_agree(res, _cls_id(case))
    gc, _, sums = res[0]
    l, g, sl, sg = ref.cls_ref(mode, x, lab, C_, gamma, alpha, q)
    scale = 1.7 / (int(cnt[0]) + 1)
    # K = 24: about 12 roundings in the loss / gradient formula (exp, log, pow, products), plus the fp32 scale 1 / (n_pos + 1) * weight
    assert_within(gc, g * scale, sg * scale + 1e-300, 24, 'grad_cls')
    ign = torch.from_numpy(lab < 0)
    assert bool((gc[ign] == 0).all()), 'ignored rows must get zero gradients'
    # sum: per-element error as above, plus fp64 accumulation (negligible)
    assert abs(float(sums[0]) - float(l.sum())) <= 24 * U * float(sl.sum()) + 1e-300, (float(sums[0]), float(l.sum()))


def reg_inputs(case):
    kind, bbox, eps, beta = case
    rng = np.random.RandomState(11 + kind * 10 + bbox)
    pt = ref.point_table(LOSS_LV)
    P = LOSS_LV['P']
    rows = LOSS_N * P
    lab = rng.choice([-1, 1, 0], rows, p=[0.15, 0.25, 0.6]).astype(np.int32)    # C = 1: label 1 is background
    hi = np.tile(pt['hi'], LOSS_N)
    if kind >= 4:
        t = rng.uniform(-0.2, 1.2, (rows, 4)).astype(np.float32)
        raw = (t + rng.randn(rows, 4).astype(np.float32) * 0.3).astype(np.float32)
        k = rng.rand(rows, 4) < 0.1                                           # SmoothL1 at |d| == beta exactly
        t[k] = 0.25
        raw[k] = np.float32(0.25) + np.float32(beta) * rng.choice([-1, 1], int(k.sum())).astype(np.float32)
    else:
        t = (rng.uniform(0.5, 1.0, (rows, 4)) * hi[:, None]).astype(np.float32)
        k = rng.rand(rows, 4) < 0.2                                           # integer target distances
        t[k] = np.floor(t[k])
        if bbox == 0:
            raw = rng.randn(rows, 4).astype(np.float32)
        else:
            raw = (np.log(t) + rng.randn(rows, 4) * 0.4).astype(np.float32)
        # edge ties on each of the four edges: raw = 0 (sigmoid: d = hi / 2; exp: d = 1) with the target distance equal to d,
        # and saturated sigmoid rows (d = hi) against a target of hi
        for e in range(4):
            r = np.arange(e, rows, 23)
            raw[r, e] = 0.0
            t[r, e] = hi[r] / np.float32(2) if bbox == 0 else 1.0
            if bbox == 0:
                r2 = np.arange(e + 5, rows, 31)
                raw[r2, e] = 40.0
                t[r2, e] = hi[r2]
        r = np.arange(3, rows, 37)                                           # disjoint boxes: the target lies right of the point
        t[r, 0], t[r, 2] = -np.float32(50), np.float32(60)
        raw[r, 2] = -3.0
        r = np.arange(9, rows, 41)                                           # IoU below eps: a tiny predicted box
        raw[r] = -20.0 if bbox == 1 else -30.0
    cnt = np.array([int((lab == 0).sum()), int((lab >= 0).sum())], np.int32)
    return raw, t, lab, cnt, pt


@pytest.mark.gpu
@pytest.mark.parametrize('case', REG_CASES, ids=_reg_id)
def test_regression_loss_elementwise(case):
    kind, bbox, eps, beta = case
    raw, t, lab, cnt, pt = reg_inputs(case)
    rows = raw.shape[0]
    x = np.zeros((rows, 1), np.float32)
    cfg = dict(N=LOSS_N, P=LOSS_LV['P'], C=1, cls_mode=0, bbox_mode=bbox, reg_loss=kind, gamma=2.0, alpha=0.25, reg_eps=eps, smooth_l1_beta=beta,
               cls_weight=1.0, reg_weight=1.3)
    res = [run_loss(cfg, LOSS_LV, x, raw, np.zeros((rows, 1), np.float32), t, lab, cnt, m) for m in GRIDS]
    grids_agree(res, _reg_id(case))
    _, gr, sums = res[0]
    pos = np.nonzero(lab == 0)[0]
    px, py = np.tile(pt['px'], LOSS_N)[pos], np.tile(pt['py'], LOSS_N)[pos]
    hi = np.tile(pt['hi'], LOSS_N)[pos]
    l, g, sl, sg = ref.reg_ref(kind, bbox, raw[pos], t[pos], px, py, hi, eps, beta)
    scale = 1.3 / int(cnt[0])
    # K = 48: the IoU-family formulas pass a term through up to ~30 fp32 roundings (GIoU / DIoU / CIoU forward-mode products), plus the
    # decode and the fp32 scale 1 / n_pos * weight
    assert_within(gr[pos], g * scale, sg * scale, 48, 'grad_reg')
    nonpos = torch.from_numpy(lab != 0)
    assert bool((gr[nonpos] == 0).all()), 'non-positive rows must get zero gradients'
    assert abs(float(sums[1]) - float(l.sum())) <= 48 * U * float(sl.sum()), (float(sums[1]), float(l.sum()))


@pytest.mark.gpu
def test_regression_loss_without_positives():
    raw, t, lab, cnt, pt = reg_inputs((0, 1, 1e-6, 0.125))
    lab = np.where(lab == 0, 1, lab).astype(np.int32)
    cnt = np.array([0, int((lab >= 0).sum())], np.int32)
    rows = raw.shape[0]
    cfg = dict(N=LOSS_N, P=LOSS_LV['P'], C=1, cls_mode=0, bbox_mode=1, reg_loss=0, gamma=2.0, alpha=0.25, reg_eps=1e-6, smooth_l1_beta=1.0,
               cls_weight=1.0, reg_weight=1.0)
    for m in GRIDS:
        _, gr, sums = run_loss(cfg, LOSS_LV, np.zeros((rows, 1), np.float32), raw, np.zeros((rows, 1), np.float32), t, lab, cnt, m)
        assert bool((gr == 0).all()) and float(sums[1]) == 0.0


# ================================================================================================ stand-alone entries
@pytest.mark.gpu
@pytest.mark.parametrize('kind', range(4))
def test_box_loss_past_the_block_cap(kind):
    n = 4096 * 256 + 1237                                                 # > 4096 blocks of 256: the grid-stride loop runs twice
    rng = np.random.RandomState(kind)
    tg = np.concatenate([rng.uniform(0, 200, (n, 2)), rng.uniform(1, 90, (n, 2))], 1).astype(np.float32)
    tg[:, 2:] += tg[:, :2]
    pr = (tg + rng.randn(n, 4).astype(np.float32) * 8).astype(np.float32)
    for e in range(4):                                                    # a predicted edge equal to the target edge, on each edge
        pr[e::29, e] = tg[e::29, e]
    pr[7::53, :2] = tg[7::53, 2:] + 5                                     # disjoint
    pr[7::53, 2:] = pr[7::53, :2] + 10
    pr[11::61] = tg[11::61]                                               # identical boxes
    loss = torch.full((n,), NAN, device=DEV)
    grad = torch.full((n, 4), NAN, device=DEV)
    pd, td = torch.from_numpy(pr).to(DEV), torch.from_numpy(tg).to(DEV)
    nat.check(nat.lib().lfd_box_loss(kind, nat.ptr(pd), nat.ptr(td), n, 1e-6, nat.ptr(loss), nat.ptr(grad), nat.stream_ptr()))
    torch.cuda.synchronize()
    l, g, sl, sg = ref.box_loss_ref(kind, pr, tg, 1e-6)
    # K = 48 as for the regression loss of lfd_detection_loss
    assert_within(loss.cpu(), l, sl, 48, 'box loss')
    assert_within(grad.cpu(), g, sg, 48, 'box loss grad')


@pytest.mark.gpu
def test_sigmoid_focal_loss_past_the_block_cap():
    M, C_ = 46703, 45                                                     # 2 101 635 logits > 4096 blocks of 512
    rng = np.random.RandomState(3)
    x = (rng.randn(M, C_) * 5).astype(np.float32)
    x[rng.rand(M, C_) < 0.1] = 40.0
    t = rng.randint(0, C_ + 1, M).astype(np.int64)
    dl = rng.uniform(0.5, 2, (M, C_)).astype(np.float32)
    xd, tdv, dld = torch.from_numpy(x).to(DEV), torch.from_numpy(t).to(DEV), torch.from_numpy(dl).to(DEV)
    out = torch.full((M, C_), NAN, device=DEV)
    dout = torch.full((M, C_), NAN, device=DEV)
    L = nat.lib()
    nat.check(L.lfd_sigmoid_focal_loss_forward(nat.ptr(xd), nat.ptr(tdv), M, C_, 1.5, 0.25, nat.ptr(out), nat.stream_ptr()))
    nat.check(L.lfd_sigmoid_focal_loss_backward(nat.ptr(xd), nat.ptr(tdv), nat.ptr(dld), M, C_, 1.5, 0.25, nat.ptr(dout), nat.stream_ptr()))
    torch.cuda.synchronize()
    l, g, sl, sg = ref.cls_ref(0, x, t, C_, 1.5, 0.25)
    # K = 24 as for the classification loss; the backward's extra product with d_losses is one more rounding
    assert_within(out.cpu(), l, sl + 1e-300, 24, 'focal forward')
    d = torch.from_numpy(dl).double()
    assert_within(dout.cpu(), g * d, sg * d + 1e-300, 25, 'focal backward')


# ================================================================================================ NMS on explicit boxes
def nms_path(K, C, agnostic, mn, seg_lengths=None):
    """The branch nms_kernel takes for K candidates: '4a' (bit matrix), '4c' (per-class sweeps; 'long' if a class has > 512), '4b'
    (lock step); in shared memory or global memory."""
    Kp = 1
    while Kp < K:
        Kp <<= 1
    if Kp <= 1024:
        return '4a'
    in_smem = Kp <= 4096
    seg_off = ((4096 * 29 + 15) & ~15) if in_smem else 0
    seg_cap = (32768 + 1024 * 128 - seg_off) // 4
    if not agnostic and C > 1 and mn >= 0 and K <= seg_cap:
        return '4c' + ('_long' if seg_lengths is not None and max(seg_lengths) > 512 else '') + ('' if in_smem else '_gmem')
    return '4b' + ('' if in_smem else '_gmem')


# (name, K, C, agnostic, special)
NMS_CASES = [('raw', k, 1, 1, None) for k in (1, 31, 32, 33, 1023, 1024, 1025, 4096, 4097)] + [
    ('batched', 3000, 45, 0, None), ('batched', 2000, 3, 0, 'seg512'), ('batched', 1500, 5, 0, 'negative'), ('batched', 41000, 4, 0, None),
    ('batched', 600, 7, 0, 'degenerate'), ('batched', 2500, 1, 1, None), ('batched', 2049, 45, 0, 'singletons'), ('batched', 6000, 30, 0, None),
    ('batched', 1800, 45, 0, 'large')]


def _nms_id(c):
    return '%s_K%d_C%d_agn%d_%s' % c


def nms_inputs(case, rng):
    name, K, C_, agn, sp = case
    if sp == 'degenerate':     # identical boxes, zero-area boxes, integer boxes with IoU exactly 0.5 (not suppressed: strict >)
        b = np.zeros((K, 4), np.float32)
        b[:, :2] = rng.randint(0, 50, (K, 2))
        b[:, 2:] = b[:, :2] + rng.randint(0, 6, (K, 2))
        b[::3, 2] = b[::3, 0]
        b[1::7] = b[0]
        b[2::11] = [0, 0, 2, 2]
        b[3::11] = [0, 0, 4, 1]           # IoU with [0,0,2,2]: 2 / (4 + 4 - 2) = 1/3; with [0,0,4,2] below: 0.5
        b[4::11] = [0, 0, 4, 2]
    elif sp == 'large':        # coordinates near 2^24 / C: the class offsets are not exact in fp32
        xy = rng.uniform(0, 2.0 ** 24 / C_ * 0.9, (K, 2))
        b = np.concatenate([xy, xy + rng.uniform(2000, 30000, (K, 2))], 1).astype(np.float32)
    else:
        span = 900 if K > 1500 else 300
        xy = rng.uniform(0, span, (K, 2))
        b = np.concatenate([xy, xy + rng.uniform(4, 90, (K, 2))], 1).astype(np.float32)
    if sp == 'negative':
        b[5, 0] = -3.0
    s = rng.uniform(0.05, 1.0, K).astype(np.float32)
    s[rng.randint(0, K, K // 20)] = np.float32(0.5)                    # score ties, across classes too
    if sp == 'seg512':
        lab = np.concatenate([np.zeros(512), np.ones(513), np.full(K - 1025, 2)]).astype(np.int64)
    elif sp == 'singletons':
        lab = np.concatenate([np.arange(C_), np.zeros(K - C_)]).astype(np.int64)
    else:
        lab = rng.randint(0, C_, K).astype(np.int64)
    if sp in (None, 'seg512'):     # the lowest-ranked candidate overall, in the last class, is a copy of that class's top box
        last = np.nonzero(lab == lab.max())[0]
        b[last[-1]] = b[last[np.argmax(s[last])]]
        s[last[-1]] = s.min() * np.float32(0.5)
    return b, s, lab


def nms_oracle(b, s, lab, C_, agn, thr):
    """The reference's batched_nms / multiclass_nms on one candidate list (nms.py:141-156): -> keep, rows."""
    if agn:
        bn = b
    else:
        off = lab.astype(np.float32) * (b.max() + np.float32(1))
        bn = (b + off[:, None]).astype(np.float32)
    keep = orc.nms(np.concatenate([bn, s[:, None]], 1), thr)
    rows = bn[keep] if agn else (bn[keep] - off[keep][:, None]).astype(np.float32)
    return keep, rows


@pytest.mark.gpu
@pytest.mark.parametrize('case', NMS_CASES, ids=_nms_id)
def test_nms_explicit_boxes_bit_exact(case):
    from lfd.model.utils import batched_nms, nms
    name, K, C_, agn, sp = case
    rng = np.random.RandomState(K + C_)
    b, s, lab = nms_inputs(case, rng)
    thr = 0.5 if sp == 'degenerate' else 0.45
    if name == 'raw':
        _, inds = nms(torch.from_numpy(np.concatenate([b, s[:, None]], 1)).to(DEV), thr)
        assert inds.cpu().tolist() == orc.nms(np.concatenate([b, s[:, None]], 1), thr).tolist()
        return
    dets, keep = batched_nms(torch.from_numpy(b).to(DEV), torch.from_numpy(s).to(DEV), torch.from_numpy(lab).to(DEV),
                             dict(type='nms', iou_thr=thr, class_agnostic=bool(agn)))
    okeep, orows = nms_oracle(b, s, lab, C_, agn, thr)
    assert keep.cpu().tolist() == okeep.tolist(), (nms_path(K, C_, agn, float(b.min())), len(keep), len(okeep))
    assert np.array_equal(dets[:, :4].cpu().numpy().view(np.uint32), orows.view(np.uint32))
    assert np.array_equal(dets[:, 4].cpu().numpy(), s[okeep])


@pytest.mark.gpu
def test_multiclass_nms_grid_strides():
    """n * C > 524 288 candidates' worth of (row, class) pairs: box_candidates_kernel strides over its 2048 blocks."""
    from lfd.model.utils import multiclass_nms
    rng = np.random.RandomState(4)
    n, C_ = 12000, 45
    boxes = np.concatenate([rng.uniform(0, 900, (n, 2)), rng.uniform(4, 90, (n, 2))], 1).astype(np.float32)
    boxes[:, 2:] += boxes[:, :2]
    scores = rng.uniform(0, 1, (n, C_)).astype(np.float32) ** 8          # about 3 % above 0.65
    padded = np.concatenate([scores, np.zeros((n, 1), np.float32)], 1)
    dets, labels = multiclass_nms(torch.from_numpy(boxes).to(DEV), torch.from_numpy(padded).to(DEV), 0.65, dict(type='nms', iou_thr=0.5))
    odets, olabels, _ = orc.multiclass_nms(boxes, scores, 0.65, 0.5)
    assert labels.tolist() == olabels.tolist()
    assert np.array_equal(dets.cpu().numpy().view(np.uint32), odets.view(np.uint32))


# ================================================================================================ post-process
# (cls_mode, C, bbox_mode, agnostic, N): every candidate kernel, each bbox_mode, per-image size / scale
POST_CASES = [(0, 1, b, 0, 3) for b in range(3)] + [(0, c, b, a, 3) for c in (2, 45) for b, a in ((0, 0), (1, 1), (2, 0))] + \
             [(1, c, b, a, 2) for c, b, a in ((1, 0, 0), (45, 1, 0), (45, 2, 1), (95, 0, 0), (96, 1, 0), (120, 2, 1))]
POST_LEVELS = [(61, 101, 8, 4, 32, 0, 0), (31, 51, 16, 32, 64, 0, 0), (16, 26, 32, 64, 128, 0, 0), (8, 13, 64, 128, 256, 0, 0)]   # P = 8262
POST_SCALES = [(300, 490, 0.5), (290, 480, 1.0), (200, 333, 1.7)]         # (img_h, img_w, resize_scale): boxes cross the right / bottom edges
SCORE_THR, IOU_THR = 0.3, 0.45


def _post_id(c):
    return 'cls%d_C%d_bbox%d_agn%d_N%d' % c


def candidate_kernel(cls_mode, C_, P, max_ctas, sms=132):
    """The candidate kernel candidates_launch picks, and the rounds of the flat kernel's loop."""
    if cls_mode == 0 and C_ > 1:
        blocks = min((P * C_ + 255) // 256, 8 * (max_ctas or sms))
        return 'flat', -(-(P * C_) // (blocks * 256))
    Cs = C_ + 1 if cls_mode == 1 else C_
    if Cs > 1 and 128 * Cs * 4 <= 48 * 1024:
        return 'rows', 1
    return 'thread', 1


def _scores64(cls_mode, x):
    x = torch.from_numpy(x).double()
    return (x.softmax(-1)[..., :-1] if cls_mode == 1 else torch.sigmoid(x)).numpy()


def _decode64(bbox_mode, reg, pt, img_h, img_w, rs):
    r = torch.from_numpy(reg).double()
    hi = torch.from_numpy(pt['hi']).double()[:, None]
    d = torch.sigmoid(r) * hi if bbox_mode == 0 else torch.exp(r) if bbox_mode == 1 else r * hi
    px, py = torch.from_numpy(pt['px']).double(), torch.from_numpy(pt['py']).double()
    b = torch.stack([(px - d[:, 0]).clamp(0, img_w), (py - d[:, 1]).clamp(0, img_h), (px + d[:, 2]).clamp(0, img_w), (py + d[:, 3]).clamp(0, img_h)], -1)
    return (b / rs).numpy()


def _decode32(reg, pt, img_h, img_w, rs):
    """'independent' decode exactly as decode_point: every step one fp32 operation."""
    d = (reg * pt['hi'][:, None]).astype(np.float32)
    px, py = pt['px'], pt['py']
    f = lambda v, m: (np.minimum(np.maximum(v.astype(np.float32), np.float32(0)), np.float32(m)) / np.float32(rs)).astype(np.float32)
    return np.stack([f(px - d[:, 0], img_w), f(py - d[:, 1], img_h), f(px + d[:, 2], img_w), f(py + d[:, 3], img_h)], -1)


def _iou64(a, b):
    lt, rb = np.maximum(a[:, None, :2], b[None, :, :2]), np.minimum(a[:, None, 2:], b[None, :, 2:])
    wh = np.clip(rb - lt, 0, None)
    inter = wh[..., 0] * wh[..., 1]
    aa, ab = (a[:, 2] - a[:, 0]) * (a[:, 3] - a[:, 1]), (b[:, 2] - b[:, 0]) * (b[:, 3] - b[:, 1])
    with np.errstate(divide='ignore', invalid='ignore'):
        return inter / (aa[:, None] + ab[None, :] - inter)


def post_inputs(case, n_cand=None):
    """Logits and regression outputs with margins: candidate scores >= 1e-5 from the threshold and from each other (exact duplicates
    only from duplicated logits), and no candidate pair of one NMS group within 1e-3 of the IoU threshold (the fp32 class offsets
    move the IoU of boxes near 1000 px by a few 1e-4)."""
    cls_mode, C_, bbox, agn, N = case
    lv = ref.level_table(POST_LEVELS)
    pt = ref.point_table(lv)
    P = lv['P']
    rng = np.random.RandomState(C_ * 10 + bbox + 100 * cls_mode)
    Cs = C_ + 1 if cls_mode == 1 else C_
    frac = (n_cand or 60) / float(P * C_)
    x = np.where(rng.rand(N, P, Cs) < frac, rng.uniform(1.0, 6.0, (N, P, Cs)), rng.uniform(-12, -4, (N, P, Cs))).astype(np.float32)
    if cls_mode == 1:
        x[..., -1] = np.where(rng.rand(N, P) < 0.3, 2.0, -2.0)
    x[:, lv['off'], 0] = 7.0 + np.arange(lv['num_levels'])   # the first point of every level is a candidate (the level lookup at its offset)
    x[:, lv['off'], -1] = -2.0 if cls_mode == 1 else x[:, lv['off'], -1]
    if bbox == 2:
        reg = rng.uniform(0.05, 0.6, (N, P, 4)).astype(np.float32)
    elif bbox == 1:
        reg = np.log(np.tile(pt['hi'], (N, 1))[..., None] * rng.uniform(0.05, 0.6, (N, P, 4))).astype(np.float32)
    else:
        reg = rng.uniform(-3, 0.5, (N, P, 4)).astype(np.float32)
    for it in range(6):
        changed = False
        for n in range(N):
            h, w, rs = POST_SCALES[n % 3]
            sc = _scores64(cls_mode, x[n])
            near = (sc > SCORE_THR - 1e-5) & (sc < SCORE_THR + 1e-5)
            cand = sc > SCORE_THR
            flat = np.sort(sc[cand])
            gaps = np.diff(flat)
            close = set(flat[1:][(gaps < 1e-5) & (gaps > 0)].tolist())
            near |= cand & np.isin(sc, list(close))
            boxes = _decode64(bbox, reg[n], pt, h, w, rs)
            ci, cc = np.nonzero(cand & ~near)
            groups = [np.arange(ci.size)] if agn else [np.nonzero(cc == c)[0] for c in range(C_)]
            for gidx in groups:
                if gidx.size < 2:
                    continue
                iou = _iou64(boxes[ci[gidx]], boxes[ci[gidx]])
                bad = np.abs(iou - IOU_THR) < 1e-3
                np.fill_diagonal(bad, False)
                for a, b2 in zip(*np.nonzero(np.triu(bad))):
                    v = a if ci[gidx[b2]] in lv['off'] else b2          # keep the level's first point
                    near[ci[gidx[v]], cc[gidx[v]]] = True
            if near.any():
                changed = True
                i_, c_ = np.nonzero(near)
                x[n, i_, c_] = -20.0
        if not changed:
            break
    assert not changed
    return lv, pt, x, reg


def run_post(case, lv, x, reg, cap, max_ctas):
    cls_mode, C_, bbox, agn, N = case
    c = nat.PostCfg()
    c.N, c.P, c.C, c.cls_channels = N, lv['P'], C_, x.shape[-1]
    c.cls_mode, c.bbox_mode, c.class_agnostic, c.num_levels = cls_mode, bbox, agn, lv['num_levels']
    for l in range(lv['num_levels']):
        c.level_off[l], c.level_w[l], c.level_stride[l], c.level_hi[l] = lv['off'][l], lv['w'][l], lv['stride'][l], float(lv['hi'][l])
    c.score_thr, c.iou_thr, c.cap, c.max_ctas = SCORE_THR, IOU_THR, cap, max_ctas
    meta = [torch.tensor([float(POST_SCALES[n % 3][i]) for n in range(N)], device=DEV) for i in (1, 0, 2)]
    ws = torch.zeros(int(nat.lib().lfd_postprocess_workspace_bytes(C.byref(c))), dtype=torch.uint8, device=DEV)
    dets = torch.full((N, cap, 5), NAN, device=DEV)
    labels = torch.full((N, cap), -7, dtype=torch.int32, device=DEV)
    src = torch.full((N, cap), -7, dtype=torch.int32, device=DEV)
    count = torch.full((N,), -7, dtype=torch.int32, device=DEV)
    ovf = torch.full((1,), -7, dtype=torch.int32, device=DEV)
    xd, rd = torch.from_numpy(x).to(DEV), torch.from_numpy(reg).to(DEV)
    nat.check(nat.lib().lfd_postprocess(C.byref(c), nat.ptr(xd), nat.ptr(rd), *[nat.ptr(t) for t in meta], nat.ptr(ws), nat.ptr(dets), nat.ptr(labels),
                                        nat.ptr(src), nat.ptr(count), nat.ptr(ovf), nat.stream_ptr()))
    torch.cuda.synchronize()
    cnt = count.cpu().tolist()
    return [(dets[n, :cnt[n]].cpu().numpy(), labels[n, :cnt[n]].cpu().numpy(), src[n, :cnt[n]].cpu().numpy()) for n in range(N)], int(ovf.item())


def _post_check(case, lv, pt, x, reg, res):
    cls_mode, C_, bbox, agn, N = case
    for n in range(N):
        h, w, rs = POST_SCALES[n % 3]
        sc64 = _scores64(cls_mode, x[n])
        b = _decode32(reg[n], pt, h, w, rs) if bbox == 2 else _decode64(bbox, reg[n], pt, h, w, rs).astype(np.float32)
        odets, olab, osrc = orc.multiclass_nms(b, sc64.astype(np.float32), SCORE_THR, IOU_THR, class_agnostic=bool(agn))
        dets, lab, src = res[n]
        assert src.tolist() == osrc.tolist(), ('image', n, len(src), len(osrc))
        assert lab.tolist() == olab.tolist()
        want = sc64.reshape(-1)[osrc]
        # sigmoid: expf and two roundings, 3 ulp; softmax: plus the fp32 sum of C + 1 exponentials in the denominator
        ulps = 3 if cls_mode == 0 else 4 + x.shape[-1]
        assert np.all(np.abs(dets[:, 4] - want) <= ulps * np.spacing(want.astype(np.float32))), 'scores off'
        if bbox == 2:
            assert np.array_equal(dets[:, :4].view(np.uint32), odets[:, :4].view(np.uint32)), 'independent decode rows must be bit-exact'
        else:   # expf and the decode: a few ulp of the largest coordinate; class-aware: the fp32 round trip through the class offset
            top = np.float32(max(h, w) / rs)
            tol = 8 * np.spacing(top) + (0 if agn else 2 * np.spacing(np.float32(C_ * (top + 1))))
            assert np.all(np.abs(dets[:, :4] - odets[:, :4]) <= tol), ('rows off', float(np.abs(dets[:, :4] - odets[:, :4]).max()))


@pytest.mark.gpu
@pytest.mark.parametrize('case', POST_CASES, ids=_post_id)
def test_postprocess_against_oracle(case):
    lv, pt, x, reg = post_inputs(case)
    results = []
    for m in GRIDS:
        res, ovf = run_post(case, lv, x, reg, 8192, m)
        assert ovf == 0
        results.append(res)
    for r in results[1:]:
        for a, b in zip(results[0], r):
            for u, v in zip(a, b):
                assert np.array_equal(np.asarray(u).view(np.uint32), np.asarray(v).view(np.uint32)), 'outputs differ between grids'
    _post_check(case, lv, pt, x, reg, results[0])


@pytest.mark.gpu
def test_postprocess_mixed_paths_and_capacity():
    """Image 0 without candidates, image 1 on the bit-matrix path (<= 1024), image 2 on the global-memory per-class path (> 4096):
    the per-image scratch stride.  Then cap == the largest count (no overflow) and cap == count - 1 (overflow reported)."""
    case = (0, 45, 2, 0, 3)
    lv, pt, x, reg = post_inputs(case, n_cand=11000)
    x[0] = -20.0
    x[1, 400:] = -20.0
    sc = [int((_scores64(0, x[n]) > SCORE_THR).sum()) for n in range(3)]
    assert sc[0] == 0 and 0 < sc[1] <= 1024 and sc[2] > 4096, sc
    res, ovf = run_post(case, lv, x, reg, max(sc), 0)
    assert ovf == 0
    _post_check(case, lv, pt, x, reg, res)
    _, ovf = run_post(case, lv, x, reg, max(sc) - 1, 0)
    assert ovf == 1


# ================================================================================================ CPU: the tables reach every decision
def test_assign_reference_matches_oracle_on_goldens():
    """assign_ref against orc.assign_targets (itself pinned to the reference's output) on the recorded batches, bit for bit."""
    from helpers import load_golden
    for name in ('WIDERFACE_S', 'WIDERFACE_L', 'TT100K_L'):
        g = load_golden('assign_%s.pt' % name)
        cfg = orc.CONFIGS[name]
        lc = cfg['lfd']
        grays = orc.gray_ranges_of(lc['regression_ranges'], lc['gray_range_factors'])
        specs = [(h, w, s, r[0], r[1], gr[0], gr[1]) for (h, w), s, r, gr in zip(g['sizes'], orc.strides_of(cfg), lc['regression_ranges'], grays)]
        lv = ref.level_table(specs)
        mode = dict(dist=0, longer=1, shorter=2)[lc['range_assign_mode']]
        for boxes, labels in g['ann']:
            ct, rt, _, _ = ref.assign_ref(lv, lc['num_classes'], mode, 0, boxes, labels)
            oct_, ort = orc.assign_targets(cfg, g['sizes'], boxes, labels)
            assert np.array_equal(ct, oct_) and np.array_equal(rt, ort), name


@pytest.mark.parametrize('kind', range(4))
def test_box_loss_reference_splits_tied_edges(kind):
    """At a predicted edge equal to the target edge the reference's gradient (torch.max / torch.min) is the mean of the two one-sided
    derivatives; pred (10, 12, 20, 25) against target (10, 10, 22, 20) ties at x1."""
    pr = torch.tensor([[10., 12., 20., 25.]], dtype=torch.float64, requires_grad=True)
    tg = torch.tensor([[10., 10., 22., 20.]], dtype=torch.float64)
    ref.iou_family(kind, pr, tg, 1e-6).sum().backward()
    h = 1e-6
    f = lambda dx: ref.iou_family(kind, pr.detach() + torch.tensor([[dx, 0., 0., 0.]], dtype=torch.float64), tg, 1e-6).item()
    right, left = (f(h) - f(0.)) / h, (f(0.) - f(-h)) / h
    assert abs(right - left) > 1e-3                                   # a real kink
    assert abs(pr.grad[0, 0].item() - 0.5 * (right + left)) < 1e-5


def test_case_tables_reach_every_decision():
    # assignment: every C, mode x independent, level count, G = 0 and padding, both P kinds; every boundary per assign_mode
    assert {c[0] for c in ASSIGN_CASES} == {1, 2, 45, 100} and {(c[1], c[2]) for c in ASSIGN_CASES} == {(m, i) for m in range(3) for i in (0, 1)}
    assert {len(_HW[c[3]]) for c in ASSIGN_CASES} == {1, 5, 8}
    Ps = {ref.level_table(level_specs(c[3])).get('P') for c in ASSIGN_CASES}
    assert 17 in Ps and all(p == 17 or p % 256 == 5 for p in Ps)
    assert any(0 in c[4] for c in ASSIGN_CASES) and {len(c[4]) for c in ASSIGN_CASES} >= {1, 2, 4}
    for mode in range(3):
        tot = {}
        for case in ASSIGN_CASES:
            if case[1] != mode:
                continue
            for k, v in assign_boundaries(case).items():
                tot[k] = tot.get(k, 0) + v
        for k in ('lo', 'hi', 'glo', 'ghi', 'edge0', 'edge1', 'edge2', 'edge3', 'tie', 'green_gray_same', 'gray_other', 'low_score', 'empty'):
            assert tot[k] > 0, (mode, k, tot)
    # losses: each cls_mode at C 1 / 2 / 45; gamma and alpha values; special batches; regression kinds x decodes, eps values
    assert {(c[0], c[1]) for c in CLS_CASES} >= {(m, c) for m in range(4) for c in (1, 2, 45)}
    assert {c[2] for c in CLS_CASES} == {0.0, 1.5, 2.0} and {c[3] for c in CLS_CASES} == {0.25, 0.5}
    assert {c[4] for c in CLS_CASES} == {'mixed', 'ignored', 'nopos'}
    assert {(c[0], c[1]) for c in REG_CASES} == {(k, b) for k in range(4) for b in (0, 1)} | {(4, 2), (5, 2)}
    assert {c[2] for c in REG_CASES} == {1e-6, 1e-3}
    # the loss launches: >= 3 passes per thread with a remainder at max_ctas 1 and 3 (4 * max_ctas blocks of 256)
    rows = LOSS_N * LOSS_LV['P']
    for m in (1, 3):
        stride = 4 * m * 256
        for n in [rows] + [rows * c for c in (1, 2, 45)]:
            assert n // stride >= 3 and n % stride, (n, m)
    # post-process: every candidate kernel, the flat kernel's rounds, every bbox_mode, agnostic both ways
    P = ref.level_table(POST_LEVELS)['P']
    assert {candidate_kernel(c[0], c[1], P, 0)[0] for c in POST_CASES} == {'flat', 'rows', 'thread'}
    assert candidate_kernel(1, 95, 1, 0)[0] == 'rows' and candidate_kernel(1, 96, 1, 0)[0] == 'thread'
    for c in POST_CASES:
        if c[0] == 0 and c[1] > 1:
            for m in (1, 3):
                assert candidate_kernel(0, c[1], P, m)[1] >= 3, c
    assert {c[2] for c in POST_CASES} == {0, 1, 2} and {c[3] for c in POST_CASES} == {0, 1}
    for c in POST_CASES:           # every level's first point stays a candidate through the margin pruning
        lv, pt, x, reg = post_inputs(c)
        for n in range(c[4]):
            assert (_scores64(c[0], x[n])[lv['off'], 0] > SCORE_THR).all(), c
    # NMS: every path of nms_kernel
    paths = set()
    for case in NMS_CASES:
        name, K, C_, agn, sp = case
        b, s, lab = nms_inputs(case, np.random.RandomState(K + C_))
        segs = np.bincount(lab) if name != 'raw' else None
        paths.add(nms_path(K, 1 if name == 'raw' else C_, agn or name == 'raw', float(b.min()), segs[segs > 0] if segs is not None else None))
        if sp == 'seg512':
            assert {512, 513} <= set(np.bincount(lab).tolist())
    assert {'4a', '4b', '4b_gmem', '4c', '4c_long', '4c_gmem'} <= paths, paths
    assert any(c[2] > 32 and not c[3] and c[1] > 1024 for c in NMS_CASES)
