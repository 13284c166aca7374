# -*- coding: utf-8 -*-
"""float64 reference of LFD.get_loss with enable_classification_weight / enable_regression_weight (lfd/model/lfd.py:313-387), built on
the element-wise references of tests/loss_post_ref.py:

  * the weight of a positive row is its maximal classification target, weight_sum their sum over the batch;
  * classification: avg_factor = weight_sum (weighted) or n_pos + 1, no per-element weight;
  * regression: row loss times its weight (weighted), avg_factor = weight_sum or n_pos; no positives: loss 0, gradients 0.

Also the level table, targets and inputs of tests/golden/loss_weighting.pt (tests/gen_golden_loss_weighting.py)."""
import numpy as np
import torch

import loss_post_ref as ref

F32 = np.float32
U = 2.0 ** -24
CLS_CODES = dict(FocalLoss=0, CrossEntropyLoss=1, BCEWithLogitsLoss=2, QualityFocalLoss=3)
REG_CODES = dict(IoULoss=0, GIoULoss=1, DIoULoss=2, CIoULoss=3, SmoothL1Loss=4, MSELoss=5)
BBOX_CODES = dict(sigmoid=0, exp=1, independent=2)
# the loss modules of the goldens (tests/gen_golden_variants.py::make_loss): (gamma or QFL beta, alpha, eps, SmoothL1 beta, loss_weight)
CLS_PARAMS = dict(FocalLoss=(2.0, 0.25, 1.0), CrossEntropyLoss=(2.0, 0.25, 1.0), BCEWithLogitsLoss=(2.0, 0.25, 1.0), QualityFocalLoss=(2.0, 0.25, 1.0))
REG_PARAMS = dict(IoULoss=(1e-6, 1.0, 1.0), GIoULoss=(1e-6, 1.0, 1.0), DIoULoss=(1e-6, 1.0, 1.0), CIoULoss=(1e-6, 1.0, 1.0),
                  SmoothL1Loss=(1e-6, 0.11, 2.0), MSELoss=(1e-6, 1.0, 1.5))


def row_weights(cls_t, label, C):
    """-> (positive mask [M], weights of every row [M] float64: the row maximum of the float32 targets, 0 elsewhere)."""
    pos = (label >= 0) & (label < C)
    w = np.where(pos, np.asarray(cls_t, F32).max(-1), F32(0)).astype(np.float64)
    return pos, w


def detection_loss_ref(cls_mode, reg_kind, bbox_mode, x, raw, cls_t, reg_t, label, px, py, hi, C, gamma, alpha, eps, beta, cls_lw, reg_lw,
                       cls_w, reg_w):
    """Rows flattened over the batch: x [M, Cp], raw [M, 4], cls_t [M, C], reg_t [M, 4], label [M], px / py / hi [M] (float32).
    -> dict of float64 tensors: cls_loss, reg_loss (the normalised values of get_loss), grad_cls [M, Cp], grad_reg [M, 4] and the
    magnitudes S_cls [M, Cp], S_reg [M, 4], S_cls_loss, S_reg_loss of the kernel's fp32 evaluation (loss_post_ref.R)."""
    M = x.shape[0]
    pos, w = row_weights(cls_t, label, C)
    n_pos = int(pos.sum())
    wsum = float(w.sum())
    l, g, sl, sg = ref.cls_ref(cls_mode, x, label, C, gamma, alpha, cls_t)
    cden = np.float64(wsum if cls_w else n_pos + 1)
    with np.errstate(divide='ignore', invalid='ignore'):         # weighted without positives: x / 0, as in the reference
        cscale = np.float64(cls_lw) / cden
        cls_loss = np.float64(cls_lw) * np.float64(l.sum()) / cden
        s_cls_loss = np.float64(cls_lw) * np.float64(sl.sum()) / cden
    ign = torch.from_numpy(np.asarray(label) < 0)[:, None]        # gray rows are not part of the loss: gradient 0 even when scaled by inf
    if cls_mode == 1 and cls_w:
        # cross entropy, weighted: softmax * s - onehot * s (autograd's log_softmax backward), so that s = inf gives NaN at the target
        onehot = torch.from_numpy(np.asarray(label, np.int64))[:, None] == torch.arange(g.shape[1])[None, :]
        sm = (g + onehot.double()) * float(cscale)
        gs = torch.where(onehot, sm - float(cscale), sm)
    else:
        gs = g * float(cscale)
    out = dict(n_pos=n_pos, weight_sum=wsum, grad_cls=gs.masked_fill(ign, 0.0), S_cls=(sg * float(cscale)).masked_fill(ign, 0.0),
               cls_loss=float(cls_loss), S_cls_loss=float(s_cls_loss))
    grad_reg = torch.zeros(M, 4, dtype=torch.float64)
    S_reg = torch.zeros(M, 4, dtype=torch.float64)
    out.update(reg_loss=0.0, S_reg_loss=0.0)
    if n_pos:
        idx = np.nonzero(pos)[0]
        rl, rg, rsl, rsg = ref.reg_ref(reg_kind, bbox_mode, raw[idx], reg_t[idx], px[idx], py[idx], hi[idx], eps, beta)
        wi = torch.from_numpy(w[idx]) if reg_w else torch.ones(idx.size, dtype=torch.float64)
        rden = wsum if reg_w else float(n_pos)
        f = float(reg_lw) * wi / rden
        grad_reg[idx] = rg * f[:, None]
        S_reg[idx] = rsg * f[:, None]
        out.update(reg_loss=float((rl * f).sum()), S_reg_loss=float((rsl * f).sum()))
    out.update(grad_reg=grad_reg, S_reg=S_reg)
    return out


def assert_close(got, want, S, K, what):
    """Finite references: |got - want| <= K * 2^-24 * S (+ a denormal floor); non-finite ones: the same inf (with sign) / NaN."""
    got, want, S = torch.as_tensor(got).double(), torch.as_tensor(want).double(), torch.as_tensor(S).double()
    fin = torch.isfinite(want)
    assert torch.equal(torch.isnan(got), torch.isnan(want)), (what, 'NaN pattern')
    assert torch.equal(got[torch.isinf(want)], want[torch.isinf(want)]), (what, 'inf pattern')
    err = (got[fin] - want[fin]).abs()
    tol = K * (U * S[fin] + 2.0 ** -126)
    bad = ~(err <= tol)
    assert not bool(bad.any()), '%s: %d / %d off, worst excess %g' % (what, int(bad.sum()), int(fin.sum()), float((err - tol).max()))


# ================================================================================================ the goldens' geometry
def golden_level_table(g):
    lo_f, hi_f = g['gray_range_factors']
    specs = [(h, w, s, lo, hi, int(lo * lo_f), int(hi * hi_f)) for (h, w), (lo, hi), s in zip(g['sizes'], g['ranges'], g['strides'])]
    return ref.level_table(specs)


def golden_targets(g, batch, independent):
    """-> cls_t [N*P, C], reg_t [N*P, 4], label [N*P] (numpy, bit-exact with lfd_assign_targets) and px, py, hi [N*P] of the golden batch."""
    lv = golden_level_table(g)
    C = g['num_classes']
    cts, rts, labs = [], [], []
    for boxes, labels in g['ann'][batch]:
        ct, rt, lab, _ = ref.assign_ref(lv, C, 0, independent, boxes, labels)
        cts.append(ct)
        rts.append(rt)
        labs.append(lab)
    pt = ref.point_table(lv)
    n = len(labs)
    return np.concatenate(cts), np.concatenate(rts), np.concatenate(labs), np.tile(pt['px'], n), np.tile(pt['py'], n), np.tile(pt['hi'], n)


def golden_grads(g, key):
    """The reference's gradients of one golden case: grad_cls [N*P, Cp] and grad_reg [N*P, 4] (zero outside the positive rows)."""
    cname, rname, cw, rw, batch = key
    gc = g['grad_cls'][(cname, cw, batch)]
    gr = torch.zeros(gc.shape[0] * gc.shape[1], 4)
    gr[g['pos_rows'][batch]] = g['grad_reg'][(rname, g['cases'][key]['bbox'], rw, batch)]
    return gc.reshape(-1, gc.shape[-1]), gr


def golden_case_ref(g, key, cls_pred=None, reg_pred=None):
    """The float64 reference of one golden case, on the golden's network outputs (or the given float32 ones)."""
    cname, rname, cw, rw, batch = key
    case = g['cases'][key]
    C = g['num_classes']
    Cp = C + 1 if cname == 'CrossEntropyLoss' else C
    x = (g['cls_pred'][Cp] if cls_pred is None else cls_pred).reshape(-1, Cp).numpy().astype(F32)
    raw = (g['reg_pred'][case['bbox']] if reg_pred is None else reg_pred).reshape(-1, 4).numpy().astype(F32)
    ct, rt, lab, px, py, hi = golden_targets(g, batch, int(case['bbox'] == 'independent'))
    gamma, alpha, clw = CLS_PARAMS[cname]
    eps, beta, rlw = REG_PARAMS[rname]
    return detection_loss_ref(CLS_CODES[cname], REG_CODES[rname], BBOX_CODES[case['bbox']], x, raw, ct, rt, lab, px, py, hi, C, gamma, alpha,
                              eps, beta, clw, rlw, cw, rw)
