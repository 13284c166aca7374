# -*- coding: utf-8 -*-
"""References for the label assignment, detection-loss and post-process kernels (csrc/losses.cu, csrc/postprocess.cu).

  * assign_ref: a float32 numpy restatement of lfd.py:155-259, vectorised over (point, gt), that takes a level table directly and
    covers every range_assign_mode, 'independent' targets (deltas / hi), the row label and the counters.  Every step is one IEEE
    fp32 operation, as in the kernel (_rn intrinsics, no FMA), so the kernel must match it bit for bit.
  * R: a float64 value carried with a running magnitude S, so that an fp32 evaluation of the same formula differs from the value by
    at most K * 2^-24 * S, where K counts the roundings along the longest path.  S follows first-order error propagation from S(x) = |x|
    for inputs and constants: S(a +- b) = S(a) + S(b), S(a * b) = S(a) |b| + |a| S(b), S(a / b) = (S(a) + |a / b| S(b)) / |b|,
    S(f(a)) = |f(a)| + |f'(a)| S(a).  Cancellations such as 1 - sigmoid(15) or log(1 + exp(-10)) therefore keep the magnitude of their
    operands.
  * cls_ref / reg_ref: float64 losses and gradients on the kernel's own fp32 inputs, from torch autograd of the reference formulas
    (tie and clamp semantics come from torch itself), with the magnitudes of the formulas the kernel evaluates.
"""
import numpy as np
import torch
import torch.nn.functional as F

F32 = np.float32


# ================================================================================================ level tables and assignment
def level_table(specs):
    """specs: [(h, w, stride, lo, hi, glo, ghi)] -> dict of per-level arrays (the fields of lfd_levels) plus P."""
    off, o = [], 0
    for h, w, *_ in specs:
        off.append(o)
        o += h * w
    cols = list(zip(*specs))
    return dict(num_levels=len(specs), off=off, h=list(cols[0]), w=list(cols[1]), stride=list(cols[2]),
                lo=[F32(v) for v in cols[3]], hi=[F32(v) for v in cols[4]], glo=[F32(v) for v in cols[5]], ghi=[F32(v) for v in cols[6]], P=o)


def point_table(lv):
    """Per point (float32): px, py, half, lo, hi, glo, ghi, level -- point_geom of losses.cu / decode_point of postprocess.cu."""
    cols = {k: [] for k in ('px', 'py', 'half', 'lo', 'hi', 'glo', 'ghi', 'level')}
    for l in range(lv['num_levels']):
        h, w, s = lv['h'][l], lv['w'][l], lv['stride'][l]
        local = np.arange(h * w)
        cols['px'].append(((local % w) * s).astype(F32))
        cols['py'].append(((local // w) * s).astype(F32))
        cols['half'].append(np.full(h * w, F32(s) / F32(2), F32))
        for k in ('lo', 'hi', 'glo', 'ghi'):
            cols[k].append(np.full(h * w, lv[k][l], F32))
        cols['level'].append(np.full(h * w, l, np.int64))
    return {k: np.concatenate(v) for k, v in cols.items()}


def _center_score(d, half):
    s = np.abs(d) / half
    s = np.where(s >= F32(1), s, F32(1)).astype(F32)
    return np.sqrt(F32(1) / s).astype(F32)


def assign_geometry(lv, mode, boxes):
    """-> per (point, gt): deltas [P,G,4], measure [P,G], hit [P,G], green [P,G], gray [P,G], score [P,G] (float32)."""
    pt = point_table(lv)
    b = np.asarray(boxes, F32).reshape(-1, 4)
    px, py = pt['px'][:, None], pt['py'][:, None]
    x, y, w, h = (b[None, :, k] for k in range(4))
    one = F32(1)
    d = np.stack([px - x, py - y, ((x + w) - one) - px, ((y + h) - one) - py], -1).astype(F32)
    if mode == 0:
        measure = d.max(-1)
    elif mode == 1:
        measure = np.broadcast_to(np.maximum(w, h), d.shape[:2])
    else:
        measure = np.broadcast_to(np.minimum(w, h), d.shape[:2])
    lo, hi, glo, ghi = (pt[k][:, None] for k in ('lo', 'hi', 'glo', 'ghi'))
    hit = d.min(-1) >= 0
    green = hit & (lo <= measure) & (measure <= hi)
    gray = hit & (((glo <= measure) & (measure < lo)) | ((hi < measure) & (measure <= ghi)))
    cx, cy = x + w / F32(2), y + h / F32(2)
    score = (_center_score(px - cx, pt['half'][:, None]) * _center_score(py - cy, pt['half'][:, None])).astype(F32)
    return dict(d=d, measure=measure, hit=hit, green=green, gray=gray, score=score, pt=pt)


def assign_ref(lv, C, mode, independent, boxes, labels):
    """One image: -> cls_target [P,C], reg_target [P,4], label [P] (-1 ignore, C background), (n_pos, n_valid)."""
    P = lv['P']
    labels = np.asarray(labels, np.int64).reshape(-1)
    G = labels.size
    cls_t = np.zeros((P, C), F32)
    reg_t = np.zeros((P, 4), F32)
    if G:
        g = assign_geometry(lv, mode, boxes)
        sc = np.where(g['green'], g['score'], F32(0))
        gray_any = np.zeros((P, C), bool)
        for c in np.unique(labels):
            m = labels == c
            cls_t[:, c] = np.maximum(cls_t[:, c], sc[:, m].max(-1))
            gray_any[:, c] = g['gray'][:, m].any(-1)
        best = sc.argmax(-1)                               # first maximum: the lowest gt index among equal scores
        has = sc.max(-1) > 0
        dl = g['d'][np.arange(P), best]
        if independent:
            dl = (dl / g['pt']['hi'][:, None]).astype(F32)
        reg_t[has] = dl[has]
        cls_t[gray_any] = F32(-1)
    mx, arg = cls_t.max(-1), cls_t.argmax(-1)
    label = np.where(cls_t.min(-1) < 0, -1, np.where(mx >= F32(0.001), arg, C)).astype(np.int32)
    return cls_t, reg_t, label, (int(((label >= 0) & (label < C)).sum()), int((label >= 0).sum()))


# ================================================================================================ magnitude-tracking float64
class R(object):
    """float64 value v with the magnitude S of the formula that produced it (see the module docstring)."""

    def __init__(self, v, s=None):
        self.v = torch.as_tensor(v, dtype=torch.float64)
        self.s = self.v.abs() if s is None else s

    @staticmethod
    def c(v):
        return v if isinstance(v, R) else R(v)

    def __add__(a, b):
        b = R.c(b)
        return R(a.v + b.v, a.s + b.s)
    __radd__ = __add__

    def __sub__(a, b):
        b = R.c(b)
        return R(a.v - b.v, a.s + b.s)

    def __rsub__(a, b):
        return R.c(b) - a

    def __neg__(a):
        return R(-a.v, a.s)

    def __mul__(a, b):
        b = R.c(b)
        return R(a.v * b.v, a.s * b.v.abs() + a.v.abs() * b.s)
    __rmul__ = __mul__

    def __truediv__(a, b):
        b = R.c(b)
        q = a.v / b.v
        return R(q, (a.s + q.abs() * b.s) / b.v.abs())

    def __rtruediv__(a, b):
        return R.c(b) / a

    def fn(a, f, df):
        v = f(a.v)
        return R(v, v.abs() + df(a.v).abs() * a.s)

    def exp(a):
        return a.fn(torch.exp, torch.exp)

    def log(a):
        return a.fn(torch.log, lambda x: 1.0 / x)

    def log1p(a):
        return a.fn(torch.log1p, lambda x: 1.0 / (1.0 + x))

    def pow(a, g):
        if g == 0:
            return R(torch.ones_like(a.v))
        return a.fn(lambda x: x.pow(g), lambda x: g * x.pow(g - 1) if g >= 1 else torch.where(x > 0, g * x.pow(g - 1), torch.zeros_like(x)))

    def abs(a):
        return R(a.v.abs(), a.s)

    def sel(m, a, b):
        a, b = R.c(a), R.c(b)
        return R(torch.where(m, a.v, b.v), torch.where(m, a.s, b.s))


def _sigmoid_r(x):
    return 1.0 / (1.0 + (-x).exp())


# ================================================================================================ classification losses
def cls_ref(mode, x32, label, C, gamma, alpha, q32=None):
    """Element-wise classification loss and d loss / d x (before the 1 / (n_pos + 1) * weight scale) on the kernel's fp32 logits.
    x32 [M, Cp] float32, label [M] (-1: ignored row), q32 [M, C] the soft targets (BCE, QFL).
    -> loss [M, Cp], grad [M, Cp], S_loss, S_grad (float64; ignored rows 0)."""
    x = torch.as_tensor(x32).double().clone().requires_grad_(True)
    M, Cp = x.shape
    t = torch.as_tensor(label).long()[:, None]
    d = torch.arange(Cp)[None, :]
    valid = (t >= 0).expand(M, Cp)
    if mode == 0:      # sigmoid focal: sigmoid_focal_loss_cuda.cu:24-97 (the backward is the reference's own analytic formula)
        c1, c2 = (t == d).double(), ((t >= 0) & (t != d)).double()
        xv = x.detach()
        p = torch.sigmoid(xv)
        l1 = -xv * (xv >= 0) - torch.log1p(torch.exp(xv - 2.0 * xv * (xv >= 0)))
        term1 = (1 - p).pow(gamma) * torch.log(p.clamp(min=torch.finfo(torch.float32).tiny))
        term2 = p.pow(gamma) * l1
        loss = -c1 * term1 * alpha - c2 * term2 * (1 - alpha)
        g1 = (1 - p).pow(gamma) * (1 - p - p * gamma * torch.log(p.clamp(min=torch.finfo(torch.float32).tiny)))
        g2 = p.pow(gamma) * (l1 * (1 - p) * gamma - p)
        grad = -c1 * g1 * alpha - c2 * g2 * (1 - alpha)
        # magnitudes of the kernel's evaluation of the same formulas
        X = R(xv)
        P_ = _sigmoid_r(X)
        pos = (xv >= 0).double()
        L1 = -(X * pos) - (1.0 + (X - 2.0 * X * pos).exp()).log()
        lp = R.sel(xv > -87, P_.log(), R(torch.log(p.clamp(min=torch.finfo(torch.float32).tiny))))
        T1 = (1.0 - P_).pow(gamma) * lp
        T2 = P_.pow(gamma) * L1
        SL = (c1 * alpha * T1.s + c2 * (1 - alpha) * T2.s)
        G1 = (1.0 - P_).pow(gamma) * (1.0 - P_ - P_ * gamma * lp)
        G2 = P_.pow(gamma) * (L1 * (1.0 - P_) * gamma - P_)
        SG = (c1 * alpha * G1.s + c2 * (1 - alpha) * G2.s)
    elif mode == 1:    # cross entropy over C + 1 logits (cross_entropy_loss.py:12-22)
        tt = t.clamp(min=0)[:, 0]
        loss_row = F.cross_entropy(x, tt, reduction='none')
        loss_row.sum().backward()
        loss = torch.zeros(M, Cp, dtype=torch.float64)
        loss[:, 0] = loss_row.detach()
        grad = x.grad.clone()
        X = R(x.detach())
        mx = x.detach().max(-1, keepdim=True)[0]
        E = (X - R(mx)).exp()
        den = R(E.v.sum(-1, keepdim=True), E.s.sum(-1, keepdim=True))
        lrow = R(X.v.gather(1, tt[:, None]), X.s.gather(1, tt[:, None])) - R(mx) - den.log()
        SL = torch.zeros(M, Cp, dtype=torch.float64)
        SL[:, 0] = lrow.s[:, 0]                                   # one value per row, kept in column 0
        SG = (E / den).s + (t == d).double()
    else:
        q = torch.as_tensor(q32).double()
        xv = x.detach()
        if mode == 2:  # BCE with logits against the soft targets (bce_with_logits_loss.py:28-44)
            loss = F.binary_cross_entropy_with_logits(x, q, reduction='none')
        else:          # quality focal loss (gfocal_loss.py:10-49): negatives BCE(x, 0) * sigmoid^beta, the label class BCE(x, quality) * |quality - sigmoid|^beta
            qual = q.max(-1, keepdim=True)[0].expand(M, Cp)
            sg = torch.sigmoid(x)
            neg = F.binary_cross_entropy_with_logits(x, torch.zeros_like(x), reduction='none') * sg.pow(gamma)
            posl = F.binary_cross_entropy_with_logits(x, qual, reduction='none') * (qual - sg).abs().pow(gamma)
            loss = torch.where(t == d, posl, neg)
        loss.sum().backward()
        grad = x.grad.clone()
        loss = loss.detach()
        X = R(xv)
        SG_ = _sigmoid_r(X)
        SP = R(xv.clamp(min=0)) + (1.0 + (-X.abs()).exp()).log()
        if mode == 2:
            Q = R(q)
            L = SP - X * Q
            Gd = SG_ - Q
        else:
            qual = q.max(-1, keepdim=True)[0].expand(M, Cp)
            Q = R(qual)
            Mn = SG_.pow(gamma)
            Ln = SP * Mn
            Gn = SG_ * Mn + SP * gamma * Mn * (1.0 - SG_)
            A = (Q - SG_).abs()
            Ma = A.pow(gamma)
            B = SP - X * Q
            Lp = B * Ma
            Gp = (SG_ - Q) * Ma + B * gamma * A.pow(gamma - 1 if gamma >= 1 else 0) * SG_ * (1.0 - SG_)
            L = R.sel(t == d, Lp, Ln)
            Gd = R.sel(t == d, Gp, Gn)
        SL, SG = L.s, Gd.s
    z = torch.zeros_like(loss)
    return (torch.where(valid, loss.detach(), z), torch.where(valid, grad.detach(), z), torch.where(valid, SL, z), torch.where(valid, SG, z))


# ================================================================================================ regression losses
def iou_family(kind, pr, tg, eps):
    """Row loss of the reference's IoU losses (iou_loss.py:66-80,105-283) on float64 xyxy boxes (pr may require grad)."""
    if kind == 0:
        lt = torch.max(pr[:, :2], tg[:, :2])
        rb = torch.min(pr[:, 2:], tg[:, 2:])
        wh = (rb - lt).clamp(min=0)
        ov = wh[:, 0] * wh[:, 1]
        a1 = (pr[:, 2] - pr[:, 0]) * (pr[:, 3] - pr[:, 1])
        a2 = (tg[:, 2] - tg[:, 0]) * (tg[:, 3] - tg[:, 1])
        un = torch.clamp(a1 + a2 - ov, min=1e-6)
        return -(ov / un).clamp(min=eps).log()
    lt = torch.max(pr[:, :2], tg[:, :2])
    rb = torch.min(pr[:, 2:], tg[:, 2:])
    wh = (rb - lt).clamp(min=0)
    overlap = wh[:, 0] * wh[:, 1]
    ap = (pr[:, 2] - pr[:, 0]) * (pr[:, 3] - pr[:, 1])
    ag = (tg[:, 2] - tg[:, 0]) * (tg[:, 3] - tg[:, 1])
    union = ap + ag - overlap + eps
    ious = overlap / union
    ewh = (torch.max(pr[:, 2:], tg[:, 2:]) - torch.min(pr[:, :2], tg[:, :2])).clamp(min=0)
    if kind == 1:
        area = ewh[:, 0] * ewh[:, 1] + eps
        return 1 - (ious - (area - union) / area)
    c2 = ewh[:, 0] ** 2 + ewh[:, 1] ** 2 + eps
    rho2 = ((tg[:, 0] + tg[:, 2]) - (pr[:, 0] + pr[:, 2])) ** 2 / 4 + ((tg[:, 1] + tg[:, 3]) - (pr[:, 1] + pr[:, 3])) ** 2 / 4
    if kind == 2:
        return 1 - (ious - rho2 / c2)
    w1, h1 = pr[:, 2] - pr[:, 0], pr[:, 3] - pr[:, 1] + eps
    w2, h2 = tg[:, 2] - tg[:, 0], tg[:, 3] - tg[:, 1] + eps
    v = (4 / np.pi ** 2) * torch.pow(torch.atan(w2 / h2) - torch.atan(w1 / h1), 2)
    return 1 - (ious - (rho2 / c2 + v ** 2 / (1 - ious + v)))


def box_row_magnitude(kind, pr, tg, loss, g):
    """Magnitude S of the kernel's fp32 evaluation of one IoU-family row and its four gradients: the terms of the formula are areas
    and extents of the two boxes, so each gradient is bounded by (|loss| + sum |g|) over the smallest positive extent, plus |g|."""
    ext = torch.cat([(pr[:, 2:] - pr[:, :2]).abs(), (tg[:, 2:] - tg[:, :2]).abs()], 1)
    ext = torch.where(ext > 0, ext, torch.full_like(ext, float('inf'))).min(-1)[0].clamp(min=1e-3)
    big = torch.cat([pr.abs(), tg.abs()], 1).max(-1)[0]
    row = (loss.abs() + 1.0 + g.abs().sum(-1)) * (1.0 + big / ext)
    return row, row[:, None] + g.abs()


def box_loss_ref(kind, pred32, target32, eps):
    """The stand-alone box losses (lfd_box_loss): -> loss [n], grad [n,4], S_loss [n], S_grad [n,4] (float64)."""
    pr = torch.as_tensor(pred32).double().clone().requires_grad_(True)
    tg = torch.as_tensor(target32).double()
    l = iou_family(kind, pr, tg, float(np.float32(eps)))
    l.sum().backward()
    sl, sg = box_row_magnitude(kind, pr.detach(), tg, l.detach(), pr.grad)
    return l.detach(), pr.grad.clone(), sl, sg


def decode32(bbox_mode, raw32, hi32):
    """The kernel's fp32 decode of the four distances and d distance / d raw (float64, from the fp32 sigmoid) with its magnitude."""
    raw = torch.as_tensor(raw32)
    hi = torch.as_tensor(hi32)[:, None]
    if bbox_mode == 0:
        s = torch.sigmoid(raw)
        d = (s * hi).float()
        s64, h64 = torch.sigmoid(raw.double()), hi.double()
        dd = h64 * s64 * (1 - s64)
        sdd = h64 * s64 * (1 + s64) + dd
    else:
        d = torch.exp(raw).float()
        dd = torch.exp(raw.double())
        sdd = dd
    return d, dd, sdd


def reg_ref(kind, bbox_mode, raw32, tgt32, px, py, hi32, eps, beta):
    """Row regression loss and d loss / d raw (before the 1 / n_pos * weight scale) of positive rows.
    -> loss [n], grad [n,4], S_loss [n], S_grad [n,4]."""
    raw = torch.as_tensor(raw32)
    tgt = torch.as_tensor(tgt32).double()
    if kind >= 4:      # SmoothL1 (smooth_l1_loss.py:10-28) / MSE on the raw outputs against the range-normalised targets
        x = raw.double().clone().requires_grad_(True)
        if kind == 4:
            l = F.smooth_l1_loss(x, tgt, reduction='none', beta=float(np.float32(beta))).sum(-1)
        else:
            l = F.mse_loss(x, tgt, reduction='none').sum(-1)
        l.sum().backward()
        df = (x.detach() - tgt).abs() + x.detach().abs() + tgt.abs()
        sg = df * (1.0 + 1.0 / float(np.float32(beta))) if kind == 4 else 2.0 * df
        return l.detach(), x.grad.clone(), (df * df / float(np.float32(beta)) + df).sum(-1) if kind == 4 else (df * df).sum(-1), sg
    d32, dd, sdd = decode32(bbox_mode, raw32, hi32)
    d = d32.double().clone().requires_grad_(True)
    px = torch.as_tensor(px).double()
    py = torch.as_tensor(py).double()
    pr = torch.stack([px - d[:, 0], py - d[:, 1], px + d[:, 2], py + d[:, 3]], -1)
    # the kernel forms both boxes in fp32 from the point and the distances
    tg = torch.stack([px - tgt[:, 0], py - tgt[:, 1], px + tgt[:, 2], py + tgt[:, 3]], -1).float().double()
    pr = pr + (pr.detach().float().double() - pr.detach())
    l = iou_family(kind, pr, tg, float(np.float32(eps)))
    l.sum().backward()
    gd = d.grad
    sl, sgd = box_row_magnitude(kind, pr.detach(), tg, l.detach(), gd)
    return l.detach(), gd * dd, sl, sgd * sdd + gd.abs() * dd
