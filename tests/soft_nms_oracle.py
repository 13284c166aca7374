# -*- coding: utf-8 -*-
"""Soft-NMS oracle: the reference's soft_nms_cpu loop (lfd/model/utils/build/nms/src/cpu/nms_cpu.cpp:76-206) restated in numpy fp32, and
the multiclass_nms / get_results of oracle/lfd_oracle.py with it as their NMS (nms.py:119-220 with nms_cfg type 'soft_nms').

The loop is the reference's: select the first position of the maximum score behind i (`max < s[pos]`, so a NaN at i is selected and a NaN
behind it never is), swap it to i, reweight every later position and drop it by swapping the last live element in when its score falls
below min_score.  Each step is one correctly rounded fp32 operation, as the reference's gcc -O2 x86-64 build computes it; the gaussian
weight is exp evaluated in float64 and rounded to fp32 (glibc's expf is not correctly rounded, so that mode matches the reference to
within an ulp per decay, and the device kernel bit for bit).
"""
import numpy as np

from oracle import lfd_oracle as orc

METHODS = {'linear': 1, 'gaussian': 2}


def soft_nms(dets, iou_thr, method='linear', sigma=0.5, min_score=1e-3):
    """dets [n,5] float32 -> (new_dets [k,5] float32 in selection order with the decayed scores, inds [k] int64 input rows)."""
    if method not in METHODS:
        raise ValueError('Invalid method for SoftNMS: {}'.format(method))
    d = np.array(dets, np.float32).reshape(-1, 5)
    n = d.shape[0]
    if n == 0:
        return np.zeros((0, 5), np.float32), np.zeros((0,), np.int64)
    f32 = np.float32
    thr, sig, mins = f32(iou_thr), f32(sigma), f32(min_score)
    box = d[:, :4].copy()
    s = d[:, 4].copy()
    area = ((box[:, 2] - box[:, 0]) * (box[:, 3] - box[:, 1])).astype(f32)
    ind = np.arange(n, dtype=np.int64)
    arrays = (box, s, area, ind)
    i = 0
    with np.errstate(divide='ignore', invalid='ignore', over='ignore'):
        while i < n:
            # selection: first position of the maximum over [i, n); a NaN at i stays, a later NaN never wins
            m = i
            if not np.isnan(s[i]):
                seg = s[i:n]
                ok = ~np.isnan(seg)
                mx = seg[ok].max()
                m = i + int(np.nonzero(ok & (seg == mx))[0][0])
            for a in arrays:
                a[[i, m]] = a[[m, i]]
            if i + 1 >= n:
                i += 1
                continue
            r = slice(i + 1, n)
            bi = box[i]
            xx1 = np.maximum(bi[0], box[r, 0])
            yy1 = np.maximum(bi[1], box[r, 1])
            xx2 = np.minimum(bi[2], box[r, 2])
            yy2 = np.minimum(bi[3], box[r, 3])
            w = np.maximum(f32(0), xx2 - xx1)
            h = np.maximum(f32(0), yy2 - yy1)
            inter = w * h
            ovr = inter / (area[i] + area[r] - inter)
            if method == 'linear':
                wt = np.where(ovr > thr, f32(1) - ovr, f32(1)).astype(f32)
            else:
                wt = np.exp((-(ovr * ovr) / sig).astype(np.float64)).astype(f32)
            s[r] = wt * s[r]
            gone = s[:n] < mins          # only positions > i are tested (the selected one never is)
            gone[:i + 1] = False
            # the reference's removal loop: at a removed position, the last live element moves in and is tested there again
            pos = i + 1
            holes = list(np.nonzero(gone)[0])
            k = 0
            while k < len(holes) and holes[k] < n:
                pos = holes[k]
                while pos < n and gone[pos]:
                    last = n - 1
                    for a in arrays:
                        a[pos] = a[last]
                    gone[pos] = gone[last]
                    n -= 1
                k += 1
            i += 1
    out = np.concatenate([box[:n], s[:n, None]], 1).astype(np.float32)
    return out, ind[:n]


def multiclass_soft_nms(boxes, scores, score_thr, iou_thr, method='linear', sigma=0.5, min_score=1e-3, class_agnostic=False, max_num=-1):
    """lfd_oracle.multiclass_nms with Soft-NMS: boxes [K,4], scores [K,C] (bg dropped) -> (dets [k,5], labels [k], src [k] = row * C + class)."""
    boxes = np.asarray(boxes, np.float32).reshape(-1, 4)
    scores = np.asarray(scores, np.float32)
    K, C = scores.shape
    b = np.repeat(boxes[:, None, :], C, axis=1).reshape(-1, 4)
    s = scores.reshape(-1)
    lab = np.tile(np.arange(C, dtype=np.int64), K)
    inds = np.nonzero(s > np.float32(score_thr))[0]
    b, s, lab = b[inds], s[inds], lab[inds]
    if inds.size == 0:
        return np.zeros((0, 5), np.float32), np.zeros((0,), np.int64), np.zeros((0,), np.int64)
    return _soft_on_candidates(b, s, lab, inds, iou_thr, method, sigma, min_score, class_agnostic, max_num)


def _soft_on_candidates(b, s, lab, src, iou_thr, method, sigma, min_score, class_agnostic, max_num=-1):
    if class_agnostic:
        bn = b
    else:
        off = lab.astype(np.float32) * (b.max() + np.float32(1))
        bn = (b + off[:, None]).astype(np.float32)
    out, keep = soft_nms(np.concatenate([bn, s[:, None]], 1), iou_thr, method, sigma, min_score)
    if not class_agnostic:
        out[:, :4] = out[:, :4] - off[keep][:, None]
    if max_num > 0:
        out, keep = out[:max_num], keep[:max_num]
    return out.astype(np.float32), lab[keep], src[keep]


def soft_on_candidates(boxes, scores, src, C, iou_thr, method='linear', sigma=0.5, min_score=1e-3, class_agnostic=False):
    """Soft-NMS of one image's candidate list (boxes [k,4], scores [k], src = point * C + class, any order): the candidates are put in the
    reference's order (src ascending) first.  -> (dets, labels, src)."""
    order = np.argsort(np.asarray(src, np.int64), kind='stable')
    src = np.asarray(src, np.int64)[order]
    return _soft_on_candidates(np.asarray(boxes, np.float32)[order], np.asarray(scores, np.float32)[order], src % C, src, iou_thr, method, sigma,
                               min_score, class_agnostic)


def rows_of(dets, labels):
    """[label, score, x, y, w, h] with w = x2 - x1 + 1, as LFD.get_results lists them."""
    return [[int(lab), float(d[4]), float(d[0]), float(d[1]), float(np.float32(d[2] - d[0]) + np.float32(1)),
             float(np.float32(d[3] - d[1]) + np.float32(1))] for d, lab in zip(dets, labels)]


def get_results(cfg, cls, reg, sizes, meta_batch, score_thr, iou_thr, method='linear', sigma=0.5, min_score=1e-3, class_agnostic=False):
    """lfd_oracle.get_results with nms_cfg type 'soft_nms': per image rows [label, score, x, y, w, h] and the kept source indices."""
    results, srcs = [], []
    for i in range(cls.shape[0]):
        m = meta_batch[i]
        sc, bx = orc.decode_image(cfg, cls[i], reg[i], sizes, m['resized_height'], m['resized_width'], m['resize_scale'])
        dets, labels, src = multiclass_soft_nms(bx.numpy(), sc.numpy(), score_thr, iou_thr, method, sigma, min_score, class_agnostic)
        results.append(rows_of(dets, labels))
        srcs.append(src)
    return results, srcs
