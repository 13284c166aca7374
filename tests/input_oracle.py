# -*- coding: utf-8 -*-
"""numpy restatement of the training input kernel (csrc/input.cu): the bit-exact reference the GPU tests compare it against.

One image goes through  R = cv2.resize(S, (0, 0), fx=s, fy=s)  (uint8, INTER_LINEAR),  crop_from_image(R, (cx, cy, W, H))
(zero outside R), an optional horizontal flip, 1 -> 3 channel replication, an optional BGR -> RGB swap and, in the fp32 mode,
albumentations' Normalize.  R is never materialised: each output pixel is computed from its source neighbourhood.

cv2's arithmetic, restated:
  - dw = round-half-even(w * s), dh = round-half-even(h * s); equal sizes are a copy.
  - 1/s == 2 exactly: INTER_AREA over 2x2 blocks, (sum + 2) >> 2; blocks cut by an odd edge: round-half-even(sum / count).
  - otherwise: f = float32((d + 0.5) / s - 0.5), i = floor(f), a = f - i; columns clamp (i, a) at both borders, rows clamp the
    two row indices only; weights round((1 - a) * 2048), round(a * 2048); horizontal pass an integer sum, vertical pass
    ((h0 >> 4) * b0 >> 16) + ((h1 >> 4) * b1 >> 16) + 2 >> 2, saturated to uint8.
"""
import numpy

OUT_U8_NHWC, OUT_F32_NCHW = 0, 1
MODE_COPY, MODE_LINEAR, MODE_AREA2 = 0, 1, 2


def resize_plan(h, w, s):
    """(mode, dh, dw) of cv2.resize(fx=fy=s) on an h x w image."""
    dw, dh = int(round(w * s)), int(round(h * s))
    if dw <= 0 or dh <= 0:
        raise ValueError('resize scale %r makes a %dx%d image empty' % (s, h, w))
    if dw == w and dh == h:
        return MODE_COPY, dh, dw
    inv = 1.0 / s
    if abs(inv - round(inv)) < numpy.finfo(numpy.float64).eps and round(inv) == 2:
        return MODE_AREA2, dh, dw
    return MODE_LINEAR, dh, dw


def _taps(d, inv, n, clamp_weights):
    f = ((d.astype(numpy.float64) + 0.5) * inv - 0.5).astype(numpy.float32)
    i = numpy.floor(f).astype(numpy.int64)
    a = (f - i.astype(numpy.float32)).astype(numpy.float32)
    if clamp_weights:
        low, high = i < 0, i >= n - 1
        a[low | high] = 0
        i[low] = 0
        i[high] = n - 1
    w0 = numpy.rint((numpy.float32(1) - a) * numpy.float32(2048)).astype(numpy.int64)
    w1 = numpy.rint(a * numpy.float32(2048)).astype(numpy.int64)
    return numpy.clip(i, 0, n - 1), numpy.clip(i + 1, 0, n - 1), w0, w1


def resized(img, s, rows, cols):
    """R[rows][:, cols] of R = cv2.resize(img, (0, 0), fx=s, fy=s); rows / cols are valid resized indices.  -> uint8 [len(rows), len(cols), C]"""
    img = img if img.ndim == 3 else img[:, :, None]
    h, w = img.shape[:2]
    mode, dh, dw = resize_plan(h, w, s)
    rows, cols = numpy.asarray(rows, numpy.int64), numpy.asarray(cols, numpy.int64)
    S = img.astype(numpy.int64)
    if mode == MODE_COPY:
        return img[rows][:, cols]
    if mode == MODE_AREA2:
        y0, x0 = 2 * rows, 2 * cols
        y1v, x1v = (y0 + 1 < h), (x0 + 1 < w)
        y1, x1 = numpy.minimum(y0 + 1, h - 1), numpy.minimum(x0 + 1, w - 1)
        a, b = S[y0][:, x0], S[y0][:, x1] * x1v[None, :, None]
        c, d = S[y1][:, x0] * y1v[:, None, None], S[y1][:, x1] * (y1v[:, None] & x1v[None, :])[:, :, None]
        total = a + b + c + d
        count = (1 + x1v[None, :].astype(numpy.int64)) * (1 + y1v[:, None].astype(numpy.int64))
        full = (total + 2) >> 2
        edge = numpy.rint(total.astype(numpy.float32) / count[:, :, None].astype(numpy.float32)).astype(numpy.int64)
        return numpy.where((count == 4)[:, :, None], full, edge).astype(numpy.uint8)
    inv = 1.0 / s
    sx0, sx1, a0, a1 = _taps(cols, inv, w, True)
    sy0, sy1, b0, b1 = _taps(rows, inv, h, False)
    h0 = S[sy0][:, sx0] * a0[None, :, None] + S[sy0][:, sx1] * a1[None, :, None]
    h1 = S[sy1][:, sx0] * a0[None, :, None] + S[sy1][:, sx1] * a1[None, :, None]
    v = (((h0 >> 4) * b0[:, None, None]) >> 16) + (((h1 >> 4) * b1[:, None, None]) >> 16) + 2 >> 2
    return numpy.clip(v, 0, 255).astype(numpy.uint8)


def render(img, s, crop_x, crop_y, out_h, out_w, flip):
    """crop_from_image(cv2.resize(img, fx=fy=s), (crop_x, crop_y, out_w, out_h)), flipped left-right if `flip`, as 3 channels.
    -> uint8 [out_h, out_w, 3] in the source's channel order (a gray source is replicated)."""
    h, w = img.shape[:2]
    _, dh, dw = resize_plan(h, w, s)
    out = numpy.zeros((out_h, out_w, img.shape[2] if img.ndim == 3 else 1), numpy.uint8)
    y0, y1 = max(0, -crop_y), min(out_h, dh - crop_y)
    x0, x1 = max(0, -crop_x), min(out_w, dw - crop_x)
    if y1 > y0 and x1 > x0:
        out[y0:y1, x0:x1] = resized(img, s, numpy.arange(y0, y1) + crop_y, numpy.arange(x0, x1) + crop_x)
    if flip:
        out = out[:, ::-1]
    if out.shape[2] == 1:
        out = numpy.repeat(out, 3, axis=2)
    return numpy.ascontiguousarray(out)


def normalize_constants(mean, std, max_pixel_value):
    """albumentations.normalize: (img - mean * max_pixel) * reciprocal(std * max_pixel), all in float32."""
    m = numpy.array(mean, numpy.float32) * numpy.float32(max_pixel_value)
    d = numpy.reciprocal(numpy.array(std, numpy.float32) * numpy.float32(max_pixel_value), dtype=numpy.float32)
    return m, d


def build_batch(items, out_mode, swap_rb=False, H=None, W=None, mean=None, scale=None):
    """items: (img, s, crop_x, crop_y, out_h, out_w, flip) per image.
    OUT_U8_NHWC -> uint8 [N, H, W, 3] (every image H x W); OUT_F32_NCHW -> float32 [N, 3, H, W], each image normalised with
    (v - mean[c]) * scale[c] and zero-padded at the bottom-right."""
    crops = [render(*it) for it in items]
    if swap_rb:
        crops = [c[:, :, ::-1] for c in crops]
    H = max(c.shape[0] for c in crops) if H is None else H
    W = max(c.shape[1] for c in crops) if W is None else W
    if out_mode == OUT_U8_NHWC:
        return numpy.stack(crops)
    mean, scale = numpy.asarray(mean, numpy.float32), numpy.asarray(scale, numpy.float32)
    out = numpy.zeros((len(crops), 3, H, W), numpy.float32)
    for i, c in enumerate(crops):
        out[i, :, :c.shape[0], :c.shape[1]] = ((c.astype(numpy.float32) - mean) * scale).transpose(2, 0, 1)
    return out
