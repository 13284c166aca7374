# -*- coding: utf-8 -*-
"""Packed camera frames -> BGR as cv2.cvtColor computes it, in numpy, for a batch of frames: the definition of LFD_INPUT_U8_YUY2 / _UYVY
(COLOR_YUV2BGR_YUY2 / _UYVY: BT.601 limited range in 20-bit fixed point, the constants of NV12) and LFD_INPUT_U8_BGRA / _RGBA
(COLOR_BGRA2BGR / _RGBA2BGR) of include/lfd_b200.h.  Also test frames that reach every clamp of the conversion."""
import numpy as np

FORMATS = ('yuy2', 'uyvy', 'bgra', 'rgba')
BYTES = {'yuy2': 2, 'uyvy': 2, 'bgra': 4, 'rgba': 4}


def yuv_to_bgr(Y, U, V):
    """uint8-valued (Y, U, V) arrays -> uint8 [..., 3] (B, G, R)."""
    Y, u, v = np.asarray(Y, np.int64), np.asarray(U, np.int64) - 128, np.asarray(V, np.int64) - 128
    y = np.maximum(Y - 16, 0) * 1220542 + (1 << 19)
    b = (y + 2116026 * u) >> 20
    g = (y - 852492 * v - 409993 * u) >> 20
    r = (y + 1673527 * v) >> 20
    return np.clip(np.stack([b, g, r], axis=-1), 0, 255).astype(np.uint8)


def yuv422_planes(frames, fmt):
    """4:2:2 frames uint8 [..., h, w, 2] -> (Y, U, V) [..., h, w], U and V those of each pixel's pair x & ~1."""
    f = np.asarray(frames)
    assert f.dtype == np.uint8 and f.shape[-1] == 2 and f.shape[-2] % 2 == 0, (f.dtype, f.shape)
    pairs = f.reshape(f.shape[:-2] + (f.shape[-2] // 2, 4))
    y0, u, y1, v = (pairs[..., k] for k in ((0, 1, 2, 3) if fmt == 'yuy2' else (1, 0, 3, 2)))
    Y = np.stack([y0, y1], axis=-1).reshape(f.shape[:-1])
    return Y, np.repeat(u, 2, axis=-1), np.repeat(v, 2, axis=-1)


def packed_oracle(frames, fmt):
    """frames: uint8 [..., h, w, 2] ('yuy2' / 'uyvy') or [..., h, w, 4] ('bgra' / 'rgba') -> uint8 BGR [..., h, w, 3]."""
    f = np.asarray(frames)
    if fmt in ('bgra', 'rgba'):
        assert f.dtype == np.uint8 and f.shape[-1] == 4, (f.dtype, f.shape)
        return np.ascontiguousarray(f[..., :3] if fmt == 'bgra' else f[..., 2::-1])
    return yuv_to_bgr(*yuv422_planes(f, fmt))


def packed_gray(frames, fmt):
    """The gray frames of 4:2:2 frames: their Y bytes (cv2.COLOR_YUV2GRAY_YUY2 / _UYVY), uint8 [..., h, w]."""
    return np.ascontiguousarray(yuv422_planes(frames, fmt)[0])


def packed_frames(n, h, w, fmt, seed=0):
    """uint8 [n, h, w, 2 or 4] frames.  4:2:2: Y in {0, 15, 16, 235, 255} and U, V in {0, 128, 255} on the borders (rows 0, 1, h-2, h-1,
    columns 0..3 and w-4..w-1) and in a band of rows and one of columns through the interior, the rest random.  4-byte: random, the
    alpha bytes included (the tests fill them with other patterns too)."""
    rng = np.random.default_rng(seed + 7919 * h + w + 104729 * FORMATS.index(fmt))
    if fmt in ('bgra', 'rgba'):
        return rng.integers(0, 256, (n, h, w, 4), dtype=np.uint8)
    assert w % 2 == 0
    ys = np.array([0, 15, 16, 235, 255], np.uint8)
    cs = np.array([0, 128, 255], np.uint8)
    Y = rng.integers(0, 256, (n, h, w), dtype=np.uint8)
    U = rng.integers(0, 256, (n, h, w // 2), dtype=np.uint8)
    V = rng.integers(0, 256, (n, h, w // 2), dtype=np.uint8)
    x, p = np.arange(w), np.arange(w // 2)
    rows = sorted({0, 1, h - 2, h - 1, h // 3}) if h > 4 else range(h)
    for r in rows:
        Y[:, r] = ys[(x + r) % 5]
        U[:, r] = cs[(p + r) % 3]
        V[:, r] = cs[(p // 3 + r) % 3]
    cols = sorted({0, 1, w // 2 - 2, w // 2 - 1, w // 6}) if w > 8 else range(w // 2)
    for c in cols:
        for dx in (0, 1):
            Y[:, :, 2 * c + dx] = ys[(np.arange(h) + c + dx) % 5]
        U[:, :, c] = cs[(np.arange(h) + c) % 3]
        V[:, :, c] = cs[(np.arange(h) // 3 + c) % 3]
    return to_packed(Y, U, V, fmt)


def to_packed(Y, U, V, fmt):
    """Y [..., h, w] and the pairs' U, V [..., h, w/2] -> 4:2:2 frames uint8 [..., h, w, 2] in byte order fmt."""
    y0, y1 = Y[..., 0::2], Y[..., 1::2]
    order = (y0, U, y1, V) if fmt == 'yuy2' else (U, y0, V, y1)
    pairs = np.stack(order, axis=-1)
    return np.ascontiguousarray(pairs.reshape(Y.shape + (2,)))


def all_triples_frame(fmt):
    """One 4:2:2 frame, uint8 [4096, 8192, 2], holding every (Y, U, V) triple at both pixels of a pair: pair k = (t << 16) | (U << 8) | V
    has Y0 = t and Y1 = (t + 85) & 255."""
    k = np.arange(1 << 24, dtype=np.int64)
    t = k >> 16
    Y = np.stack([t, (t + 85) & 255], axis=-1).reshape(4096, 8192).astype(np.uint8)
    U = ((k >> 8) & 255).reshape(4096, 4096).astype(np.uint8)
    V = (k & 255).reshape(4096, 4096).astype(np.uint8)
    return to_packed(Y, U, V, fmt)
