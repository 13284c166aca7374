# -*- coding: utf-8 -*-
"""NV12 -> BGR as cv2.cvtColor(f, cv2.COLOR_YUV2BGR_NV12) computes it (BT.601 limited range, 20-bit fixed point), in numpy, for a batch
of frames: the definition of LFD_INPUT_U8_NV12 (include/lfd_b200.h).  Also the inverse direction for the tests' frames."""
import numpy as np


def nv12_oracle(frames):
    """frames: uint8 [N, 3h/2, w] or [3h/2, w] (Y plane of h rows, then the interleaved UV plane of h/2 rows, U at even bytes) ->
    uint8 BGR [N, h, w, 3] or [h, w, 3]."""
    f = np.asarray(frames)
    single = f.ndim == 2
    if single:
        f = f[None]
    n, rows, w = f.shape
    assert f.dtype == np.uint8 and rows % 3 == 0 and w % 2 == 0, (f.dtype, f.shape)
    h = rows // 3 * 2
    Y = f[:, :h].astype(np.int64)
    uv = f[:, h:].reshape(n, h // 2, w // 2, 2).astype(np.int64)
    U = np.repeat(np.repeat(uv[..., 0], 2, axis=1), 2, axis=2) - 128
    V = np.repeat(np.repeat(uv[..., 1], 2, axis=1), 2, axis=2) - 128
    y = np.maximum(Y - 16, 0) * 1220542 + (1 << 19)
    b = (y + 2116026 * U) >> 20
    g = (y - 852492 * V - 409993 * U) >> 20
    r = (y + 1673527 * V) >> 20
    out = np.clip(np.stack([b, g, r], axis=-1), 0, 255).astype(np.uint8)
    return out[0] if single else out


def nv12_frames(n, h, w, seed=0):
    """uint8 NV12 [n, 3h/2, w] frames that reach every clamp of the conversion: Y in {0, 15, 16, 235, 255} and U, V in {0, 128, 255} on
    the borders (rows and columns 0, 1, h-2, h-1 / w-2, w-1) and in runs through the interior, the rest random."""
    assert h % 2 == 0 and w % 2 == 0
    rng = np.random.default_rng(seed + 7919 * h + w)
    ys = np.array([0, 15, 16, 235, 255], np.uint8)
    cs = np.array([0, 128, 255], np.uint8)
    Y = rng.integers(0, 256, (n, h, w), dtype=np.uint8)
    UV = rng.integers(0, 256, (n, h // 2, w), dtype=np.uint8)
    # borders
    for r in (0, 1, h - 2, h - 1):
        Y[:, r] = ys[(np.arange(w) + r) % 5]
    for c in (0, 1, w - 2, w - 1):
        Y[:, :, c] = ys[(np.arange(h) + c) % 5]
    for r in (0, h // 2 - 1):
        UV[:, r] = cs[(np.arange(w) // 2 * 5 + np.arange(w) % 2 + r) % 3]
    for c in (0, 1, w - 2, w - 1):
        UV[:, :, c] = cs[(np.arange(h // 2) + c) % 3]
    # interior: a band of rows and one of columns with every (Y, U, V) combination in turn
    if h > 8 and w > 8:
        r0, c0 = h // 3 // 2 * 2, w // 3 // 2 * 2
        Y[:, r0:r0 + 2] = ys[np.arange(w) % 5]
        UV[:, r0 // 2] = cs[(np.arange(w) // 2 * 3 + np.arange(w) % 2 + np.arange(w) // 10) % 3]
        Y[:, :, c0:c0 + 2] = ys[(np.arange(h) // 2 % 5)][:, None]
        UV[:, :, c0] = cs[np.arange(h // 2) % 3]
        UV[:, :, c0 + 1] = cs[(np.arange(h // 2) // 3) % 3]
    return np.ascontiguousarray(np.concatenate([Y, UV], axis=1))


def all_triples_frame():
    """One NV12 frame holding every (Y, U, V) triple: 2^24 pixels, 4096 x 4096, each 2x2 block one (U, V) pair and four Y values."""
    n_uv = 1 << 16                                      # (U, V) pairs, one per 2x2 block: 128 x 512 blocks per Y group of 4
    uv = np.arange(n_uv)
    U, V = (uv >> 8).astype(np.uint8), (uv & 255).astype(np.uint8)
    # 64 copies of the block grid, each carrying 4 of the 256 Y values in its 2x2 blocks: blocks [64][256][256] -> 2048 x 2048 blocks
    h, w = 4096, 4096
    by, bx = np.meshgrid(np.arange(h // 2), np.arange(w // 2), indexing='ij')
    copy = (by // 256) * 8 + bx // 256                  # 0..63
    pair = (by % 256) * 256 + bx % 256                  # 0..65535
    Y = np.empty((h, w), np.uint8)
    for dy in range(2):
        for dx in range(2):
            Y[dy::2, dx::2] = (copy * 4 + dy * 2 + dx).astype(np.uint8)
    UVp = np.empty((h // 2, w), np.uint8)
    UVp[:, 0::2] = U[pair]
    UVp[:, 1::2] = V[pair]
    return np.ascontiguousarray(np.concatenate([Y, UVp], axis=0))
