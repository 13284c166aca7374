# -*- coding: utf-8 -*-
"""NV12 input, host side: the numpy oracle against cv2, the shape and format checks of the host entry points, the capacity staging
layout of a smaller frame and the StreamingDetector arguments -- everything that runs without a device."""
import os
import re

import numpy as np
import pytest
import torch

from lfd import _native as nat
from lfd._engine import check_nv12_frame, stage_nv12
from nv12_oracle import all_triples_frame, nv12_frames, nv12_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_oracle_equals_cv2_on_every_yuv_triple():
    cv2 = pytest.importorskip('cv2')
    f = all_triples_frame()
    Y = f[:4096].astype(np.int64)
    uv = f[4096:].reshape(2048, 2048, 2).astype(np.int64)
    U = np.repeat(np.repeat(uv[..., 0], 2, 0), 2, 1)
    V = np.repeat(np.repeat(uv[..., 1], 2, 0), 2, 1)
    assert np.unique((Y << 16) | (U << 8) | V).size == 1 << 24          # every (Y, U, V) triple is a pixel of the frame
    assert np.array_equal(nv12_oracle(f), cv2.cvtColor(f, cv2.COLOR_YUV2BGR_NV12))


@pytest.mark.parametrize('h,w', [(2, 2), (4, 6), (38, 42), (40, 44), (400, 656), (720, 1280), (1080, 1920)])
def test_oracle_equals_cv2_on_frames(h, w):
    cv2 = pytest.importorskip('cv2')
    x = nv12_frames(2, h, w, seed=h)
    got = nv12_oracle(x)
    assert got.shape == (2, h, w, 3)
    for i in range(2):
        assert np.array_equal(got[i], cv2.cvtColor(x[i], cv2.COLOR_YUV2BGR_NV12)), (h, w, i)
    assert np.array_equal(nv12_oracle(x[0]), got[0])


def test_test_frames_reach_every_clamp():
    x = nv12_frames(1, 38, 42)
    Y, UV = x[0, :38], x[0, 38:]
    for v in (0, 15, 16, 235, 255):
        assert (Y[0] == v).any() and (Y[:, 0] == v).any() and (Y[12] == v).any(), v     # borders and the interior band
    for v in (0, 128, 255):
        assert (UV[0] == v).any() and (UV[:, 0] == v).any(), v
    bgr = nv12_oracle(x)
    assert (bgr == 0).any() and (bgr == 255).any()


def test_abi_constant():
    assert nat.INPUT_U8_NV12 == 2
    header = open(os.path.join(ROOT, 'include', 'lfd_b200.h')).read()
    assert re.search(r'LFD_INPUT_F32_NCHW = 0, LFD_INPUT_U8_NHWC = 1, LFD_INPUT_U8_NV12 = 2', header)


def _nv12(n, h, w, **kw):
    return torch.zeros((n, h * 3 // 2, w), dtype=torch.uint8, **kw)


@pytest.mark.parametrize('shape,what', [
    ((2, 97 * 3 // 2, 160), 'even'),            # 145 rows: not 3h/2 of an even h
    ((2, 144, 161), 'even'),                    # odd w
    ((2, 144, 160, 3), 'uint8 [N, 3h/2, w]'),   # a 4-D (BGR-shaped) tensor passed as NV12
    ((3, 144, 160), 'N=2'),                     # wrong N
    ((1, 144, 160), 'N=2'),
    ((2, 150, 160), 'capacity'),                # h = 100 > 96
    ((2, 144, 162), 'capacity'),                # w > 160
    ((2, 0, 160), 'capacity'),
])
def test_nv12_frame_checks(shape, what):
    x = torch.zeros(shape, dtype=torch.uint8)
    with pytest.raises(ValueError) as e:
        check_nv12_frame(x, 2, 96, 160)
    assert what in str(e.value), str(e.value)


def test_nv12_frame_checks_dtype_device_and_capacity():
    with pytest.raises(ValueError, match='uint8'):
        check_nv12_frame(torch.zeros((2, 144, 160), dtype=torch.float32), 2, 96, 160)
    with pytest.raises(ValueError, match='even height and width, this plan'):
        check_nv12_frame(_nv12(2, 96, 160), 2, 97, 160)
    with pytest.raises(ValueError, match='even height and width, this plan'):
        check_nv12_frame(_nv12(2, 96, 160), 2, 96, 161)
    with pytest.raises(ValueError, match='CUDA'):               # every shape check passes: the device is what is missing here
        check_nv12_frame(_nv12(2, 64, 100), 2, 96, 160)


def test_staging_layout_of_a_smaller_frame():
    N, H, W, h, w = 2, 12, 16, 6, 10
    x = torch.from_numpy(nv12_frames(N, h, w, seed=3))
    stage = torch.full((N, H * 3 // 2, W), 0xAA, dtype=torch.uint8)
    stage_nv12(stage, x, h, w)
    s, xs = stage.numpy(), x.numpy()
    for n in range(N):
        for r in range(H * 3 // 2):
            for c in range(W):
                if r < h and c < w:                                     # Y plane: rows 0..h-1 of the frame
                    want = xs[n, r, c]
                elif H <= r < H + h // 2 and c < w:                     # UV plane at row H: the frame's UV rows h..3h/2-1
                    want = xs[n, h + r - H, c]
                else:
                    want = 0xAA
                assert s[n, r, c] == want, (n, r, c)
    # the staged frame converts like the frame itself in its corner
    full = nv12_oracle(s)
    assert np.array_equal(full[:, :h, :w], nv12_oracle(xs))


def test_streaming_detector_arguments():
    from lfd.pipeline import StreamingDetector
    with pytest.raises(ValueError, match="'bgr' or 'nv12'"):
        StreamingDetector(None, 2, 96, 160, 0.3, 0.3, frame_format='i420')
    for h, w in ((97, 160), (96, 161)):
        with pytest.raises(ValueError, match='even height and width'):
            StreamingDetector(None, 2, h, w, 0.3, 0.3, frame_format='nv12')
