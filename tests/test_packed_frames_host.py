# -*- coding: utf-8 -*-
"""Packed camera frames (YUY2 / UYVY / BGRA / RGBA), host side: the numpy oracle against cv2, the ABI constants, the shape and format
checks of InferencePlan.forward and StreamingDetector, and the C-ABI refusals that are decided before any CUDA call."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

import input_oracle
from lfd import _native as nat
from lfd._engine import PACKED_FORMATS, check_packed
from packed_oracle import FORMATS, BYTES, all_triples_frame, packed_frames, packed_gray, packed_oracle, yuv_to_bgr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LFD_ERR_INVALID, LFD_ERR_CUDA, LFD_ERR_UNSUPPORTED, LFD_ERR_CAPACITY = 1, 2, 3, 4
CV2_CODES = {'yuy2': ('COLOR_YUV2BGR_YUY2', 'COLOR_YUV2GRAY_YUY2'), 'uyvy': ('COLOR_YUV2BGR_UYVY', 'COLOR_YUV2GRAY_UYVY'),
             'bgra': ('COLOR_BGRA2BGR', None), 'rgba': ('COLOR_RGBA2BGR', None)}


@pytest.mark.parametrize('fmt', ['yuy2', 'uyvy'])
def test_oracle_equals_cv2_on_every_yuv_triple_at_both_pixels_of_a_pair(fmt):
    cv2 = pytest.importorskip('cv2')
    f = all_triples_frame(fmt)
    bgr_code, gray_code = (getattr(cv2, c) for c in CV2_CODES[fmt])
    for r0 in range(0, 4096, 512):                     # 8 bands: the int64 intermediates of the whole frame do not fit comfortably
        band = f[r0:r0 + 512]
        want = cv2.cvtColor(band, bgr_code)
        assert np.array_equal(packed_oracle(band, fmt), want), (fmt, r0)
        assert np.array_equal(packed_gray(band, fmt), cv2.cvtColor(band, gray_code)), (fmt, r0)
    # every (Y, U, V) is a first and a second pixel of some pair
    pairs = f.reshape(-1, 4).astype(np.int64)
    y0, u, y1, v = (pairs[:, k] for k in ((0, 1, 2, 3) if fmt == 'yuy2' else (1, 0, 3, 2)))
    assert np.unique((y0 << 16) | (u << 8) | v).size == 1 << 24 and np.unique((y1 << 16) | (u << 8) | v).size == 1 << 24


@pytest.mark.parametrize('fmt', FORMATS)
@pytest.mark.parametrize('h,w', [(1, 2), (3, 6), (38, 42), (40, 44), (400, 656), (1080, 1920)])
def test_oracle_equals_cv2_on_frames(fmt, h, w):
    cv2 = pytest.importorskip('cv2')
    x = packed_frames(2, h, w, fmt, seed=h)
    got = packed_oracle(x, fmt)
    assert got.shape == (2, h, w, 3)
    bgr_code, gray_code = CV2_CODES[fmt]
    for i in range(2):
        assert np.array_equal(got[i], cv2.cvtColor(x[i], getattr(cv2, bgr_code))), (fmt, h, w, i)
        if gray_code:
            assert np.array_equal(packed_gray(x[i], fmt), cv2.cvtColor(x[i], getattr(cv2, gray_code))), (fmt, h, w, i)


def test_yuv_formula_is_the_nv12_oracles():
    from nv12_oracle import nv12_frames, nv12_oracle
    f = nv12_frames(1, 40, 44)[0]
    Y, uv = f[:40], f[40:].reshape(20, 22, 2)
    U = np.repeat(np.repeat(uv[..., 0], 2, 0), 2, 1)
    V = np.repeat(np.repeat(uv[..., 1], 2, 0), 2, 1)
    assert np.array_equal(yuv_to_bgr(Y, U, V), nv12_oracle(f))


def test_test_frames_reach_every_clamp():
    for fmt in ('yuy2', 'uyvy'):
        x = packed_frames(1, 38, 42, fmt)
        bgr = packed_oracle(x, fmt)
        assert (bgr == 0).any() and (bgr == 255).any()
        Y = packed_gray(x, fmt)
        for v in (0, 15, 16, 235, 255):
            assert (Y[0, 0] == v).any() and (Y[0, :, 0] == v).any(), (fmt, v)
    for fmt in ('bgra', 'rgba'):
        x = packed_frames(1, 38, 42, fmt)
        assert not np.array_equal(packed_oracle(x, 'bgra'), packed_oracle(x, 'rgba'))


def test_tap_arithmetic_is_cv2_of_the_converted_frame():
    """The resize converts each tap before its arithmetic (input.cu packed_pixel): cv2.resize of the converted frame."""
    cv2 = pytest.importorskip('cv2')
    for fmt in FORMATS:
        f = packed_frames(1, 1080, 1920, fmt, seed=5)[0]
        bgr = packed_oracle(f, fmt)
        for s in (1 / 6, 2 / 3, 0.5, 1.5):
            _, dh, dw = nat.resize_query(1080, 1920, s)
            got = input_oracle.resized(bgr, s, np.arange(dh), np.arange(dw))
            assert np.array_equal(got, cv2.resize(bgr, (0, 0), fx=s, fy=s)), (fmt, s)


def test_abi_constants():
    assert (nat.INPUT_U8_YUY2, nat.INPUT_U8_UYVY, nat.INPUT_U8_BGRA, nat.INPUT_U8_RGBA) == (4, 5, 6, 7)
    header = open(os.path.join(ROOT, 'include', 'lfd_b200.h')).read()
    assert re.search(r'LFD_INPUT_U8_YUY2 = 4, LFD_INPUT_U8_UYVY = 5, LFD_INPUT_U8_BGRA = 6,\s+LFD_INPUT_U8_RGBA = 7', header)
    assert {k: v[0] for k, v in PACKED_FORMATS.items()} == {'yuy2': 4, 'uyvy': 5, 'bgra': 6, 'rgba': 7}
    assert nat.lib().lfd_abi_version() == 5 and nat.ABI_VERSION == 5


def _frames(fmt, n=2, h=8, w=12, dtype=torch.uint8):
    return torch.zeros((n, h, w, BYTES[fmt]), dtype=dtype)


@pytest.mark.parametrize('fmt', FORMATS)
def test_packed_frame_checks(fmt):
    b = BYTES[fmt]
    with pytest.raises(ValueError, match=r'uint8 \[N, h, w, %d\]' % b):
        check_packed(_frames(fmt, dtype=torch.float32), fmt, 2, 3)
    with pytest.raises(ValueError, match=r'uint8 \[N, h, w, %d\]' % b):
        check_packed(torch.zeros((2, 8, 12, 6 - b), dtype=torch.uint8), fmt, 2, 3)      # the other packed layout
    with pytest.raises(ValueError, match=r'uint8 \[N, h, w, %d\]' % b):
        check_packed(torch.zeros((2, 8, 12 * b), dtype=torch.uint8), fmt, 2, 3)
    with pytest.raises(ValueError, match='N=2'):
        check_packed(_frames(fmt, n=3), fmt, 2, 3)
    with pytest.raises(ValueError, match='capacity'):
        check_packed(_frames(fmt, h=9), fmt, 2, 3, 8, 12)
    with pytest.raises(ValueError, match='capacity'):
        check_packed(_frames(fmt, w=14), fmt, 2, 3, 8, 12)
    with pytest.raises(ValueError, match='CUDA'):               # every shape check passes: the device is what is missing here
        check_packed(_frames(fmt), fmt, 2, 3, 8, 12)
    with pytest.raises(ValueError, match='CUDA'):               # above the capacity is fine when the frames are resized
        check_packed(_frames(fmt, h=64, w=96), fmt, 2, 3)


def test_odd_widths_and_gray_models():
    for fmt in ('yuy2', 'uyvy'):
        with pytest.raises(ValueError, match='even width, got 8x11'):
            check_packed(_frames(fmt, w=11), fmt, 2, 3)
        with pytest.raises(ValueError, match='even width, this plan'):
            check_packed(_frames(fmt, w=10), fmt, 2, 3, 8, 13)
        with pytest.raises(ValueError, match='CUDA'):           # a gray model reads the Y bytes
            check_packed(_frames(fmt), fmt, 2, 1, 8, 12)
    for fmt in ('bgra', 'rgba'):
        with pytest.raises(ValueError, match="gray model reads 4:2:2 frames"):
            check_packed(_frames(fmt), fmt, 2, 1, 8, 12)
        with pytest.raises(ValueError, match='CUDA'):           # any width
            check_packed(_frames(fmt, w=11), fmt, 2, 3, 8, 13)


def _gray_model():
    from gray_models import gray_pair
    return gray_pair('WIDERFACE_XS')[0]


def test_streaming_detector_arguments():
    from lfd.pipeline import StreamingDetector
    with pytest.raises(ValueError, match="'bgr' or 'nv12'.*'i420'.*'yuy2', 'uyvy', 'bgra', 'rgba'"):
        StreamingDetector(None, 2, 96, 160, 0.3, 0.3, frame_format='i420')
    for fmt in ('yuy2', 'uyvy'):
        with pytest.raises(ValueError, match='4:2:2 frames have an even width, got 96x161'):
            StreamingDetector(None, 2, 96, 161, 0.3, 0.3, frame_format=fmt)
        with pytest.raises(ValueError, match='4:2:2 frames have an even width, got 1080x1919'):
            StreamingDetector(None, 2, 96, 160, 0.3, 0.3, frame_format=fmt, source_size=(1080, 1919))


def test_streaming_detector_gray_model_formats():
    from lfd.pipeline import StreamingDetector
    model = _gray_model()
    for fmt in ('bgra', 'rgba'):
        with pytest.raises(ValueError, match="gray model takes frame_format 'gray', 'nv12', 'yuy2' or 'uyvy'; '%s' frames are colour" % fmt):
            StreamingDetector(model, 2, 96, 160, 0.3, 0.3, frame_format=fmt)
    with pytest.raises(ValueError, match="a gray model takes frame_format 'gray' or 'nv12', got 'bgr'"):   # unchanged
        StreamingDetector(model, 2, 96, 160, 0.3, 0.3, frame_format='bgr')


def test_forward_refuses_unknown_formats_on_a_host_plan():
    """A host-only plan refuses any forward first; the format check itself is covered on the device (tests/test_gpu_packed_frames.py)."""
    from lfd._engine import InferencePlan
    from helpers import model_of
    plan = InferencePlan(model_of('WIDERFACE_XS'), 2, 64, 96, torch.device('cpu'), nat.CONV_UMMA, create_native=False)
    with pytest.raises(nat.LfdError, match='host-side inspection'):
        plan.forward(_frames('yuy2'), frame_format='yuy2')


# ------------------------------------------------------------------------------------------------------------------ C-ABI refusals
def _resize(src=1, fmt=nat.INPUT_U8_YUY2, ch=3, n=2, h=64, w=96, s=0.5, dst=1, H=32, W=48):
    lib = nat.lib()
    rc = lib.lfd_resize_frames(C.c_void_p(src), fmt, ch, n, h, w, s, C.c_void_p(dst), H, W, None)
    return rc, lib.lfd_last_error().decode()


@pytest.mark.parametrize('kw,code,what', [
    (dict(fmt=nat.INPUT_U8_YUY2, w=95), LFD_ERR_INVALID, 'even width'),
    (dict(fmt=nat.INPUT_U8_UYVY, w=95), LFD_ERR_INVALID, 'even width'),
    (dict(fmt=nat.INPUT_U8_BGRA, ch=1), LFD_ERR_UNSUPPORTED, 'colour'),
    (dict(fmt=nat.INPUT_U8_RGBA, ch=1), LFD_ERR_UNSUPPORTED, 'colour'),
    (dict(fmt=3), LFD_ERR_INVALID, 'format'),
    (dict(fmt=8), LFD_ERR_INVALID, 'format'),
    (dict(fmt=-2), LFD_ERR_INVALID, 'format'),
    (dict(fmt=nat.INPUT_U8_BGRA, s=0.6), LFD_ERR_CAPACITY, 'beyond'),
    (dict(fmt=nat.INPUT_U8_UYVY, ch=2), LFD_ERR_INVALID, 'channels'),
])
def test_resize_frames_refusals_before_any_cuda_call(kw, code, what):
    rc, msg = _resize(**kw)
    assert rc == code and what in msg, (rc, msg)


def test_a_valid_packed_resize_reaches_the_device_check():
    if torch.cuda.is_available():
        pytest.skip('checks the no-GPU failure mode')
    for kw in (dict(), dict(ch=1), dict(fmt=nat.INPUT_U8_UYVY), dict(fmt=nat.INPUT_U8_UYVY, ch=1), dict(fmt=nat.INPUT_U8_BGRA),
               dict(fmt=nat.INPUT_U8_RGBA, h=63, w=95, s=0.5)):
        rc, msg = _resize(**kw)
        assert rc == LFD_ERR_CUDA and 'no CUDA device' in msg, (kw, rc, msg)


def test_engine_detect_entry_points_refuse_a_null_engine():
    lib = nat.lib()
    one = C.c_void_p(256)
    for fmt in (nat.INPUT_U8_YUY2, nat.INPUT_U8_RGBA):
        rc = lib.lfd_engine_detect(None, one, fmt, 64, 96, one, one, one, None, None, 1, None)
        assert rc == LFD_ERR_INVALID and 'null' in lib.lfd_last_error().decode()
        rc = lib.lfd_engine_detect_resized(None, one, fmt, 64, 96, 0.5, one, one, one, one, None, None, 1, None)
        assert rc == LFD_ERR_INVALID and 'null' in lib.lfd_last_error().decode()
