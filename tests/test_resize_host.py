# -*- coding: utf-8 -*-
"""CPU tests of resized inference input (lfd_resize_query / lfd_resize_frames / lfd_engine_detect_resized, include/lfd_b200.h): the
library's size and interpolation rule is region_sampler.resize_plan's and gives the shapes cv2.resize gives; the per-tap arithmetic the
kernel runs (input_oracle restates input.cu) is cv2's down to the deployment scales; every refusal decided before a CUDA call returns its
code without a device."""
import ctypes as C

import cv2
import numpy as np
import pytest
import torch

import input_oracle
from lfd import _native as nat
from lfd._engine import check_source
from lfd.data_pipeline.sampler.region_sampler import resize_plan
from nv12_oracle import nv12_frames, nv12_oracle

LFD_ERR_INVALID, LFD_ERR_CUDA, LFD_ERR_UNSUPPORTED, LFD_ERR_CAPACITY = 1, 2, 3, 4

SIZES = [(1080, 1920), (2160, 3840), (720, 1280), (37, 53), (31, 30), (481, 641), (7, 5), (1, 1), (482, 642), (99, 101), (2, 3)]
# exactly 0.5 (AREA) and 1 (COPY), the deployment scales 1/3 and 1/6, 0.6667, 1.5, upscaling, and scales whose h * s lands on .5
SCALES = [0.5, 1.0, 1 / 3, 1 / 6, 0.6667, 1.5, 2.0, 2 / 3, 0.25, 0.125, 0.1, 0.3, 720 / 1080, 640 / 3840, 1 / 2.5, 0.75, 3.0,
          1 / 1.5, 0.49999999999999994, 0.5000000000000001]


def _half_scales(h):
    """Scales that put h * s exactly on k + 0.5 (round-half-even decides)."""
    return [(k + 0.5) / h for k in range(max(0, h // 3 - 1), h // 3 + 2)]


@pytest.mark.parametrize('h,w', SIZES)
def test_rule_is_resize_plan_and_cv2_shapes(h, w):
    scales = SCALES + _half_scales(h) + _half_scales(w)
    img = np.zeros((h, w), np.uint8)
    for s in scales:
        try:
            want = resize_plan(h, w, s)
        except ValueError:
            with pytest.raises(nat.LfdError, match='empty'):
                nat.resize_query(h, w, s)
            continue
        got = nat.resize_query(h, w, s)
        assert got == want, (h, w, s, got, want)
        assert cv2.resize(img, (0, 0), fx=s, fy=s).shape == (got[1], got[2]), (h, w, s)


def test_rule_modes():
    assert nat.resize_query(1080, 1920, 1.0) == (nat.RESIZE_COPY, 1080, 1920)
    assert nat.resize_query(1080, 1920, 0.5) == (nat.RESIZE_AREA2, 540, 960)
    assert nat.resize_query(1081, 1921, 0.5) == (nat.RESIZE_AREA2, 540, 960)         # 540.5 and 960.5: half to even
    assert nat.resize_query(2160, 3840, 1 / 6) == (nat.RESIZE_LINEAR, 360, 640)
    assert nat.resize_query(1080, 1920, 2 / 3) == (nat.RESIZE_LINEAR, 720, 1280)
    assert nat.resize_query(4, 4, 1.1) == (nat.RESIZE_COPY, 4, 4)                     # 4.4 rounds back to the source size
    assert nat.resize_query(5, 7, 0.5) == (nat.RESIZE_AREA2, 2, 4)                    # 2.5 -> 2, 3.5 -> 4


@pytest.mark.parametrize('s', [0.0, -0.5, float('nan'), float('inf'), -float('inf'), 1e-9])
def test_rule_refuses(s):
    with pytest.raises(nat.LfdError):
        nat.resize_query(1080, 1920, s)
    for h, w in ((0, 10), (10, 0), (-1, 4)):
        with pytest.raises(nat.LfdError):
            nat.resize_query(h, w, 0.5)


def test_rule_of_a_huge_result_exceeds_every_capacity():
    assert nat.resize_query(1000, 1000, 1e12)[1:] == (2 ** 31 - 1, 2 ** 31 - 1)


# The arithmetic the kernel runs, against cv2, where the tests on the device cannot afford 4K frames of every kind
@pytest.mark.parametrize('h,w,c', [(2160, 3840, 3), (1080, 1920, 3), (721, 1283, 1), (37, 53, 3), (33, 31, 1)])
def test_tap_arithmetic_is_cv2_down_to_deployment_scales(h, w, c):
    rng = np.random.default_rng(h * w + c)
    img = rng.integers(0, 256, (h, w, c) if c == 3 else (h, w), dtype=np.uint8)
    for s in (1 / 6, 1 / 3, 0.125, 0.1, 640 / 3840, 2 / 3, 0.6667, 0.5, 1.0, 1.5, 2.0):
        _, dh, dw = nat.resize_query(h, w, s)
        got = input_oracle.resized(img, s, np.arange(dh), np.arange(dw))
        want = cv2.resize(img, (0, 0), fx=s, fy=s).reshape(got.shape)
        assert np.array_equal(got, want), (h, w, c, s, int((got != want).sum()))


def test_nv12_tap_arithmetic_is_cv2_of_the_converted_frame():
    f = nv12_frames(1, 1080, 1920, seed=5)[0]
    bgr = nv12_oracle(f)
    assert np.array_equal(bgr, cv2.cvtColor(f, cv2.COLOR_YUV2BGR_NV12))
    for s in (1 / 6, 2 / 3, 0.5, 1.5):
        _, dh, dw = nat.resize_query(1080, 1920, s)
        got = input_oracle.resized(bgr, s, np.arange(dh), np.arange(dw))
        assert np.array_equal(got, cv2.resize(cv2.cvtColor(f, cv2.COLOR_YUV2BGR_NV12), (0, 0), fx=s, fy=s)), s


def _resize(src=1, fmt=nat.INPUT_U8_NHWC, ch=3, n=2, h=64, w=96, s=0.5, dst=1, H=32, W=48):
    lib = nat.lib()
    rc = lib.lfd_resize_frames(C.c_void_p(src), fmt, ch, n, h, w, s, C.c_void_p(dst), H, W, None)
    return rc, lib.lfd_last_error().decode()


@pytest.mark.parametrize('kw,code,what', [
    (dict(s=0.0), LFD_ERR_INVALID, 'scale'),
    (dict(s=-0.5), LFD_ERR_INVALID, 'scale'),
    (dict(s=float('nan')), LFD_ERR_INVALID, 'scale'),
    (dict(s=float('inf')), LFD_ERR_INVALID, 'scale'),
    (dict(s=1e-6), LFD_ERR_INVALID, 'empty'),
    (dict(src=0), LFD_ERR_INVALID, 'null'),
    (dict(dst=0), LFD_ERR_INVALID, 'null'),
    (dict(fmt=nat.INPUT_U8_NV12, h=63), LFD_ERR_INVALID, 'even'),
    (dict(fmt=nat.INPUT_U8_NV12, w=95), LFD_ERR_INVALID, 'even'),
    (dict(fmt=3), LFD_ERR_INVALID, 'format'),
    (dict(fmt=-1), LFD_ERR_INVALID, 'format'),
    (dict(ch=2), LFD_ERR_INVALID, 'channels'),
    (dict(n=0), LFD_ERR_INVALID, 'n=0'),
    (dict(h=0), LFD_ERR_INVALID, '0x96'),
    (dict(s=0.6), LFD_ERR_CAPACITY, 'beyond'),
    (dict(H=31), LFD_ERR_CAPACITY, 'beyond'),
    (dict(W=47), LFD_ERR_CAPACITY, 'beyond'),
    (dict(s=1e12), LFD_ERR_CAPACITY, 'beyond'),
    (dict(fmt=nat.INPUT_F32_NCHW), LFD_ERR_UNSUPPORTED, 'float32'),
    (dict(w=20000, s=0.5, W=10000), LFD_ERR_UNSUPPORTED, '6144'),
    (dict(n=70000), LFD_ERR_UNSUPPORTED, '65535'),
])
def test_resize_frames_refusals_before_any_cuda_call(kw, code, what):
    rc, msg = _resize(**kw)
    assert rc == code and what in msg, (rc, msg)


def test_a_valid_call_reaches_the_device_check():
    if torch.cuda.is_available():
        pytest.skip('checks the no-GPU failure mode')
    for kw in (dict(), dict(fmt=nat.INPUT_U8_NV12), dict(ch=1), dict(fmt=nat.INPUT_U8_NV12, ch=1), dict(s=0.3), dict(h=32, w=48, s=1.0)):
        rc, msg = _resize(**kw)
        assert rc == LFD_ERR_CUDA and 'no CUDA device' in msg, (kw, rc, msg)


def test_engine_detect_resized_refuses_a_null_engine():
    lib = nat.lib()
    one = C.c_void_p(256)
    rc = lib.lfd_engine_detect_resized(None, one, nat.INPUT_U8_NHWC, 64, 96, 0.5, one, one, one, one, None, None, 1, None)
    assert rc == LFD_ERR_INVALID and 'null' in lib.lfd_last_error().decode()


def test_source_checks():
    with pytest.raises(ValueError, match='uint8'):
        check_source(torch.zeros((2, 3, 8, 8)), 2, 3, False)                 # float32 frames are not resized
    with pytest.raises(ValueError, match=r'uint8 \[N, h, w\]'):
        check_source(torch.zeros((2, 8, 8, 3), dtype=torch.uint8), 2, 1, False)   # BGR frames on a gray model
    with pytest.raises(ValueError, match='N=2'):
        check_source(torch.zeros((3, 8, 8, 3), dtype=torch.uint8), 2, 3, False)
    with pytest.raises(ValueError, match='even'):
        check_source(torch.zeros((2, 12, 9), dtype=torch.uint8), 2, 3, True)
    with pytest.raises(ValueError, match='CUDA'):
        check_source(torch.zeros((2, 8, 8, 3), dtype=torch.uint8), 2, 3, False)   # a host tensor


def test_new_entry_points_keep_the_abi():
    assert nat.lib().lfd_abi_version() == 5 and nat.ABI_VERSION == 5
    for name in ('lfd_resize_query', 'lfd_resize_frames', 'lfd_engine_detect_resized'):
        assert name in nat.SYMBOLS and hasattr(nat.lib(), name)
