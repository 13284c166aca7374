# -*- coding: utf-8 -*-
"""Resized inference input on the H100: lfd_resize_frames writes, byte for byte, what cv2.resize gives (BGR, gray, NV12 -> BGR through
cv2.cvtColor, NV12 -> gray from the Y plane) into the resized extent of a capacity-layout buffer and nothing outside it;
InferencePlan.forward(resize_scale=) and StreamingDetector(source_size=) give the network outputs of the same plan on host-resized frames
bit for bit, and the rows of the reference's get_results with the meta of a resized image; a model file run through
lfd_engine_detect_resized (and examples/lfd_detect --scale) gives what the Python path gives; repeated batches add no CUDA graph; and a
refused call writes nothing."""
import ctypes as C
import os
import subprocess

import cv2
import numpy as np
import pytest
import torch

import synth
from engine_file import Engine, rows
from gray_models import gray_pair
from helpers import misaligned, model_of, same_bits
from lfd import _native as nat
from lfd.deployment import export_model
from lfd.model.lfd import LFD
from lfd.pipeline import StreamingDetector
from nv12_oracle import nv12_frames
from test_input_transform_host import tl_val_pipeline

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROGRAM = os.path.join(ROOT, 'lfd-a-light-and-fast-detector_b200', 'lfd_detect')
LFD_ERR_INVALID, LFD_ERR_UNSUPPORTED, LFD_ERR_CAPACITY = 1, 3, 4
GUARD = 0xa5
KINDS = {'bgr': (nat.INPUT_U8_NHWC, 3), 'gray': (nat.INPUT_U8_NHWC, 1), 'nv12': (nat.INPUT_U8_NV12, 3), 'nv12_gray': (nat.INPUT_U8_NV12, 1)}


def sources(kind, n, h, w, seed=0):
    """n distinct host frames of h x w: uint8 BGR [n,h,w,3], gray [n,h,w] or NV12 [n,3h/2,w]."""
    if kind.startswith('nv12'):
        return nv12_frames(n, h, w, seed)
    rng = np.random.default_rng(seed + 31 * h + w)
    return rng.integers(0, 256, (n, h, w, 3) if kind == 'bgr' else (n, h, w), dtype=np.uint8)


def cv2_resized(kind, frames, s):
    """What the host path gives: cv2.resize(frame, (0, 0), fx=s, fy=s) of every frame (NV12 converted by cv2 first, or its Y plane)."""
    out = []
    for f in frames:
        if kind == 'nv12':
            f = cv2.cvtColor(f, cv2.COLOR_YUV2BGR_NV12)
        elif kind == 'nv12_gray':
            f = f[:f.shape[0] // 3 * 2]
        out.append(cv2.resize(f, (0, 0), fx=s, fy=s))
    return np.ascontiguousarray(np.stack(out))


def resize_frames(x, kind, h, w, s, H, W, dst=None):
    """lfd_resize_frames on the device frames x into a guard-filled uint8 [n,H,W(,3)] -> (return code, dst)."""
    fmt, ch = KINDS[kind]
    n = x.shape[0]
    if dst is None:
        dst = torch.full((n, H, W, 3) if ch == 3 else (n, H, W), GUARD, dtype=torch.uint8, device='cuda')
    rc = nat.lib().lfd_resize_frames(nat.ptr(x), fmt, ch, n, h, w, s, nat.ptr(dst), H, W, nat.stream_ptr())
    torch.cuda.synchronize()
    return rc, dst


SCALES = [1 / 6, 1 / 3, 0.5, 2 / 3, 0.6667, 1.0, 1.5, 2.0]


@pytest.mark.parametrize('kind', list(KINDS))
@pytest.mark.parametrize('h,w', [(1080, 1920), (97, 131), (62, 86)])
def test_frames_are_cv2s(kind, h, w):
    if kind.startswith('nv12'):
        h, w = h + h % 2, w + w % 2                             # (98 x 132: W % 4 != 0 all the same)
    n = 3
    frames = sources(kind, n, h, w, seed=h)
    x = misaligned(torch.from_numpy(frames).cuda())            # any source address: the taps are byte loads
    for s in SCALES + [(h // 3 + 0.5) / h]:                    # and a scale whose h * s lands on .5
        _, dh, dw = nat.resize_query(h, w, s)
        want = cv2_resized(kind, frames, s)
        assert want.shape[1:3] == (dh, dw)
        H, W = dh + 3, dw + 5                                   # guard rows and columns right of and below the extent
        rc, dst = resize_frames(x, kind, h, w, s, H, W)
        assert rc == 0, nat.lib().lfd_last_error()
        got = dst[:, :dh, :dw].cpu().numpy()
        assert np.array_equal(got, want), (kind, h, w, s, int((got != want).sum()))
        assert bool((dst[:, dh:] == GUARD).all()) and bool((dst[:, :, dw:] == GUARD).all()), (kind, h, w, s, 'wrote outside the extent')


@pytest.mark.parametrize('kind', ['bgr', 'nv12', 'nv12_gray'])
def test_4k_frames_at_deployment_scales(kind):
    h, w = 2160, 3840
    frames = sources(kind, 2, h, w, seed=4)
    x = torch.from_numpy(frames).cuda()
    for s in (1 / 6, 1 / 3, 2 / 9):
        _, dh, dw = nat.resize_query(h, w, s)
        rc, dst = resize_frames(x, kind, h, w, s, dh + 1, dw + 4)
        assert rc == 0, nat.lib().lfd_last_error()
        assert np.array_equal(dst[:, :dh, :dw].cpu().numpy(), cv2_resized(kind, frames, s)), (kind, s)
        assert bool((dst[:, dh:] == GUARD).all()) and bool((dst[:, :, dw:] == GUARD).all())


def _host_rows(dets, labels, counts, cap):
    return LFD._rows(dets, labels, counts.clone(), torch.zeros(1, dtype=torch.int32), cap)


def _gray_model():
    return gray_pair('WIDERFACE_XS')[0].cuda()


E2E = [
    # name, dtype, network H x W, source h x w, frame format, pipeline
    ('WIDERFACE_S', 'bf16', (720, 1280), (1080, 1920), 'bgr'),     # the fused four-conv stem; extent == capacity
    ('WIDERFACE_S', 'fp16', (720, 1280), (1080, 1920), 'nv12'),
    ('WIDERFACE_S', 'bf16', (720, 1280), (1000, 1700), 'bgr'),     # s = 0.72: 720 x 1224, below the capacity
    ('TL_S', 'bf16', (256, 320), (480, 640), 'bgr'),               # s = 0.5 (INTER_AREA); 48-wide stem, BGR2RGB + standard_normalize
    ('TL_S', 'fp16', (256, 320), (300, 500), 'nv12'),
    ('GRAY', 'bf16', (256, 320), (540, 720), 'gray'),
    ('GRAY', 'bf16', (256, 320), (540, 720), 'nv12'),
]


@pytest.mark.parametrize('name,dtype,net,src,fmt', E2E)
def test_streaming_detector_with_source_size(name, dtype, net, src, fmt):
    model = _gray_model() if name == 'GRAY' else model_of(name, 'cuda')
    pipeline = tl_val_pipeline if name == 'TL_S' else None
    (H, W), (h, w), N = net, src, 2
    thr = {'WIDERFACE_S': 0.5, 'TL_S': 0.9}.get(name, 0.3)      # (fewer detections than max_out rows per frame)
    own = model.act_dtype, model._classification_threshold, model._nms_cfg
    model.act_dtype, model._classification_threshold, model._nms_cfg = dtype, thr, dict(type='nms', iou_thr=0.4)
    try:
        det = StreamingDetector(model, N, H, W, thr, 0.4, max_out=model.max_detections_per_image, input_pipeline=pipeline, frame_format=fmt, source_size=(h, w))
        s = det.resize_scale
        assert s == min(H / h, W / w)
        _, dh, dw = nat.resize_query(h, w, s)
        kind = fmt if fmt != 'nv12' or name != 'GRAY' else 'nv12_gray'
        if kind == 'bgr' and name != 'GRAY':
            host = np.stack([synth.synth_image_u8(h, w, seed=i) for i in range(N)])
        else:
            host = sources(kind, N, h, w, seed=h)
        assert det.h2d_bytes == host.nbytes
        dets, labels, counts = det.infer(torch.from_numpy(host).pin_memory())
        assert int(counts.max()) < det.max_out, 'every row read back'
        got = _host_rows(dets, labels, counts, det.max_out)
        assert _host_rows(*det.infer(torch.from_numpy(host).pin_memory()), det.max_out) == got      # (both output slots in use now)
        graphs = det.plan.num_graphs()
        for _ in range(3):                                       # repeated batches at one source size: no further graph
            assert _host_rows(*det.infer(torch.from_numpy(host).pin_memory()), det.max_out) == got
        assert det.plan.num_graphs() == graphs
        # the same plan on the frames cv2 resized on the host, at the same extent
        x = torch.from_numpy(host).cuda()
        with torch.no_grad():
            cls, reg = (t.clone() for t in det.plan.forward(x, resize_scale=s, frame_format='nv12' if fmt == 'nv12' else None))
            assert det.plan.num_graphs() == graphs
            ref = torch.from_numpy(cv2_resized(kind, host, s)).cuda()
            assert tuple(ref.shape[1:3]) == (dh, dw)
            rcls, rreg = (t.clone() for t in det.plan.forward(ref))
        same_bits(cls, rcls, '%s %s cls' % (name, fmt))
        same_bits(reg, rreg, '%s %s reg' % (name, fmt))
        for i, hw in enumerate(det.plan.frame_level_sizes):
            model._head_indexes_to_feature_map_sizes[i] = hw
        meta = [dict(resize_scale=s, resized_height=int(h * s), resized_width=int(w * s))] * N
        want = model.get_results((rcls, rreg), meta)
        assert got == want, (name, fmt, [len(r) for r in got], [len(r) for r in want])
        assert sum(len(r) for r in got) > 0
        # dets in source-frame coordinates: clamped to int(w * s) x int(h * s), then divided by s (x + w = x2 + 1, float32)
        boxes = [r[2:] for rr in got for r in rr]
        assert max(b[0] + b[2] for b in boxes) <= w + 1.01 and max(b[1] + b[3] for b in boxes) <= h + 1.01
    finally:
        model.act_dtype, model._classification_threshold, model._nms_cfg = own


def test_explicit_scale_and_refusals_of_the_python_path():
    model = model_of('WIDERFACE_S', 'cuda')
    with pytest.raises(ValueError, match='beyond'):
        StreamingDetector(model, 2, 360, 640, 0.3, 0.4, source_size=(1080, 1920), resize_scale=0.5)
    with pytest.raises(ValueError):
        StreamingDetector(model, 2, 360, 640, 0.3, 0.4, source_size=(1080, 1920), resize_scale=0.0)
    with pytest.raises(ValueError, match='even'):
        StreamingDetector(model, 2, 360, 640, 0.3, 0.4, frame_format='nv12', source_size=(1081, 1920))
    det = StreamingDetector(model, 2, 360, 640, 0.3, 0.4, source_size=(1080, 1920), resize_scale=0.25)
    assert det.resize_scale == 0.25 and det.post._meta_host == ((480.0,) * 2, (270.0,) * 2, (0.25,) * 2)
    plan = det.plan
    with pytest.raises(ValueError, match='beyond'):
        plan.forward(torch.zeros((2, 1080, 1920, 3), dtype=torch.uint8, device='cuda'), resize_scale=0.5)
    with pytest.raises(ValueError, match='uint8'):
        plan.forward(torch.zeros((2, 3, 1080, 1920), device='cuda'), resize_scale=0.25)
    gray = _gray_model()
    gplan = gray.inference_plan(2, 128, 160, torch.device('cuda'), exact=True)
    with pytest.raises(ValueError, match=r'uint8 \[N, h, w\]'):                   # a BGR source on a gray model
        gplan.forward(torch.zeros((2, 256, 320, 3), dtype=torch.uint8, device='cuda'), resize_scale=0.5)


def test_refused_calls_write_nothing():
    x = torch.from_numpy(sources('bgr', 2, 64, 96)).cuda()
    nv = torch.from_numpy(sources('nv12', 2, 64, 96)).cuda()
    dst = torch.full((2, 32, 48, 3), GUARD, dtype=torch.uint8, device='cuda')
    lib = nat.lib()
    cases = [((x, 'bgr', 64, 96, 0.6, 32, 48), LFD_ERR_CAPACITY),     # a result larger than the capacity
             ((x, 'bgr', 64, 96, 0.0, 32, 48), LFD_ERR_INVALID),
             ((x, 'bgr', 64, 96, float('nan'), 32, 48), LFD_ERR_INVALID),
             ((x, 'bgr', 64, 96, -0.5, 32, 48), LFD_ERR_INVALID),
             ((nv, 'nv12', 63, 96, 0.5, 32, 48), LFD_ERR_INVALID),    # an odd NV12 source
             ((nv, 'nv12', 64, 95, 0.5, 32, 48), LFD_ERR_INVALID)]
    for args, code in cases:
        rc, _ = resize_frames(*args, dst=dst)
        assert rc == code, (args[1:], rc, lib.lfd_last_error())
        assert bool((dst == GUARD).all()), args[1:]
    f32 = torch.zeros((2, 3, 64, 96), device='cuda')
    rc = lib.lfd_resize_frames(nat.ptr(f32), nat.INPUT_F32_NCHW, 3, 2, 64, 96, 0.5, nat.ptr(dst), 32, 48, nat.stream_ptr())
    torch.cuda.synchronize()
    assert rc == LFD_ERR_UNSUPPORTED and bool((dst == GUARD).all())


def test_engine_detect_resized_equals_the_python_path(tmp_path):
    model = model_of('WIDERFACE_S', 'cuda')
    N, H, W = 2, 360, 640
    path = str(tmp_path / 'm.lfd')
    plan, post = export_model(model, path, N, H, W, classification_threshold=0.3, autotune=False)
    eng = Engine(open(path, 'rb').read(), poison=0xff)
    nat.check(eng.bind())
    frames = torch.full((N, H, W, 3), GUARD, dtype=torch.uint8, device='cuda')
    assert frames.data_ptr() % 256 == 0
    lib = nat.lib()

    def engine_resized(x, fmt, h, w, s, buf=frames):
        with torch.cuda.device(0):
            return lib.lfd_engine_detect_resized(eng.handle, nat.ptr(x), fmt, h, w, s, nat.ptr(buf), nat.ptr(eng.dets), nat.ptr(eng.labels),
                                                 nat.ptr(eng.count), nat.ptr(eng.cls), nat.ptr(eng.reg), 1, nat.stream_ptr())

    total = 0
    for (h, w), kind, s in (((540, 960), 'bgr', 2 / 3), ((1080, 1920), 'nv12', 0.3), ((700, 1000), 'bgr', 0.5), ((200, 400), 'bgr', 1.5)):
        host = np.stack([synth.synth_image_u8(h, w, seed=i) for i in range(N)]) if kind == 'bgr' else sources(kind, N, h, w)
        x = torch.from_numpy(host).cuda()
        fmt = KINDS[kind][0]
        with torch.no_grad():
            cls, reg = (t.clone() for t in plan.forward(x, resize_scale=s, frame_format='nv12' if kind == 'nv12' else None))
        model._post_levels(post.cfg, plan.frame_level_sizes)
        post.set_meta([int(w * s)] * N, [int(h * s)] * N, [s] * N)
        post.run(cls, reg)
        want = [t.clone() for t in (post.dets, post.labels, post.count)]
        for _ in range(2):
            assert engine_resized(x, fmt, h, w, s) == 0, lib.lfd_last_error()
            torch.cuda.synchronize()
            ecls, ereg = eng.frame_outputs(plan.frame_P)
            assert torch.equal(ecls, cls) and torch.equal(ereg, reg), (h, w, kind, s)
            assert torch.equal(eng.count, want[2]), (h, w, kind, s)
            for i in range(N):
                k = int(want[2][i])
                assert torch.equal(eng.dets[i, :k], want[0][i, :k]) and torch.equal(eng.labels[i, :k], want[1][i, :k]), (h, w, kind, s, i)
        total += int(want[2][:N].sum())
        if (h, w, kind) == (540, 960, 'bgr'):
            program_rows = rows(*want)
            program_input = host
    assert total > 0
    # refusals: nothing is written to the frames buffer or the outputs
    eng.dets.fill_(-1.0)
    frames.fill_(GUARD)
    x = torch.from_numpy(sources('bgr', N, 540, 960)).cuda()
    odd = torch.empty(frames.numel() + 256, dtype=torch.uint8, device='cuda')
    for call, code in ((lambda: engine_resized(x, nat.INPUT_U8_NHWC, 540, 960, 0.7), LFD_ERR_CAPACITY),
                       (lambda: engine_resized(x, nat.INPUT_U8_NHWC, 540, 960, 0.0), LFD_ERR_INVALID),
                       (lambda: engine_resized(x, nat.INPUT_F32_NCHW, 540, 960, 0.5), LFD_ERR_UNSUPPORTED),
                       (lambda: engine_resized(x, nat.INPUT_U8_NHWC, 540, 960, 0.5, buf=odd[16:]), LFD_ERR_INVALID)):
        assert call() == code, lib.lfd_last_error()
        torch.cuda.synchronize()
        assert bool((frames == GUARD).all()) and bool((eng.dets == -1.0).all())
    # examples/lfd_detect --scale prints the same rows
    assert os.path.exists(PROGRAM), 'build() links examples/lfd_detect.c next to the library'
    (tmp_path / 'src.raw').write_bytes(program_input.tobytes())
    env = dict(os.environ)
    for line in open('/proc/self/maps'):
        if 'libcudart.so' in line:
            env['LD_LIBRARY_PATH'] = os.path.dirname(line.split()[-1]) + os.pathsep + env.get('LD_LIBRARY_PATH', '')
            break
    r = subprocess.run([PROGRAM, path, str(tmp_path / 'src.raw'), '540', '960', 'bgr', '--scale', repr(2 / 3)], capture_output=True, text=True,
                       env=env, timeout=300)
    assert r.returncode == 0, r.stderr
    got, cur = [], None
    for line in r.stdout.splitlines():
        f = line.split()
        if f[0] == 'frame':
            cur = []
            got.append(cur)
        else:
            cur.append([int(f[0])] + [float(np.float32(v)) for v in f[1:]])
    assert got == program_rows
