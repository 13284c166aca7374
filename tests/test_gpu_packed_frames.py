# -*- coding: utf-8 -*-
"""Packed camera frames (LFD_INPUT_U8_YUY2 / _UYVY / _BGRA / _RGBA).  The defining property: every op and every plan gives on a packed
frame f, bit for bit, what the uint8 BGR path gives on cv2.cvtColor(f, COLOR_{YUY2,UYVY,BGRA,RGBA}2BGR) (tests/packed_oracle.py) under
the same input transform, and a gray model on a 4:2:2 frame what it gives on the frame's Y bytes.  Every comparison runs the same op or
plan on the packed frames and on their oracle frames.  Each packed frame lies in a buffer with guard bytes behind it, and the guard
bytes (and the alpha bytes of BGRA / RGBA) are filled with two different patterns: neither may change a result."""
import ctypes as C

import numpy as np
import pytest
import torch

from gpu_ops import run_stem0
from gray_models import gray_pair
from helpers import (CONV_KINDS, close_downstream_of_gn, downstream_of_gn, misaligned, model_of, poison, same_bits, synth_model,
                     untouched)
from lfd import _native as nat
from lfd._engine import InferencePlan
from lfd.data_pipeline.augmentation import input_transform_of, typical_coco_val_pipeline
from packed_oracle import BYTES, FORMATS, packed_frames, packed_gray, packed_oracle
from test_input_transform_host import tl_val_pipeline

pytestmark = pytest.mark.gpu

LFD_ERR_INVALID, LFD_ERR_UNSUPPORTED = 1, 3
CODES = {'yuy2': nat.INPUT_U8_YUY2, 'uyvy': nat.INPUT_U8_UYVY, 'bgra': nat.INPUT_U8_BGRA, 'rgba': nat.INPUT_U8_RGBA}
YUV = ('yuy2', 'uyvy')
PATTERNS = (0x00, 0xff)
# zero fields = simple_normalize; the TrafficLight pipeline (BGR -> RGB, per-channel constants); caffe (BGR, per-channel constants)
TRANSFORMS = {'zero-fields': None, 'rgb-standard': tl_val_pipeline, 'caffe': typical_coco_val_pipeline}


def guarded(host, fmt, pattern):
    """A device copy of packed frames `host` [n, h, w, b] in a buffer whose 4096 bytes behind the frames hold `pattern`; BGRA / RGBA
    frames get `pattern` as their alpha bytes too."""
    x = torch.from_numpy(np.ascontiguousarray(host))
    if BYTES[fmt] == 4:
        x = x.clone()
        x[..., 3] = pattern
    buf = torch.full((x.numel() + 4096,), pattern, dtype=torch.uint8, device='cuda')
    buf[:x.numel()].copy_(x.view(-1).cuda())
    return buf[:x.numel()].view(x.shape)


def frames(fmt, n, h, w, seed=0):
    """(host packed frames [n, h, w, b], their oracle BGR frames on the device)"""
    host = packed_frames(n, h, w, fmt, seed)
    return host, torch.from_numpy(packed_oracle(host, fmt)).cuda()


SIZES = [(40, 44), (42, 46), (41, 46), (42, 44)]           # W = 0 and 2 (mod 4), an odd height


@pytest.mark.parametrize('fmt', FORMATS)
@pytest.mark.parametrize('name', sorted(TRANSFORMS))
@pytest.mark.parametrize('dtype', ['bf16', 'fp16'])
@pytest.mark.parametrize('cout', [16, 32, 48, 64])
def test_stem0_equals_stem0_on_the_converted_frames(cout, dtype, name, fmt):
    transform = input_transform_of(TRANSFORMS[name])
    g = torch.Generator().manual_seed(cout)
    w = torch.randn((cout, 3, 3, 3), generator=g) * 0.05
    shift = torch.randn(cout, generator=g) * 0.1
    tail = (torch.randn((cout, cout, 1, 1), generator=g) * 0.1, torch.ones(cout), torch.randn(cout, generator=g) * 0.1, True)
    for h, wd in SIZES:
        host, bgr = frames(fmt, 2, h, wd, seed=cout)
        for t in (None, tail):
            for ctas in (0, 3):
                ref = run_stem0(bgr, nat.INPUT_U8_NHWC, w, shift, tail=t, transform=transform, dtype=dtype, max_ctas=ctas)[0]
                for pattern in PATTERNS:
                    what = 'stem0 %s Cout=%d%s %s %s %dx%d, max_ctas=%d, guard 0x%02x' % (fmt, cout, ' + tail' if t else '', dtype, name, h, wd,
                                                                                         ctas, pattern)
                    same_bits(run_stem0(guarded(host, fmt, pattern), CODES[fmt], w, shift, tail=t, transform=transform, dtype=dtype,
                                        max_ctas=ctas)[0], ref, what)
        same_bits(run_stem0(guarded(host, fmt, 0xff), CODES[fmt], w, shift, transform=transform, dtype=dtype, impl=nat.CONV_SIMT)[0],
                  run_stem0(bgr, nat.INPUT_U8_NHWC, w, shift, transform=transform, dtype=dtype, impl=nat.CONV_SIMT)[0],
                  'SIMT stem0 %s Cout=%d %s %s %dx%d' % (fmt, cout, dtype, name, h, wd))


@pytest.mark.parametrize('fmt', YUV)
@pytest.mark.parametrize('dtype', ['bf16', 'fp16'])
@pytest.mark.parametrize('cout', [16, 32, 48, 64])
def test_gray_stem0_reads_the_y_bytes(cout, dtype, fmt):
    g = torch.Generator().manual_seed(cout)
    w = torch.randn((cout, 1, 3, 3), generator=g) * 0.05
    shift = torch.randn(cout, generator=g) * 0.1
    for h, wd in SIZES:
        host = packed_frames(2, h, wd, fmt, seed=cout)
        gray = torch.from_numpy(packed_gray(host, fmt)).cuda()
        for impl in (nat.CONV_UMMA, nat.CONV_SIMT):
            ref = run_stem0(gray, nat.INPUT_U8_NHWC, w, shift, cin=1, dtype=dtype, impl=impl)[0]
            for pattern in PATTERNS:
                same_bits(run_stem0(guarded(host, fmt, pattern), CODES[fmt], w, shift, cin=1, dtype=dtype, impl=impl)[0], ref,
                          'gray stem0 %s Cout=%d %s %dx%d impl %d guard 0x%02x' % (fmt, cout, dtype, h, wd, impl, pattern))


# ------------------------------------------------------------------------------------------------------------------ plans
def _has_gn(plan):
    return any(op['kind'] == nat.OP_GN_APPLY or (op['kind'] == nat.OP_HEAD_FINAL and op.get('gn_groups')) for op in plan._ops)


def snapshot(plan, x, frame_format, graph, h, w, resize_scale=None):
    """Forward of x on a poisoned plan (built with reuse=False) -> (conv outputs cropped to the frame's valid region, cls, reg)."""
    poison(plan)
    with torch.no_grad():
        for _ in range(2 if graph else 1):
            cls, reg = plan.forward(x, use_graph=graph, frame_format=frame_format, resize_scale=resize_scale)
    torch.cuda.synchronize()
    rows = plan.extent_table(h, w)[0]
    tensors = {}
    for op, r in zip(plan._ops, rows):
        if op['kind'] in CONV_KINDS:
            for k in ('out', 'out2'):
                if op.get(k) is not None:
                    tensors[op[k]] = plan.tensor(op[k])[:, :r[2], :r[3]].clone()
    return tensors, cls.clone(), reg.clone()


def compare(what, plan, got, ref):
    """Every conv output that does not depend on a GroupNorm bit for bit; the rest, and the heads of GroupNorm configs, up to the fp64
    atomics of the statistics; the heads of the other configs bit for bit."""
    tainted = downstream_of_gn(plan)
    (gt, gc, gr), (rt, rc, rr) = got, ref
    assert sorted(gt) == sorted(rt)
    for name in rt:
        if name in tainted:
            close_downstream_of_gn('%s: %s' % (what, name), gt[name].float(), rt[name].float())
        else:
            same_bits(gt[name], rt[name], '%s: %s' % (what, name))
    assert gc.shape == rc.shape and gr.shape == rr.shape, what
    if _has_gn(plan):
        close_downstream_of_gn(what + ': cls', gc, rc)
        close_downstream_of_gn(what + ': reg', gr, rr)
    else:
        assert torch.equal(gc, rc) and torch.equal(gr, rr), '%s: head outputs differ' % what


def _replan(plan, ctas):
    plan._op_array[0].max_ctas = ctas
    old, plan.handle = plan.handle, plan._create_handle()
    nat.lib().lfd_plan_destroy(old)


@pytest.mark.parametrize('fmt', FORMATS)
@pytest.mark.parametrize('name', ['zero-fields', 'rgb-standard'])
@pytest.mark.parametrize('dtype', ['bf16', 'fp16'])
def test_fused_stem_on_both_loaders(dtype, name, fmt):
    """STEM4 (WIDERFACE_S, forced): the word loader (W % 4 == 0 at an aligned base), the per-pixel loader (W % 4 == 2, or a base address
    = 1 mod 4); the default grid and the stem bounded to 1 and 7 CTAs: the whole plan against the same plan on the converted frames."""
    model = model_of('WIDERFACE_S', 'cuda')
    for h, w in ((186, 252), (186, 254), (187, 252)):
        plan = InferencePlan(model, 2, h, w, torch.device('cuda'), act_dtype=dtype, fuse_stem=True, input_transform=input_transform_of(TRANSFORMS[name]),
                             reuse=False)
        assert plan._ops[0]['kind'] == nat.OP_STEM4
        host, bgr = frames(fmt, 2, h, w, seed=h + w)
        ref = snapshot(plan, bgr, None, False, h, w)
        for pattern in PATTERNS:
            x = guarded(host, fmt, pattern)
            for xin in ([x, misaligned(x)] if w % 4 == 0 else [x]):
                for ctas in (0, 1, 7):
                    _replan(plan, ctas)
                    got = snapshot(plan, xin, fmt, False, h, w)
                    what = 'stem4 %s %s %s %dx%d base %% 4 = %d, max_ctas=%d, guard 0x%02x' % (fmt, dtype, name, h, w, xin.data_ptr() % 4, ctas,
                                                                                               pattern)
                    same_bits(got[0]['stem3'], ref[0]['stem3'], what)
                    compare(what, plan, got, ref)
                _replan(plan, 0)


PLANS = [('WIDERFACE_XS', None, 'bf16'), ('WIDERFACE_S', True, 'bf16'), ('WIDERFACE_S', False, 'fp16'), ('TL_S', None, 'bf16'),
         ('TL_S', None, 'fp16')]


@pytest.mark.parametrize('fmt', FORMATS)
@pytest.mark.parametrize('cfg,fuse,dtype', PLANS)
def test_whole_plans(cfg, fuse, dtype, fmt):
    model = model_of(cfg, 'cuda')
    plan = InferencePlan(model, 2, 400, 656, torch.device('cuda'), act_dtype=dtype, fuse_stem=fuse,
                         input_transform=input_transform_of(tl_val_pipeline if cfg.startswith('TL') else None), reuse=False)
    if fuse is not None:
        assert (plan._ops[0]['kind'] == nat.OP_STEM4) == fuse
    host, bgr = frames(fmt, 2, 400, 656, seed=5)
    for graph in (False, True):
        ref = snapshot(plan, bgr, None, graph, 400, 656)
        for pattern in PATTERNS:
            what = '%s fuse=%s %s %s graph=%d guard 0x%02x' % (cfg, fuse, dtype, fmt, graph, pattern)
            compare(what, plan, snapshot(plan, guarded(host, fmt, pattern), fmt, graph, 400, 656), ref)


# the capacity; h = 0 and 2 (mod 4) and odd; w = 0 and 2 (mod 4); deepest levels of 1 x 1; the smallest frame
BELOW = [(400, 656), (398, 654), (397, 652), (396, 650), (258, 130), (130, 260), (100, 120), (36, 6), (1, 2)]


@pytest.mark.parametrize('cfg,fuse', [('WIDERFACE_S', True), ('TL_S', None)])
def test_frames_below_the_capacity(cfg, fuse):
    """One 2 x 400 x 656 plan and frames of every size below it (lfd_plan_forward_extent through the plan's staging input), in every
    packed format, at the default grid and with the image op bounded to 3 CTAs."""
    model = model_of(cfg, 'cuda')
    plan = InferencePlan(model, 2, 400, 656, torch.device('cuda'), fuse_stem=fuse, reuse=False,
                         input_transform=input_transform_of(tl_val_pipeline if cfg.startswith('TL') else None))
    for ctas in (0, 3):
        _replan(plan, ctas)
        for i, (h, w) in enumerate(BELOW):
            fmt = FORMATS[i % 4]
            host, bgr = frames(fmt, 2, h, w, seed=i)
            for graph in (False, True):
                what = '%s %s %dx%d graph=%d max_ctas=%d' % (cfg, fmt, h, w, graph, ctas)
                got = snapshot(plan, guarded(host, fmt, 0xff), fmt, graph, h, w)
                assert got[1].shape[1] == plan.frame_P
                compare(what, plan, got, snapshot(plan, bgr, None, graph, h, w))


@pytest.mark.parametrize('fmt', YUV)
@pytest.mark.parametrize('cfg,fuse', [('TL_S', None), ('WIDERFACE_S', True), ('WIDERFACE_S', False)])
def test_gray_models_read_the_y_bytes(cfg, fuse, fmt):
    gray = gray_pair(cfg)[0].cuda()
    plan = InferencePlan(gray, 2, 400, 656, torch.device('cuda'), fuse_stem=fuse, reuse=False)
    assert plan.in_channels == 1
    for h, w in ((400, 656), (398, 654), (37, 42)):
        host = packed_frames(2, h, w, fmt, seed=h)
        y = torch.from_numpy(packed_gray(host, fmt)).cuda()
        for graph in (False, True):
            ref = snapshot(plan, y, None, graph, h, w)
            for pattern in PATTERNS:
                compare('gray %s fuse=%s %s %dx%d graph=%d guard 0x%02x' % (cfg, fuse, fmt, h, w, graph, pattern), plan,
                        snapshot(plan, guarded(host, fmt, pattern), fmt, graph, h, w), ref)
    for fmt4 in ('bgra', 'rgba'):
        x = torch.zeros((2, 400, 656, 4), dtype=torch.uint8, device='cuda')
        assert 'colour' in untouched(plan, lambda: plan.forward(x, frame_format=fmt4))


@pytest.mark.parametrize('fmt', FORMATS)
def test_resized_forward_from_1080p(fmt):
    """forward(x, frame_format=fmt, resize_scale=s) from 1080p sources: LINEAR (1/3), AREA (1/2) and an upscale (1.1), against the same
    resize of the converted frames; a gray model on 4:2:2 against the resize of the Y bytes."""
    model = model_of('WIDERFACE_S', 'cuda')
    plan = InferencePlan(model, 2, 1188, 2112, torch.device('cuda'), reuse=False)
    host, bgr = frames(fmt, 2, 1080, 1920, seed=11)
    for s in (1 / 3, 0.5, 1.1):
        _, dh, dw = nat.resize_query(1080, 1920, s)
        ref = snapshot(plan, bgr, None, True, dh, dw, resize_scale=s)
        for pattern in PATTERNS:
            compare('resized %s s=%r guard 0x%02x' % (fmt, s, pattern), plan,
                    snapshot(plan, guarded(host, fmt, pattern), fmt, True, dh, dw, resize_scale=s), ref)
    if fmt in YUV:
        gplan = InferencePlan(gray_pair('TL_S')[0].cuda(), 2, 720, 1280, torch.device('cuda'), reuse=False)
        y = torch.from_numpy(packed_gray(host, fmt)).cuda()
        for s in (1 / 3, 2 / 3):
            _, dh, dw = nat.resize_query(1080, 1920, s)
            compare('gray resized %s s=%r' % (fmt, s), gplan, snapshot(gplan, guarded(host, fmt, 0xff), fmt, True, dh, dw, resize_scale=s),
                    snapshot(gplan, y, None, True, dh, dw, resize_scale=s))


def _detections(det, batches):
    out = []
    for x in batches:
        d, labels, counts = det.infer(x)
        out.append([(d[j, :int(counts[j])].clone(), labels[j, :int(counts[j])].clone()) for j in range(det.N)])
    return out


@pytest.mark.parametrize('fmt', FORMATS)
def test_streaming_detector(fmt):
    """StreamingDetector on pinned packed host frames against the synchronous path (plan.forward on the converted frames, the same
    post-process), at the network's size and from 1080p sources resized on the device; the TrafficLight input transform (BGR -> RGB
    and per-channel constants)."""
    from lfd.pipeline import StreamingDetector
    model = synth_model('TL_L', cls_bias=-1.0)[0].cuda().eval()
    n, h, w = 2, 232, 328
    for source in (None, (1080, 1920)):
        sh, sw = source or (h, w)
        det = StreamingDetector(model, n, h, w, 0.3, 0.3, max_out=512, input_pipeline=tl_val_pipeline, frame_format=fmt, source_size=source)
        assert det.h2d_bytes == n * sh * sw * BYTES[fmt]
        hosts = [packed_frames(n, sh, sw, fmt, seed=s) for s in range(3)]
        got = _detections(det, [torch.from_numpy(x).pin_memory() for x in hosts])
        ref = StreamingDetector(model, n, h, w, 0.3, 0.3, max_out=512, input_pipeline=tl_val_pipeline, frame_format='bgr', source_size=source)
        want = _detections(ref, [torch.from_numpy(packed_oracle(x, fmt)).pin_memory() for x in hosts])
        total = 0
        for b, (g, r) in enumerate(zip(got, want)):
            for j in range(n):
                (gd, gl), (rd, rl) = g[j], r[j]
                total += rd.shape[0]
                assert gd.shape == rd.shape and torch.equal(gl, rl) and torch.equal(gd, rd), (fmt, source, b, j)
        assert total > 0, (fmt, source)


def test_model_file_on_packed_frames(tmp_path):
    """lfd_engine_detect (at the capacity and below it) and lfd_engine_detect_resized on packed frames give what they give on the
    converted BGR frames, under the TrafficLight input transform."""
    from engine_file import Engine
    from lfd.deployment import export_model
    model = synth_model('TL_L', cls_bias=-1.0)[0].cuda().eval()
    N, H, W = 2, 360, 640
    path = str(tmp_path / 'm.lfd')
    plan, _ = export_model(model, path, N, H, W, input_pipeline=tl_val_pipeline, classification_threshold=0.3, autotune=False)
    lib = nat.lib()
    eng = Engine(open(path, 'rb').read(), poison=0xff)
    nat.check(eng.bind())
    frames_buf = torch.zeros((N, H, W, 3), dtype=torch.uint8, device='cuda')

    def outputs(P):
        """the frame's network outputs, the counts and each image's detections (the rows below its count)"""
        torch.cuda.synchronize()
        c, r = eng.frame_outputs(P)
        rows = [(eng.dets[i, :int(eng.count[i])].clone(), eng.labels[i, :int(eng.count[i])].clone()) for i in range(N)]
        return [c.clone(), r.clone(), eng.count.clone()] + [t for pair in rows for t in pair]

    def same(a, b, what):
        assert len(a) == len(b), what
        for u, v in zip(a, b):
            assert torch.equal(u, v), what

    total = 0
    for fmt in FORMATS:
        stage = torch.zeros((N, H, W, BYTES[fmt]), dtype=torch.uint8, device='cuda')
        for h, w in ((360, 640), (358, 500)):
            host, bgr = frames(fmt, N, h, w, seed=h)
            P = plan.extent_table(h, w)[2]
            eng.detect(bgr, nat.INPUT_U8_NHWC, h, w)
            want = outputs(P)
            stage[:, :h, :w].copy_(guarded(host, fmt, 0x5a))
            nat.check(eng.detect_raw(stage, CODES[fmt], h, w))
            same(outputs(P), want, (fmt, h, w))
            total += int(want[2][:N].sum())
        host, bgr = frames(fmt, N, 1080, 1920, seed=3)
        for s in (1 / 3, 0.25):
            _, dh, dw = nat.resize_query(1080, 1920, s)
            P = plan.extent_table(dh, dw)[2]
            for x, code in ((bgr, nat.INPUT_U8_NHWC), (guarded(host, fmt, 0xa5), CODES[fmt])):
                with torch.cuda.device(0):
                    nat.check(lib.lfd_engine_detect_resized(eng.handle, nat.ptr(x), code, 1080, 1920, s, nat.ptr(frames_buf), nat.ptr(eng.dets),
                                                            nat.ptr(eng.labels), nat.ptr(eng.count), nat.ptr(eng.cls), nat.ptr(eng.reg), 1,
                                                            nat.stream_ptr()))
                if code == nat.INPUT_U8_NHWC:
                    want = outputs(P)
                else:
                    same(outputs(P), want, (fmt, 'resized', s))
    assert total > 0


# ------------------------------------------------------------------------------------------------------------------ errors
def _rc(plan, call):
    """The return code of a C entry point that must fail before anything is enqueued."""
    box = []

    def run():
        box.append(call())
        nat.check(box[-1])
    untouched(plan, run)
    return box[0]


def test_refusals_launch_nothing():
    model = model_of('TEST_FAST', 'cuda')
    lib = nat.lib()
    plan = InferencePlan(model, 2, 96, 160, torch.device('cuda'))
    # the Python checks
    for fmt in FORMATS:
        b = BYTES[fmt]
        for shape in [(2, 96, 160, 6 - b), (3, 96, 160, b), (2, 97, 160, b), (2, 96, 162, b), (2, 96, 160)]:
            x = torch.zeros(shape, dtype=torch.uint8, device='cuda')
            untouched(plan, lambda: plan.forward(x, frame_format=fmt))
    for fmt in YUV:
        assert 'even width' in untouched(plan, lambda: plan.forward(torch.zeros((2, 96, 159, 2), dtype=torch.uint8, device='cuda'), frame_format=fmt))
    stage = plan.staging(nat.INPUT_U8_BGRA)
    ms = (C.c_float * lib.lfd_plan_num_launches(plan.handle))()

    def extent(p, fmt, h, w, x):
        return lambda: lib.lfd_plan_forward_extent(p.handle, nat.ptr(x), fmt, h, w, p._extent(h, w)[0], nat.ptr(p.workspace),
                                                   nat.ptr(p.cls_out), nat.ptr(p.reg_out), 1, nat.stream_ptr())

    def forward(p, fmt, x):
        return lambda: lib.lfd_plan_forward(p.handle, nat.ptr(x), fmt, nat.ptr(p.workspace), nat.ptr(p.cls_out), nat.ptr(p.reg_out), 1,
                                            nat.stream_ptr())

    def profile(p, fmt, x):
        return lambda: lib.lfd_plan_profile(p.handle, nat.ptr(x), fmt, nat.ptr(p.workspace), nat.ptr(p.cls_out), nat.ptr(p.reg_out), ms,
                                            nat.stream_ptr())

    with torch.cuda.device(plan.device):
        for fmt in (nat.INPUT_U8_YUY2, nat.INPUT_U8_UYVY):      # an odd frame width
            assert _rc(plan, extent(plan, fmt, 64, 101, stage)) == LFD_ERR_INVALID
        for fmt in (3, -1, -2, 8):
            assert _rc(plan, extent(plan, fmt, 64, 100, stage)) == LFD_ERR_INVALID
            assert _rc(plan, forward(plan, fmt, stage)) == LFD_ERR_INVALID
            assert _rc(plan, profile(plan, fmt, stage)) == LFD_ERR_INVALID
        # 4:2:2 on a plan of odd capacity width
        odd = InferencePlan(model, 2, 96, 161, torch.device('cuda'))
        ostage = odd.staging(nat.INPUT_U8_BGRA)
        assert 'even width' in untouched(odd, lambda: odd.forward(torch.zeros((2, 96, 160, 2), dtype=torch.uint8, device='cuda'), frame_format='yuy2'))
        for fmt in (nat.INPUT_U8_YUY2, nat.INPUT_U8_UYVY):
            assert _rc(odd, forward(odd, fmt, ostage)) == LFD_ERR_UNSUPPORTED
            assert _rc(odd, profile(odd, fmt, ostage)) == LFD_ERR_UNSUPPORTED
            assert _rc(odd, extent(odd, fmt, 64, 100, ostage)) == LFD_ERR_UNSUPPORTED
        # BGRA / RGBA on a gray plan
        gplan = InferencePlan(gray_pair('WIDERFACE_XS')[0].cuda(), 2, 96, 160, torch.device('cuda'))
        gstage = gplan.staging(nat.INPUT_U8_BGRA)
        for fmt in (nat.INPUT_U8_BGRA, nat.INPUT_U8_RGBA):
            assert _rc(gplan, forward(gplan, fmt, gstage)) == LFD_ERR_UNSUPPORTED
            assert _rc(gplan, profile(gplan, fmt, gstage)) == LFD_ERR_UNSUPPORTED
            assert _rc(gplan, extent(gplan, fmt, 64, 100, gstage)) == LFD_ERR_UNSUPPORTED
    # lfd_run_op: a 4:2:2 STEM0 op of odd width, BGRA / RGBA on a gray op, formats outside the set
    w3, w1 = torch.randn((16, 3, 3, 3)) * 0.05, torch.randn((16, 1, 3, 3)) * 0.05
    for H, W, fmt, cin, want in ((40, 45, nat.INPUT_U8_YUY2, 3, LFD_ERR_UNSUPPORTED), (40, 45, nat.INPUT_U8_UYVY, 1, LFD_ERR_UNSUPPORTED),
                                 (40, 44, nat.INPUT_U8_BGRA, 1, LFD_ERR_UNSUPPORTED), (40, 44, nat.INPUT_U8_RGBA, 1, LFD_ERR_UNSUPPORTED),
                                 (40, 44, 3, 3, LFD_ERR_INVALID), (40, 44, 8, 3, LFD_ERR_INVALID)):
        x = torch.zeros((2, H, W, 4), dtype=torch.uint8, device='cuda')
        for impl in (nat.CONV_UMMA, nat.CONV_SIMT):
            rc, ws = run_stem0(x, fmt, w3 if cin == 3 else w1, torch.zeros(16), cin=cin, impl=impl, raw_rc=True)
            assert rc == want and bool((ws == 0xff).all()), (H, W, fmt, cin, impl, rc)
    # lfd_resize_frames: an odd 4:2:2 width, BGRA to gray
    src = torch.zeros((2, 64, 96, 4), dtype=torch.uint8, device='cuda')
    dst = torch.full((2, 32, 48, 3), 0x77, dtype=torch.uint8, device='cuda')
    for fmt, ch, w, want in ((nat.INPUT_U8_YUY2, 3, 95, LFD_ERR_INVALID), (nat.INPUT_U8_BGRA, 1, 96, LFD_ERR_UNSUPPORTED),
                             (nat.INPUT_U8_RGBA, 1, 96, LFD_ERR_UNSUPPORTED)):
        assert lib.lfd_resize_frames(nat.ptr(src), fmt, ch, 2, 64, w, 0.5, nat.ptr(dst), 32, 48, nat.stream_ptr()) == want
        torch.cuda.synchronize()
        assert bool((dst == 0x77).all())
    # training refuses the four packed formats (UNSUPPORTED), before anything is enqueued
    tm = synth_model('TL_L', cls_bias=-2.0)[0].cuda().train()
    tp = tm.train_plan_for(2, 128, 160, torch.device('cuda'))
    img = torch.zeros((2, 128, 160, 4), dtype=torch.uint8, device='cuda')
    tms = (C.c_float * max(len(tp.fwd_ops), len(tp.bwd_ops)))()
    for fmt in CODES.values():
        for call in (lambda: lib.lfd_train_plan_run(tp.fwd_handle, nat.ptr(img), fmt, nat.ptr(tp.workspace), 0, nat.stream_ptr()),
                     lambda: lib.lfd_train_plan_run(tp.fwd_handle, nat.ptr(img), fmt, nat.ptr(tp.workspace), 1, nat.stream_ptr()),
                     lambda: lib.lfd_train_plan_profile(tp.fwd_handle, nat.ptr(img), fmt, nat.ptr(tp.workspace), tms, nat.stream_ptr()),
                     lambda: lib.lfd_run_top(C.byref(tp._fwd_arr[0]), nat.ptr(img), fmt, nat.ptr(tp.workspace), nat.stream_ptr())):
            tp.workspace.view(torch.uint8).fill_(0xff)
            torch.cuda.synchronize()
            with torch.cuda.device(tp.device):
                rc = call()
            torch.cuda.synchronize()
            assert rc == LFD_ERR_UNSUPPORTED, (fmt, rc)
            assert bool((tp.workspace.view(torch.uint8) == 0xff).all())
