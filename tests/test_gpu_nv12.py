# -*- coding: utf-8 -*-
"""NV12 video frames (LFD_INPUT_U8_NV12).  The defining property: every op and every plan gives on an NV12 frame f, bit for bit, what the
uint8 BGR path gives on cv2.cvtColor(f, cv2.COLOR_YUV2BGR_NV12) (tests/nv12_oracle.py) under the same input transform.  Every comparison
here runs the same op or plan on the NV12 frames and on their oracle BGR frames."""
import ctypes as C
import functools

import numpy as np
import pytest
import torch

import tl_s
from gpu_ops import DTYPES, conv_out
from helpers import synth_model
from lfd import _native as nat
from lfd._engine import InferencePlan, fold_scale, pack_conv_weight, pack_stem_weight
from lfd.data_pipeline.augmentation import BGR2RGB, Compose, input_transform_of, simple_widerface_val_pipeline, typical_coco_val_pipeline
from nv12_oracle import nv12_frames, nv12_oracle
from test_input_transform_host import tl_val_pipeline

pytestmark = pytest.mark.gpu

LFD_ERR_INVALID, LFD_ERR_UNSUPPORTED = 1, 3

# the transforms of test_gpu_input_transform.py: name -> pipeline given to the kernels
TRANSFORMS = {
    'zero-fields': None,
    'simple': simple_widerface_val_pipeline,
    'swap-only': Compose([BGR2RGB()]),
    'rgb-standard': tl_val_pipeline,
    'caffe': typical_coco_val_pipeline,
}


def frames(n, h, w, seed=0):
    """(NV12 uint8 [n, 3h/2, w], its oracle BGR uint8 [n, h, w, 3]) on the device; the NV12 frames reach every clamp (nv12_frames)."""
    x = nv12_frames(n, h, w, seed)
    return torch.from_numpy(x).cuda(), torch.from_numpy(nv12_oracle(x)).cuda()


def same_bits(a, b, what):
    bad = a.view(torch.int16) != b.view(torch.int16)
    if bool(bad.any()):
        i = tuple(bad.nonzero()[0].tolist())
        raise AssertionError('%s: %d of %d elements differ, first at %s: %r vs %r' % (what, int(bad.sum()), bad.numel(), i, float(a[i]), float(b[i])))


def misaligned(x):
    raw = torch.empty(x.numel() + 1, dtype=torch.uint8, device='cuda')
    y = raw[1:].view(x.shape)                        # base address 1 (mod 4): the fused stem's per-pixel loader
    y.copy_(x)
    assert y.data_ptr() % 4 == 1
    return y


# ------------------------------------------------------------------------------------------------------------------ single ops
def run_stem0(x, fmt, transform, w, shift, tail, dtype, impl=nat.CONV_UMMA, max_ctas=0, raw_rc=False):
    """LFD_OP_STEM0 through lfd_run_op on uint8 BGR [N, H, W, 3] or NV12 [N, 3H/2, W] x -> [N, Ho, Wo, Cf]
    (raw_rc: -> (lfd_run_op's return code, the workspace))."""
    tdt, code = DTYPES[dtype][0], DTYPES[dtype][3]
    N, H, W = (x.shape[0], x.shape[1], x.shape[2]) if fmt == nat.INPUT_U8_NHWC else (x.shape[0], x.shape[1] * 2 // 3, x.shape[2])
    Cout = w.shape[0]
    Ho, Wo = conv_out(H, 3, 2), conv_out(W, 3, 2)
    Cf = tail[0].shape[0] if tail is not None else Cout
    keep = [pack_stem_weight(w, tdt).cuda(), shift.float().cuda()]
    out_b = N * Ho * Wo * Cf * 2
    ws = torch.full((4096 + ((out_b + 255) & ~255) + 256,), 0xff, dtype=torch.uint8, device='cuda')
    op = nat.Op()
    op.kind, op.dtype = nat.OP_STEM0, code
    op.N, op.H, op.W, op.Cin, op.Ho, op.Wo, op.Cout = N, H, W, 3, Ho, Wo, Cout
    op.ksize, op.stride, op.relu, op.max_ctas = 3, 2, 1, max_ctas
    op.in_off, op.out_off, op.res_off, op.stats_off, op.ds_out_off = -1, 4096, -1, -1, -1
    op.weight, op.shift = keep[0].data_ptr(), keep[1].data_ptr()
    if tail is not None:
        keep += [pack_conv_weight(fold_scale(tail[0], torch.ones(Cf)), Cout, tdt).cuda(), tail[1].float().cuda()]
        op.tail_cout, op.tail_relu, op.tail_weight, op.tail_shift = Cf, 1, keep[2].data_ptr(), keep[3].data_ptr()
    nat.set_input_transform(op, transform)
    torch.cuda.synchronize()
    rc = nat.lib().lfd_run_op(C.byref(op), nat.ptr(x), fmt, nat.ptr(ws), None, None, 0, 0, impl, nat.stream_ptr())
    torch.cuda.synchronize()
    if raw_rc:
        return rc, ws
    nat.check(rc)
    return ws[4096:4096 + out_b].view(tdt).view(N, Ho, Wo, Cf).clone()


SIZES = [(40, 44), (42, 46), (40, 46), (42, 44)]           # H and W = 0 and 2 (mod 4)


@pytest.mark.parametrize('name', sorted(TRANSFORMS))
@pytest.mark.parametrize('dtype', ['bf16', 'fp16'])
@pytest.mark.parametrize('cout', [16, 32, 48, 64])
def test_stem0_on_nv12_frames_equals_stem0_on_the_converted_frames(cout, dtype, name):
    transform = input_transform_of(TRANSFORMS[name])
    g = torch.Generator().manual_seed(cout)
    w = torch.randn((cout, 3, 3, 3), generator=g) * 0.05
    shift = torch.randn(cout, generator=g) * 0.1
    tail = (torch.randn((cout, cout, 1, 1), generator=g) * 0.1, torch.randn(cout, generator=g) * 0.1)
    for h, wd in SIZES:
        nv, bgr = frames(2, h, wd, seed=cout)
        for t in (None, tail):
            for ctas in (0, 3):
                what = 'stem0 Cout=%d%s %s %s %dx%d, max_ctas=%d' % (cout, ' + tail' if t else '', dtype, name, h, wd, ctas)
                same_bits(run_stem0(nv, nat.INPUT_U8_NV12, transform, w, shift, t, dtype, max_ctas=ctas),
                          run_stem0(bgr, nat.INPUT_U8_NHWC, transform, w, shift, t, dtype, max_ctas=ctas), what)
        same_bits(run_stem0(nv, nat.INPUT_U8_NV12, transform, w, shift, None, dtype, impl=nat.CONV_SIMT),
                  run_stem0(bgr, nat.INPUT_U8_NHWC, transform, w, shift, None, dtype, impl=nat.CONV_SIMT),
                  'SIMT stem0 Cout=%d %s %s %dx%d' % (cout, dtype, name, h, wd))


# ------------------------------------------------------------------------------------------------------------------ plans
@functools.lru_cache(maxsize=None)
def model_of(name):
    model = tl_s.synth_model()[0] if name == 'TL_S' else synth_model(name)[0]
    return model.cuda().eval()


CONV_KINDS = (nat.OP_STEM0, nat.OP_CONV, nat.OP_STEM4)


def _downstream_of_gn(plan):
    tainted = set()
    for op in plan._ops:
        if op['kind'] == nat.OP_GN_APPLY or any(op.get(k) in tainted for k in ('inp', 'res')):
            tainted |= {op[k] for k in ('out', 'out2') if op.get(k) is not None}
    return tainted


def _has_gn(plan):
    return any(op['kind'] == nat.OP_GN_APPLY or (op['kind'] == nat.OP_HEAD_FINAL and op.get('gn_groups')) for op in plan._ops)


def _poison(plan):
    plan.workspace.fill_(0xff)
    if plan._stage is not None:
        plan._stage.fill_(0xff)
    for c, r in plan._outputs:
        c.view(torch.uint8).fill_(0xff)
        r.view(torch.uint8).fill_(0xff)


def snapshot(plan, x, frame_format, graph, h, w):
    """Forward of x on a poisoned plan (built with reuse=False) -> (conv outputs cropped to the frame's valid region, cls, reg)."""
    _poison(plan)
    with torch.no_grad():
        for _ in range(2 if graph else 1):
            cls, reg = plan.forward(x, use_graph=graph, frame_format=frame_format)
    torch.cuda.synchronize()
    rows = plan.extent_table(h, w)[0]
    tensors = {}
    for op, r in zip(plan._ops, rows):
        if op['kind'] in CONV_KINDS:
            for k in ('out', 'out2'):
                if op.get(k) is not None:
                    tensors[op[k]] = plan.tensor(op[k])[:, :r[2], :r[3]].clone()
    return tensors, cls.clone(), reg.clone()


def _close(what, a, b):
    """Downstream of a GroupNorm: its fp64 statistics atomics add in another order from run to run (test_gpu_schedule_invariance.py)."""
    assert bool(torch.isfinite(a).all()), what
    d = (a - b).abs()
    assert float(d.max()) <= 2.0 ** -6 * float(b.abs().max()), (what, float(d.max()), int((d > 0).sum()))


def compare(what, plan, got, ref):
    """Every conv output that does not depend on a GroupNorm bit for bit; the rest, and the heads of GroupNorm configs, up to the fp64
    atomics of the statistics; the heads of the other configs bit for bit."""
    tainted = _downstream_of_gn(plan)
    (gt, gc, gr), (rt, rc, rr) = got, ref
    assert sorted(gt) == sorted(rt)
    for name in rt:
        if name in tainted:
            _close('%s: %s' % (what, name), gt[name].float(), rt[name].float())
        else:
            same_bits(gt[name], rt[name], '%s: %s' % (what, name))
    assert gc.shape == rc.shape and gr.shape == rr.shape, what
    if _has_gn(plan):
        _close(what + ': cls', gc, rc)
        _close(what + ': reg', gr, rr)
    else:
        assert torch.equal(gc, rc) and torch.equal(gr, rr), '%s: head outputs differ' % what


@pytest.mark.parametrize('name', sorted(TRANSFORMS))
@pytest.mark.parametrize('dtype', ['bf16', 'fp16'])
def test_fused_stem_on_both_loaders(dtype, name):
    """STEM4 (WIDERFACE_S, forced): the word loader (W % 4 == 0 at an aligned base), the per-pixel loader (W % 4 == 2, or a base address
    = 1 mod 4); the default grid and the stem bounded to 1, 7 and 131 CTAs (runs that start mid-row and cross images): the stem3 map bit
    for bit against the same plan on the converted frames."""
    model = model_of('WIDERFACE_S')
    for h, w in ((186, 252), (186, 254), (188, 250)):
        plan = InferencePlan(model, 2, h, w, torch.device('cuda'), act_dtype=dtype, fuse_stem=True, input_transform=input_transform_of(TRANSFORMS[name]),
                             reuse=False)
        assert plan._ops[0]['kind'] == nat.OP_STEM4
        nv, bgr = frames(2, h, w, seed=h + w)
        ref = snapshot(plan, bgr, None, False, h, w)
        inputs = [nv, misaligned(nv)] if w % 4 == 0 else [nv]
        for x in inputs:
            assert (w % 4 == 0 and x.data_ptr() % 4 == 0) or w % 4 == 2 or x.data_ptr() % 4 == 1
            for ctas in (0, 1, 7, 131):
                plan._op_array[0].max_ctas = ctas
                old, plan.handle = plan.handle, plan._create_handle()
                nat.lib().lfd_plan_destroy(old)
                got = snapshot(plan, x, 'nv12', False, h, w)
                what = 'stem4 %s %s %dx%d base %% 4 = %d, max_ctas=%d' % (dtype, name, h, w, x.data_ptr() % 4, ctas)
                same_bits(got[0]['stem3'], ref[0]['stem3'], what)
                compare(what, plan, got, ref)


PLANS = [('WIDERFACE_S', True, 'bf16'), ('WIDERFACE_S', False, 'bf16'), ('TL_L', None, 'bf16'), ('TL_S', None, 'bf16'),
         ('TT100K_L', None, 'bf16'), ('WIDERFACE_L', None, 'fp16')]


@pytest.mark.parametrize('cfg,fuse,dtype', PLANS)
def test_whole_plans(cfg, fuse, dtype):
    model = model_of(cfg)
    plan = InferencePlan(model, 2, 400, 656, torch.device('cuda'), act_dtype=dtype, fuse_stem=fuse,
                         input_transform=input_transform_of(tl_val_pipeline if cfg.startswith('TL') else None), reuse=False)
    assert (plan._ops[0]['kind'] == nat.OP_STEM4) == bool(fuse)
    nv, bgr = frames(2, 400, 656, seed=5)
    for graph in (False, True):
        what = '%s fuse=%s %s graph=%d' % (cfg, fuse, dtype, graph)
        compare(what, plan, snapshot(plan, nv, 'nv12', graph, 400, 656), snapshot(plan, bgr, None, graph, 400, 656))


# the capacity; h, w = 0 and 2 (mod 4); deepest levels of 1 x 1 (100 x 120, 36 x 6); the smallest frame; widths with and without the
# word loader's w % 4 == 0
BELOW = [(400, 656), (398, 654), (396, 652), (398, 652), (396, 654), (258, 130), (130, 260), (100, 120), (36, 6), (2, 2)]


@pytest.mark.parametrize('cfg,fuse', [('WIDERFACE_S', True), ('TL_L', None), ('TT100K_L', None)])
def test_frames_below_the_capacity(cfg, fuse):
    """One 2 x 400 x 656 plan, a scrambled sequence of even frame sizes, every buffer pre-filled with 0xff before each frame: each NV12
    frame gives what its converted BGR frame gives on the same plan; two graphs per format (the caller's tensor at the capacity, the
    plan's staging buffer below it)."""
    model = model_of(cfg)
    plan = InferencePlan(model, 2, 400, 656, torch.device('cuda'), fuse_stem=fuse, reuse=False,
                         input_transform=input_transform_of(tl_val_pipeline if cfg.startswith('TL') else None))
    assert (plan._ops[0]['kind'] == nat.OP_STEM4) == bool(fuse)
    plan.staging(nat.INPUT_U8_NHWC)
    rng = np.random.RandomState(3)
    seq = BELOW[1:] * 2
    rng.shuffle(seq)
    held_nv = torch.empty((2, 600, 656), dtype=torch.uint8, device='cuda')
    held_bgr = torch.empty((2, 400, 656, 3), dtype=torch.uint8, device='cuda')
    for i, (h, w) in enumerate([BELOW[0]] + seq[:9] + [BELOW[0]] + seq[9:]):
        nv, bgr = frames(2, h, w, seed=i)
        if (h, w) == (400, 656):
            held_nv.copy_(nv)
            held_bgr.copy_(bgr)
            nv, bgr = held_nv, held_bgr
        for graph in (False, True):
            what = '%s %dx%d graph=%d' % (cfg, h, w, graph)
            got = snapshot(plan, nv, 'nv12', graph, h, w)
            assert got[1].shape[1] == plan.frame_P
            compare(what, plan, got, snapshot(plan, bgr, None, graph, h, w))
    assert plan.num_graphs() == 4, plan.num_graphs()


@pytest.mark.parametrize('cfg,pipeline', [('TL_L', tl_val_pipeline), ('WIDERFACE_S', None)], ids=['TL_L', 'WIDERFACE_S'])
def test_streaming_detector_on_nv12_frames(cfg, pipeline):
    from lfd.pipeline import StreamingDetector
    model = synth_model(cfg, cls_bias=-1.0)[0].cuda().eval()
    n, h, w = 2, 232, 328
    dets = {}
    for fmt in ('nv12', 'bgr'):
        det = StreamingDetector(model, n, h, w, 0.3, 0.3, max_out=512, input_pipeline=pipeline, frame_format=fmt)
        assert det.h2d_bytes == (n * h * w * 3 if fmt == 'bgr' else n * h * w * 3 // 2)
        out = []
        for s in range(4):
            nv = nv12_frames(n, h, w, seed=s)
            x = torch.from_numpy(nv if fmt == 'nv12' else nv12_oracle(nv)).pin_memory()
            d, labels, counts = det.infer(x)
            out.append([(d[j, :int(counts[j])].clone(), labels[j, :int(counts[j])].clone()) for j in range(n)])
        dets[fmt] = out
    total = 0
    for b, (got, ref) in enumerate(zip(dets['nv12'], dets['bgr'])):
        for j in range(n):
            (gd, gl), (rd, rl) = got[j], ref[j]
            total += rd.shape[0]
            assert gd.shape == rd.shape and torch.equal(gl, rl), (cfg, b, j, gd.shape, rd.shape)
            if cfg == 'WIDERFACE_S':          # GroupNorm: the heads up to the fp64 atomics, the boxes and scores accordingly
                assert torch.allclose(gd, rd, rtol=1e-3, atol=1e-2), (cfg, b, j)
            else:
                assert torch.equal(gd, rd), (cfg, b, j)
    assert total > 0


# ------------------------------------------------------------------------------------------------------------------ errors
def _untouched(plan, call):
    """call() must fail before anything reaches the device: the workspace, the outputs and the staging keep their bytes."""
    plan.staging(nat.INPUT_U8_NHWC)
    _poison(plan)
    torch.cuda.synchronize()
    with pytest.raises((ValueError, nat.LfdError)) as e:
        call()
    torch.cuda.synchronize()
    assert bool((plan.workspace == 0xff).all()) and bool((plan._stage == 0xff).all())
    for c, r in plan._outputs:
        assert bool((c.view(torch.uint8) == 0xff).all()) and bool((r.view(torch.uint8) == 0xff).all())
    return str(e.value)


def _rc(plan, call):
    """The return code of a C entry point that must fail before anything is enqueued."""
    box = []

    def run():
        box.append(call())
        nat.check(box[-1])
    _untouched(plan, run)
    return box[0]


def test_errors_launch_nothing():
    model = model_of('TEST_FAST')
    lib = nat.lib()
    plan = InferencePlan(model, 2, 96, 160, torch.device('cuda'))
    # the host checks
    for shape in [(2, 145, 160), (2, 144, 161), (2, 96, 160, 3), (3, 144, 160), (1, 144, 160), (2, 150, 160), (2, 144, 162)]:
        x = torch.zeros(shape, dtype=torch.uint8, device='cuda')
        _untouched(plan, lambda: plan.forward(x, frame_format='nv12'))
    x = torch.zeros((2, 96, 160, 3), dtype=torch.uint8, device='cuda')
    assert 'frame_format' in _untouched(plan, lambda: plan.forward(x, frame_format='i420'))
    # the C entry points: an odd frame, a format outside 0..2
    stage = plan.staging(nat.INPUT_U8_NV12)
    ms = (C.c_float * lib.lfd_plan_num_launches(plan.handle))()

    def extent(fmt, h, w):
        return lambda: lib.lfd_plan_forward_extent(plan.handle, nat.ptr(stage), fmt, h, w, plan._extent(h, w)[0], nat.ptr(plan.workspace),
                                                   nat.ptr(plan.cls_out), nat.ptr(plan.reg_out), 1, nat.stream_ptr())

    def forward(p, fmt, x):
        return lambda: lib.lfd_plan_forward(p.handle, nat.ptr(x), fmt, nat.ptr(p.workspace), nat.ptr(p.cls_out), nat.ptr(p.reg_out), 1,
                                            nat.stream_ptr())

    def profile(p, fmt, x):
        return lambda: lib.lfd_plan_profile(p.handle, nat.ptr(x), fmt, nat.ptr(p.workspace), nat.ptr(p.cls_out), nat.ptr(p.reg_out), ms,
                                            nat.stream_ptr())

    with torch.cuda.device(plan.device):
        assert _rc(plan, extent(nat.INPUT_U8_NV12, 63, 100)) == LFD_ERR_INVALID
        assert _rc(plan, extent(nat.INPUT_U8_NV12, 64, 101)) == LFD_ERR_INVALID
        for fmt in (3, -1, 255):
            assert _rc(plan, extent(fmt, 64, 100)) == LFD_ERR_INVALID
            assert _rc(plan, forward(plan, fmt, stage)) == LFD_ERR_INVALID
            assert _rc(plan, profile(plan, fmt, stage)) == LFD_ERR_INVALID
        # NV12 on a plan of odd capacity
        odd = InferencePlan(model, 2, 97, 160, torch.device('cuda'))
        x = torch.zeros((2, 97 * 3 // 2 + 1, 160), dtype=torch.uint8, device='cuda')
        assert 'even' in _untouched(odd, lambda: odd.forward(x, frame_format='nv12'))
        assert _rc(odd, forward(odd, nat.INPUT_U8_NV12, x)) == LFD_ERR_UNSUPPORTED
        assert _rc(odd, profile(odd, nat.INPUT_U8_NV12, x)) == LFD_ERR_UNSUPPORTED
        ostage = odd.staging(nat.INPUT_U8_NHWC)
        assert _rc(odd, lambda: lib.lfd_plan_forward_extent(odd.handle, nat.ptr(ostage), nat.INPUT_U8_NV12, 64, 100, odd._extent(64, 100)[0],
                                                            nat.ptr(odd.workspace), nat.ptr(odd.cls_out), nat.ptr(odd.reg_out), 1,
                                                            nat.stream_ptr())) == LFD_ERR_UNSUPPORTED
    # lfd_run_op: a STEM0 op of odd width, a format outside 0..2
    w = torch.randn((16, 3, 3, 3)) * 0.05
    for H, W, fmt, want in ((40, 45, nat.INPUT_U8_NV12, LFD_ERR_UNSUPPORTED), (40, 44, 3, LFD_ERR_INVALID), (40, 44, -2, LFD_ERR_INVALID)):
        x = torch.zeros((2, H * 3 // 2, W), dtype=torch.uint8, device='cuda')
        for impl in (nat.CONV_UMMA, nat.CONV_SIMT):
            rc, ws = run_stem0(x, fmt, None, w, torch.zeros(16), None, 'bf16', impl=impl, raw_rc=True)
            assert rc == want and bool((ws == 0xff).all()), (H, W, fmt, impl, rc)
    # training refuses NV12 (UNSUPPORTED) and any format outside 0..2 (INVALID), before anything is enqueued
    tm = synth_model('TL_L', cls_bias=-2.0)[0].cuda().train()
    tp = tm.train_plan_for(2, 128, 160, torch.device('cuda'))
    img = torch.zeros((2, 192, 160), dtype=torch.uint8, device='cuda')
    tms = (C.c_float * max(len(tp.fwd_ops), len(tp.bwd_ops)))()
    for fmt, want in ((nat.INPUT_U8_NV12, LFD_ERR_UNSUPPORTED), (3, LFD_ERR_INVALID)):
        for call in (lambda: lib.lfd_train_plan_run(tp.fwd_handle, nat.ptr(img), fmt, nat.ptr(tp.workspace), 0, nat.stream_ptr()),
                     lambda: lib.lfd_train_plan_run(tp.fwd_handle, nat.ptr(img), fmt, nat.ptr(tp.workspace), 1, nat.stream_ptr()),
                     lambda: lib.lfd_train_plan_profile(tp.fwd_handle, nat.ptr(img), fmt, nat.ptr(tp.workspace), tms, nat.stream_ptr()),
                     lambda: lib.lfd_run_top(C.byref(tp._fwd_arr[0]), nat.ptr(img), fmt, nat.ptr(tp.workspace), nat.stream_ptr())):
            tp.workspace.view(torch.uint8).fill_(0xff)
            torch.cuda.synchronize()
            with torch.cuda.device(tp.device):
                rc = call()
            torch.cuda.synchronize()
            assert rc == want, (fmt, rc)
            assert bool((tp.workspace.view(torch.uint8) == 0xff).all())
