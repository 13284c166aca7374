# -*- coding: utf-8 -*-
"""Model files on the H100: a file run through the C ABI alone (lfd_engine_bind / lfd_engine_detect) gives, bit for bit, what the
InferencePlan and PostPlan it was exported from give -- on float32, uint8 BGR and NV12 frames, at the capacity and below it, eagerly
and replayed as a CUDA graph, with greedy NMS and Soft-NMS -- with the same launches; examples/lfd_detect prints the rows of
predict_for_single_image; and a call the engine refuses enqueues nothing."""
import ctypes as C
import functools
import os
import subprocess

import numpy as np
import pytest
import torch

import synth
import tl_s
from engine_file import Engine, rows
from helpers import synth_model
from lfd import _native as nat
from lfd._engine import InferencePlan, PostPlan
from lfd.data_pipeline.augmentation import input_transform_of
from lfd.deployment import export_model
from nv12_oracle import nv12_frames, nv12_oracle
from test_input_transform_host import tl_val_pipeline

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROGRAM = os.path.join(ROOT, 'lfd-a-light-and-fast-detector_b200', 'lfd_detect')
LFD_ERR_INVALID, LFD_ERR_CAPACITY = 1, 4
SOFT = dict(type='soft_nms', iou_thr=0.3, method='linear', min_score=0.05)


@functools.lru_cache(maxsize=None)
def model_of(name):
    model = tl_s.synth_model(cls_bias=-1.0)[0] if name == 'TL_S' else synth_model(name, cls_bias=-1.0)[0]
    return model.cuda().eval()


def pipeline_of(name):
    return tl_val_pipeline if name.startswith('TL') else None


def post_of(model, plan, soft):
    own = model._nms_cfg
    model._nms_cfg = dict(SOFT) if soft else dict(type='nms', iou_thr=0.4)
    try:
        return PostPlan(model._post_cfg(plan.N, plan.level_sizes, 0.3, model._nms_cfg['iou_thr'], False), plan.device, model._soft_nms_cfg())
    finally:
        model._nms_cfg = own


def inputs(N, h, w, seed):
    """{format: frames of h x w} on the device: float32 NCHW, uint8 BGR, NV12."""
    nv = nv12_frames(N, h, w, seed)
    g = torch.Generator().manual_seed(seed)
    return {nat.INPUT_F32_NCHW: synth.synth_input(N, h, w, seed=seed).cuda(),
            nat.INPUT_U8_NHWC: torch.randint(0, 256, (N, h, w, 3), generator=g, dtype=torch.uint8).cuda(),
            nat.INPUT_U8_NV12: torch.from_numpy(nv).cuda()}


def same_detections(what, eng, post, N):
    count = eng.count.cpu()
    assert torch.equal(count, post.count.cpu()), (what, count, post.count)
    for i in range(N):
        k = int(count[i])
        assert torch.equal(eng.dets[i, :k], post.dets[i, :k]) and torch.equal(eng.labels[i, :k], post.labels[i, :k]), (what, i)


CASES = [(name, 'bf16', None) for name in ('WIDERFACE_XS', 'WIDERFACE_S', 'WIDERFACE_M', 'WIDERFACE_L', 'TT100K_S', 'TT100K_L', 'TL_L', 'TL_S')] + \
        [('WIDERFACE_S', 'fp16', None), ('TL_L', 'fp16', None), ('WIDERFACE_S', 'bf16', True), ('WIDERFACE_S', 'bf16', False)]


@pytest.mark.parametrize('name,dtype,fuse', CASES)
def test_engine_equals_the_plan(tmp_path, name, dtype, fuse):
    model = model_of(name)
    N, H, W = 2, 256, 320
    plan = InferencePlan(model, N, H, W, torch.device('cuda'), act_dtype=dtype, fuse_stem=fuse, input_transform=input_transform_of(pipeline_of(name)))
    if fuse is not None:
        assert (plan._ops[0]['kind'] == nat.OP_STEM4) == fuse
    for soft in (False, True):
        post = post_of(model, plan, soft)
        path = str(tmp_path / ('m%d.lfd' % soft))
        plan.export(path, post)
        eng = Engine(open(path, 'rb').read())
        nat.check(eng.bind())
        assert eng.num_launches() == plan.num_launches
        for (h, w) in ((H, W), (200, 264), (130, 178)):
            for fmt, x in inputs(N, h, w, seed=h).items():
                what = '%s %s fuse=%s soft=%d %dx%d format %d' % (name, dtype, fuse, soft, h, w, fmt)
                with torch.no_grad():
                    cls, reg = plan.forward(x, use_graph=True, frame_format='nv12' if fmt == nat.INPUT_U8_NV12 else None)
                    cls, reg = cls.clone(), reg.clone()
                model._post_levels(post.cfg, plan.frame_level_sizes)
                post.set_meta([w] * N, [h] * N, [1.0] * N)
                post.run(cls, reg)
                for use_graph in (False, True, True):
                    eng.detect(x, fmt, h, w, use_graph=use_graph)
                    torch.cuda.synchronize()
                    ecls, ereg = eng.frame_outputs(plan.frame_P)
                    assert torch.equal(ecls, cls) and torch.equal(ereg, reg), '%s graph=%d: network outputs differ' % (what, use_graph)
                    same_detections('%s graph=%d' % (what, use_graph), eng, post, N)
                # detections only: the engine's own output region
                eng.detect(x, fmt, h, w, outputs=False)
                same_detections(what + ' without cls/reg', eng, post, N)
        del eng


@pytest.mark.parametrize('name', ['WIDERFACE_S', 'TL_L', 'TL_S'])
@pytest.mark.parametrize('soft', [False, True], ids=['nms', 'soft_nms'])
def test_rows_equal_predict_for_single_image(tmp_path, name, soft):
    model = model_of(name)
    own = model._nms_cfg
    model._nms_cfg = dict(SOFT) if soft else dict(type='nms', iou_thr=0.4)
    try:
        h, w = 184, 248
        path = str(tmp_path / 'm.lfd')
        export_model(model, path, 1, h, w, input_pipeline=pipeline_of(name), classification_threshold=0.3, autotune=False)
        eng = Engine(open(path, 'rb').read())
        nat.check(eng.bind())
        total = 0
        for seed in range(3):
            image = synth.synth_image_u8(h, w, seed=seed)
            want = model.predict_for_single_image(image, pipeline_of(name), classification_threshold=0.3)
            eng.detect(torch.from_numpy(image)[None].cuda(), nat.INPUT_U8_NHWC, h, w)
            got = rows(eng.dets, eng.labels, eng.count)[0]
            assert got == want, (name, soft, seed, len(got), len(want))
            total += len(got)
        assert total > 0
    finally:
        model._nms_cfg = own


def test_autotuned_export_replays_its_bounds(tmp_path):
    """The CTA bounds autotune picks are in the file, and the results do not depend on them (TL_L: no GroupNorm statistics, whose fp64
    atomics would add in another order under another grid)."""
    model = model_of('TL_L')
    N, H, W = 2, 256, 320
    path = str(tmp_path / 'tuned.lfd')
    tuned, post = export_model(model, path, N, H, W, input_pipeline=tl_val_pipeline, autotune=True)
    assert tuned.autotuned
    eng = Engine(open(path, 'rb').read())
    for i, o in enumerate(tuned._op_array):
        assert eng.op(i)[0].max_ctas == o.max_ctas, i
    forced = {b: 16 for b in set(op['branch'] for op in tuned._ops if op['branch'] > 0)}
    tuned.apply_side_ctas(forced)             # a bound that certainly bites, exported as well
    tuned.export(str(tmp_path / 'forced.lfd'), post)
    untuned = InferencePlan(model, N, H, W, torch.device('cuda'), input_transform=input_transform_of(tl_val_pipeline))
    x = inputs(N, H, W, seed=1)[nat.INPUT_U8_NHWC]
    with torch.no_grad():
        cls, reg = (t.clone() for t in untuned.forward(x, use_graph=True))
    for f in ('tuned.lfd', 'forced.lfd'):
        eng = Engine(open(str(tmp_path / f), 'rb').read())
        nat.check(eng.bind())
        assert any(eng.op(i)[0].max_ctas for i in range(eng.desc.n_ops)) or f == 'tuned.lfd'
        eng.detect(x, nat.INPUT_U8_NHWC, H, W)
        torch.cuda.synchronize()
        assert torch.equal(eng.cls, cls) and torch.equal(eng.reg, reg), f


def _cudart_dir():
    """The directory of the cudart this process loaded: lfd_detect runs on it as well."""
    for line in open('/proc/self/maps'):
        if 'libcudart.so' in line:
            return os.path.dirname(line.split()[-1])
    return None


def _program_rows(out):
    frames, cur = [], None
    for line in out.splitlines():
        f = line.split()
        if f[0] == 'frame':
            cur = []
            frames.append(cur)
        else:
            cur.append([int(f[0])] + [float(np.float32(v)) for v in f[1:]])      # %.9g reads back to the float32 it printed
    return frames


@pytest.mark.parametrize('name', ['WIDERFACE_S', 'TL_S'])
def test_c_program_prints_the_rows_of_predict_for_single_image(tmp_path, name):
    assert os.path.exists(PROGRAM), 'build() links examples/lfd_detect.c next to the library'
    model = model_of(name)
    h, w = 184, 248
    path = str(tmp_path / 'm.lfd')
    export_model(model, path, 1, h, w, input_pipeline=pipeline_of(name), classification_threshold=0.3, autotune=False)
    nv = nv12_frames(3, h, w, seed=7)
    images = [synth.synth_image_u8(h, w, seed=s) for s in range(3)] + list(nv12_oracle(nv))
    want = [model.predict_for_single_image(im, pipeline_of(name), classification_threshold=0.3) for im in images]
    assert sum(len(r) for r in want) > 0
    env = dict(os.environ)
    if _cudart_dir():
        env['LD_LIBRARY_PATH'] = _cudart_dir() + os.pathsep + env.get('LD_LIBRARY_PATH', '')
    (tmp_path / 'bgr.raw').write_bytes(np.stack(images[:3]).tobytes())
    (tmp_path / 'nv12.raw').write_bytes(nv.tobytes())
    got = []
    for raw, fmt in (('bgr.raw', 'bgr'), ('nv12.raw', 'nv12')):
        r = subprocess.run([PROGRAM, path, str(tmp_path / raw), str(h), str(w), fmt], capture_output=True, text=True, env=env, timeout=300)
        assert r.returncode == 0, r.stderr
        got += _program_rows(r.stdout)
    assert len(got) == len(want)
    for i, (g, wt) in enumerate(zip(got, want)):
        assert g == wt, (name, i, len(g), len(wt))


def test_errors_launch_nothing(tmp_path):
    """Each refused call returns its code before anything reaches the device: every caller buffer keeps its bytes."""
    model = model_of('WIDERFACE_S')
    path = str(tmp_path / 'm.lfd')
    export_model(model, path, 2, 96, 160, autotune=False)
    data = open(path, 'rb').read()
    eng = Engine(data, poison=0xff)
    x = torch.zeros((2, 96, 160, 3), dtype=torch.uint8, device='cuda')
    lib = nat.lib()

    def untouched(call, want):
        for t in (eng.workspace, eng.post_ws, eng.dets, eng.labels, eng.count, eng.cls, eng.reg):
            t.view(torch.uint8).fill_(0xff)
        torch.cuda.synchronize()
        rc = call()
        torch.cuda.synchronize()
        assert rc == want, (rc, lib.lfd_last_error())
        for t in (eng.weights, eng.workspace, eng.post_ws, eng.dets, eng.labels, eng.count, eng.cls, eng.reg):
            assert bool((t.view(torch.uint8) == 0xff).all())
        return lib.lfd_last_error().decode()

    untouched(lambda: eng.detect_raw(x, nat.INPUT_U8_NHWC, 96, 160), LFD_ERR_INVALID)             # not bound
    assert 'workspace' in untouched(lambda: eng.bind(workspace_bytes=eng.desc.workspace_bytes - 256), LFD_ERR_CAPACITY)
    with torch.cuda.device(0):
        assert lib.lfd_engine_bind(eng.handle, nat.ptr(eng.weights), eng.desc.weights_bytes - 1, nat.ptr(eng.workspace), eng.desc.workspace_bytes,
                                   nat.ptr(eng.post_ws), eng.desc.post_workspace_bytes, nat.stream_ptr()) == LFD_ERR_CAPACITY
        assert lib.lfd_engine_bind(eng.handle, nat.ptr(eng.weights), eng.desc.weights_bytes, nat.ptr(eng.workspace), eng.desc.workspace_bytes,
                                   nat.ptr(eng.post_ws), eng.desc.post_workspace_bytes - 1, nat.stream_ptr()) == LFD_ERR_CAPACITY
        # buffers not aligned to 256 bytes (what cudaMalloc returns)
        big = torch.full((eng.desc.weights_bytes + 256,), 0xff, dtype=torch.uint8, device='cuda')
        for shift in (16, 128):
            assert lib.lfd_engine_bind(eng.handle, big.data_ptr() + shift, eng.desc.weights_bytes, nat.ptr(eng.workspace), eng.desc.workspace_bytes,
                                       nat.ptr(eng.post_ws), eng.desc.post_workspace_bytes, nat.stream_ptr()) == LFD_ERR_INVALID
            assert 'aligned' in lib.lfd_last_error().decode()
    torch.cuda.synchronize()
    assert bool((eng.weights == 0xff).all()) and bool((big == 0xff).all())
    nat.check(eng.bind())
    torch.cuda.synchronize()
    eng.weights.fill_(0xff)          # (the weights are the engine's now; refused calls must not read or write any buffer)
    nv = torch.zeros((2, 144, 160), dtype=torch.uint8, device='cuda')
    for h, w in ((97, 160), (96, 161), (0, 160), (96, 0)):
        assert 'capacity' in untouched(lambda: eng.detect_raw(x, nat.INPUT_U8_NHWC, h, w), LFD_ERR_INVALID)
    for h, w in ((63, 100), (64, 101)):
        assert 'even' in untouched(lambda: eng.detect_raw(nv, nat.INPUT_U8_NV12, h, w), LFD_ERR_INVALID)
    for fmt in (3, -1):
        untouched(lambda: eng.detect_raw(x, fmt, 96, 160), LFD_ERR_INVALID)
    untouched(lambda: lib.lfd_engine_detect(eng.handle, nat.ptr(x), nat.INPUT_U8_NHWC, 96, 160, None, nat.ptr(eng.labels), nat.ptr(eng.count),
                                            None, None, 1, nat.stream_ptr()), LFD_ERR_INVALID)


def test_a_call_on_another_stream_writes_the_image_sizes_again(tmp_path):
    """The per-image width / height the post-process reads are written on the stream of the call that writes them: a call of the same size
    on another stream writes them again, so its post-process is ordered after them (the region is overwritten here to show it)."""
    model = model_of('TL_L')
    path = str(tmp_path / 'm.lfd')
    export_model(model, path, 2, 256, 320, input_pipeline=tl_val_pipeline, classification_threshold=0.3, autotune=False)
    eng = Engine(open(path, 'rb').read())
    nat.check(eng.bind())
    x = inputs(2, 256, 320, seed=3)[nat.INPUT_U8_NHWC]
    eng.detect(x, nat.INPUT_U8_NHWC, 256, 320)
    torch.cuda.synchronize()
    want = [t.clone() for t in (eng.dets, eng.labels, eng.count)]
    assert int(want[2][:2].sum()) > 0
    side = torch.cuda.Stream()
    eng.post_ws.fill_(0xff)
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        eng.detect(x, nat.INPUT_U8_NHWC, 256, 320)
    side.synchronize()
    c = want[2]
    assert torch.equal(eng.count, c)
    for i in range(2):
        k = int(c[i])
        assert torch.equal(eng.dets[i, :k], want[0][i, :k]) and torch.equal(eng.labels[i, :k], want[1][i, :k])
