# -*- coding: utf-8 -*-
"""Gray (1-channel) models on the H100.  The defining property (tests/gray_models.py): a gray model with stem weights W1 gives, bit for
bit, what its 3-channel twin with stem weights [W1, 0, 0] gives on frames whose channel 0 is the gray frame (uint8: bytes 1 and 2 random;
float32: planes 1 and 2 zero).  Checked per stem op and per plan; the gray stem against float64; NV12 frames against their Y plane; one
training step against the twin's and the stem weight gradient against float64; the public paths; and the SIMT cross-check."""
import ctypes as C
import functools

import numpy as np
import pytest
import torch

import synth
from engine_file import Engine, rows
from gpu_ops import DTYPES, assert_faithful, conv_out, ref_conv64, run_stem0
from gpu_train_ops import Workspace, assert_within, cdiv, make_top, run_top, stem_wgrad_grid
from gray_models import gray_pair, twin_f32, twin_u8
from helpers import misaligned, same_bits
from lfd import _native as nat
from lfd._engine import InferencePlan
from lfd.data_pipeline.augmentation import Compose, Normalize, input_transform_of
from nv12_oracle import nv12_frames
from test_gpu_nv12 import compare, snapshot

pytestmark = pytest.mark.gpu

LFD_ERR_INVALID, LFD_ERR_UNSUPPORTED = 1, 3
GRAY_NORM = Compose([Normalize(mean=(0.4,), std=(0.2,), max_pixel_value=255.0, p=1.0)])     # one constant
TRANSFORMS = {'zero-fields': None, 'one-constant': input_transform_of(GRAY_NORM, channels=1)}


def gray_u8(n, h, w, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (n, h, w), generator=g, dtype=torch.uint8).cuda()


def gray_f32(n, h, w, seed=0):
    return synth.synth_input(n, h, w, seed=seed)[:, :1].contiguous().cuda()


def luma(nv):
    """The Y planes of NV12 frames [N, 3h/2, w] -> uint8 [N, h, w] (cv2.COLOR_YUV2GRAY_NV12)."""
    h = nv.shape[1] // 3 * 2
    return nv[:, :h].contiguous()


# ------------------------------------------------------------------------------------------------------------------ single ops
def weights(cout):
    g = torch.Generator().manual_seed(cout)
    w1 = torch.randn((cout, 1, 3, 3), generator=g) * 0.1
    shift = torch.randn(cout, generator=g) * 0.1
    tail = (torch.randn((cout, cout, 1, 1), generator=g) * 0.1, torch.ones(cout), torch.randn(cout, generator=g) * 0.1, True)
    return w1, torch.cat([w1, torch.zeros(cout, 2, 3, 3)], 1), shift, tail


SIZES = [(38, 44), (40, 42), (37, 41)]          # W = 0 / 2 (mod 4); odd (no NV12)


@pytest.mark.parametrize('name', sorted(TRANSFORMS))
@pytest.mark.parametrize('dtype', ['bf16', 'fp16'])
@pytest.mark.parametrize('cout', [16, 32, 48, 64])
def test_stem0_gray_equals_its_twin(cout, dtype, name):
    """STEM0 (every width, with and without the fused tail, default grid and 3 CTAs; the 48-wide one is conv_umma_c48_kernel) on uint8,
    float32 and NV12 gray frames: bit for bit the 3-channel op with weights [W1, 0, 0] on the twin frames; the SIMT kernel likewise."""
    transform = TRANSFORMS[name]
    w1, w3, shift, tail = weights(cout)
    for h, wd in SIZES:
        g8 = gray_u8(2, h, wd, seed=h * wd + cout)
        gf = gray_f32(2, h, wd, seed=cout)
        cases = [(g8, nat.INPUT_U8_NHWC, twin_u8(g8, seed=cout), nat.INPUT_U8_NHWC), (gf, nat.INPUT_F32_NCHW, twin_f32(gf), nat.INPUT_F32_NCHW)]
        if h % 2 == 0 and wd % 2 == 0:
            nv = torch.from_numpy(nv12_frames(2, h, wd, seed=cout)).cuda()
            cases.append((nv, nat.INPUT_U8_NV12, twin_u8(luma(nv), seed=cout + 1), nat.INPUT_U8_NHWC))
        for xg, fg, xt, ft in cases:
            for t in (None, tail):
                for ctas in (0, 3):
                    what = 'stem0 Cout=%d%s %s %s fmt=%d %dx%d max_ctas=%d' % (cout, ' + tail' if t else '', dtype, name, fg, h, wd, ctas)
                    same_bits(run_stem0(xg, fg, w1, shift, cin=1, tail=t, transform=transform, dtype=dtype, max_ctas=ctas)[0],
                              run_stem0(xt, ft, w3, shift, tail=t, transform=transform, dtype=dtype, max_ctas=ctas)[0], what)
            same_bits(run_stem0(xg, fg, w1, shift, cin=1, transform=transform, dtype=dtype, impl=nat.CONV_SIMT)[0],
                      run_stem0(xt, ft, w3, shift, transform=transform, dtype=dtype, impl=nat.CONV_SIMT)[0],
                      'SIMT stem0 Cout=%d %s %s fmt=%d %dx%d' % (cout, dtype, name, fg, h, wd))


@pytest.mark.parametrize('dtype', ['bf16', 'fp16'])
@pytest.mark.parametrize('cout', [16, 32, 48, 64])
def test_gray_stem0_is_a_faithful_rounding_of_float64(cout, dtype):
    """The gray stem against a float64 conv of the same 16-bit-rounded input (byte - mean) * scale (or the fp32 plane) and weights:
    within one 16-bit spacing plus the fp32 accumulation bound, as test_gpu_input_transform.py states it for BGR."""
    rnd = DTYPES[dtype][1]
    w1, _, shift, _ = weights(cout)
    t = TRANSFORMS['one-constant']
    for h, wd in SIZES:
        g8 = gray_u8(2, h, wd, seed=h + wd)
        gf = gray_f32(2, h, wd, seed=h)
        x8 = rnd((g8.cpu().float() - t.mean[0]) * t.scale[0])[..., None]           # fp32: one subtract, one multiply, then R0
        xf = rnd(gf.cpu().permute(0, 2, 3, 1))
        for x, inp, fmt in ((x8, g8, nat.INPUT_U8_NHWC), (xf, gf, nat.INPUT_F32_NCHW)):
            ref, S, K = ref_conv64(x, w1, torch.ones(cout), shift, 2, True, dtype=dtype)
            for impl in (nat.CONV_UMMA, nat.CONV_SIMT):
                out, _ = run_stem0(inp, fmt, w1, shift, cin=1, transform=t, dtype=dtype, impl=impl)
                assert_faithful(out.float(), ref, S, K, dtype, 'gray stem0 Cout=%d %s fmt=%d impl=%d %dx%d' % (cout, dtype, fmt, impl, h, wd))


# ------------------------------------------------------------------------------------------------------------------ plans
@functools.lru_cache(maxsize=None)
def pair_of(name):
    gray, twin = gray_pair(name)
    return gray.cuda().eval(), twin.cuda().eval()


def plan_pair(name, H, W, dtype, fuse, transform):
    gray, twin = pair_of(name)
    return [InferencePlan(m, 2, H, W, torch.device('cuda'), act_dtype=dtype, fuse_stem=fuse, input_transform=transform, reuse=False)
            for m in (gray, twin)]


PLANS = [('WIDERFACE_S', True, 'bf16'), ('WIDERFACE_S', True, 'fp16'), ('WIDERFACE_S', False, 'bf16'), ('WIDERFACE_L', None, 'bf16'),
         ('TL_S', None, 'bf16'), ('TL_S', None, 'fp16')]
H, W = 200, 264


@pytest.mark.parametrize('cfg,fuse,dtype', PLANS)
def test_whole_plans_equal_their_twins(cfg, fuse, dtype):
    """Whole plans of WIDERFACE-S (fused stem: the word loader at an aligned capacity of W % 4 == 0 and below it with an odd width, the
    byte loader on a misaligned frame; and unfused), WIDERFACE-L and TL_S (the 48-wide stem): uint8, float32 and NV12 gray frames at the
    capacity and below it, eager and with the CUDA graph, every conv output and the heads against the twin's."""
    transform = TRANSFORMS['one-constant']
    gp, tp = plan_pair(cfg, H, W, dtype, fuse, transform)
    assert gp._ops[0]['Cin'] == 1 and (gp._ops[0]['kind'] == nat.OP_STEM4) == bool(fuse)
    for h, w in ((H, W), (198, 259), (196, 258)):
        g8 = gray_u8(2, h, w, seed=h + w)
        gf = gray_f32(2, h, w, seed=w)
        cases = [('u8', g8, None, twin_u8(g8, seed=3)), ('f32', gf, None, twin_f32(gf)), ('u8 [N,h,w,1]', g8[..., None], None, twin_u8(g8, seed=4))]
        if h % 2 == 0 and w % 2 == 0:
            nv = torch.from_numpy(nv12_frames(2, h, w, seed=h)).cuda()
            cases.append(('nv12', nv, 'nv12', twin_u8(luma(nv), seed=5)))
        if (h, w) == (H, W) and fuse:
            cases.append(('u8 misaligned', misaligned(g8), None, twin_u8(g8, seed=3)))
        for tag, xg, fmt, xt in cases:
            for graph in ((False, True) if (h, w) == (H, W) else (True,)):
                what = '%s fuse=%s %s %s %dx%d graph=%d' % (cfg, fuse, dtype, tag, h, w, graph)
                compare(what, gp, snapshot(gp, xg, fmt, graph, h, w), snapshot(tp, xt, None, graph, h, w))


@pytest.mark.parametrize('dtype', ['bf16', 'fp16'])
def test_fused_gray_stem_equals_the_unfused_gray_stem(dtype):
    """STEM4 rounds every intermediate as the STEM0 + CONV pair does: the gray fused stem's stem3 map bit for bit against the same gray
    model's two-launch stem (whose STEM0 the float64 test above pins), on both loaders and every input format."""
    transform = TRANSFORMS['zero-fields']
    gray, _ = pair_of('WIDERFACE_S')
    for h, w in ((H, W), (H, W - 2)):
        fused, pair = [InferencePlan(gray, 2, h, w, torch.device('cuda'), act_dtype=dtype, fuse_stem=f, input_transform=transform, reuse=False)
                       for f in (True, False)]
        g8 = gray_u8(2, h, w, seed=w)
        nv = torch.from_numpy(nv12_frames(2, h, w, seed=w)).cuda()
        for tag, x, fmt in (('u8', g8, None), ('u8 misaligned', misaligned(g8), None), ('f32', gray_f32(2, h, w, seed=1), None), ('nv12', nv, 'nv12')):
            a = snapshot(fused, x, fmt, False, h, w)[0]['stem3']
            b = snapshot(pair, x, fmt, False, h, w)[0]['stem3']
            same_bits(a, b, 'gray stem4 vs stem0 + conv %s %s %dx%d' % (dtype, tag, h, w))


def test_nv12_frames_give_what_their_luma_gives():
    """A gray model on NV12 frames = the same model on cv2.cvtColor(f, COLOR_YUV2GRAY_NV12), bit for bit; rewriting every UV byte
    changes nothing."""
    import cv2
    for cfg, fuse in (('WIDERFACE_S', True), ('TL_S', None)):
        gray, _ = pair_of(cfg)
        plan = InferencePlan(gray, 2, H, W, torch.device('cuda'), fuse_stem=fuse, input_transform=TRANSFORMS['one-constant'], reuse=False)
        for h, w in ((H, W), (196, 258)):
            nv_np = nv12_frames(2, h, w, seed=h)
            y = torch.from_numpy(np.stack([cv2.cvtColor(f, cv2.COLOR_YUV2GRAY_NV12) for f in nv_np])).cuda()
            assert torch.equal(y, luma(torch.from_numpy(nv_np)).cuda())
            nv = torch.from_numpy(nv_np).cuda()
            for graph in (False, True):
                ref = snapshot(plan, y, None, graph, h, w)
                compare('%s %dx%d graph=%d' % (cfg, h, w, graph), plan, snapshot(plan, nv, 'nv12', graph, h, w), ref)
                other = nv.clone()
                other[:, h:] = torch.randint(0, 256, other[:, h:].shape, dtype=torch.uint8, device='cuda')
                compare('%s %dx%d graph=%d, other UV' % (cfg, h, w, graph), plan, snapshot(plan, other, 'nv12', graph, h, w), ref)


# ------------------------------------------------------------------------------------------------------------------ training
def _step(model, x, ann):
    out = model(x)
    ld = model.get_loss(out, ann)
    model._flat_parameters.grad.zero_()
    ld['loss'].backward()
    torch.cuda.synchronize()
    return float(ld['loss'].detach()), {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None}


@pytest.mark.parametrize('fmt', ['f32', 'u8'])
@pytest.mark.parametrize('frozen', [None, 1])
def test_training_step_gray_equals_twin(fmt, frozen):
    """One native step of the gray model and of its twin (float32: planes 1 and 2 zero; uint8: bytes 1 and 2 random): the losses, every
    gradient outside the stem conv, and the gray stem gradient = channel 0 of the twin's, within the run-to-run tolerance of the fp32
    atomics (test_gpu_input_transform.py).  With frozen_stages=1 the frozen prefix runs the gray inference stem."""
    n, h, w = 2, 128, 160
    ann = synth.synth_annotations(n, h, w, 1, seed=5)
    gray, twin = gray_pair('WIDERFACE_L', cls_bias=-2.0)
    xs = {}
    if fmt == 'f32':
        xs['gray'] = gray_f32(n, h, w, seed=7)
        xs['twin'] = twin_f32(xs['gray'])
    else:
        xs['gray'] = gray_u8(n, h, w, seed=7)
        xs['twin'] = twin_u8(xs['gray'], seed=8)
    res = {}
    for key, m in (('gray', gray), ('twin', twin)):
        if frozen:
            m._backbone._frozen_stages = frozen
        m.cuda().train()
        m.input_transform = TRANSFORMS['one-constant']
        res[key] = _step(m, xs[key], ann)
    (lg, gg), (lt, gt) = res['gray'], res['twin']
    assert abs(lg - lt) <= 1e-3 * abs(lt), (lg, lt)
    assert sorted(gg) == sorted(gt)
    stem = '_backbone._stem.0.weight'
    if stem in gt:
        gt[stem] = gt[stem][:, :1]
    top = max(float(t.abs().max()) for t in gt.values())
    for name in gt:
        a, b = gg[name], gt[name]
        assert a.shape == b.shape, name
        assert float((a - b).abs().max()) <= 1e-3 * top, (name, float((a - b).abs().max()), top)
    if not frozen:
        assert float(gg[stem].abs().max()) > 0


@pytest.mark.parametrize('frozen', [None, 1])
def test_gray_training_loss_matches_aten(frozen):
    """The native step of the gray model against the same module graph evaluated by ATen in fp32 (tests/aten_train_reference.py): the
    loss within the bound smoke() uses; with frozen_stages=1 the gray stem runs on the inference kernels of the frozen prefix."""
    from aten_train_reference import train_forward as aten_forward
    from oracle import lfd_oracle as orc
    n, h, w = 2, 128, 160
    x = gray_f32(n, h, w, seed=11)
    ann = synth.synth_annotations(n, h, w, 1, seed=3)
    gray, _ = gray_pair('WIDERFACE_L', cls_bias=-2.0)
    ref, _ = gray_pair('WIDERFACE_L', cls_bias=-2.0)
    for m in (gray, ref):
        if frozen:
            m._backbone._frozen_stages = frozen
        m.train()
    gray.cuda()
    ld = gray.get_loss(gray(x), ann)
    rcls, rreg = aten_forward(ref, x.cpu())
    sizes = [ref._head_indexes_to_feature_map_sizes[i] for i in range(len(ref._head_indexes_to_feature_map_sizes))]
    want = float(orc.get_loss(orc.CONFIGS['WIDERFACE_L'], rcls, rreg, sizes, ann)['loss'])
    assert abs(ld['loss_values']['loss'] - want) < 3e-2 * abs(want), (ld['loss_values'], want)


@pytest.mark.parametrize('path', ['umma', 'simt'])
@pytest.mark.parametrize('fmt', ['u8', 'f32'])
@pytest.mark.parametrize('cout', [16, 32, 64])
def test_gray_stem_weight_gradient_matches_fp64(cout, fmt, path):
    """LFD_TOP_WGRAD_STEM with Cin = 1 (im2col X9 padded to 32 columns + the tensor-core wgrad, or the SIMT kernel): the 9 staging rows
    against float64 conv2d_weight of the normalised, rounded image, the rows past them zero."""
    N, Hs, Ws = 2, 75, 131
    Ho, Wo = conv_out(Hs, 3, 2), conv_out(Ws, 3, 2)
    sms = nat.lib().lfd_device_sm_count()
    blocks, n_seg = stem_wgrad_grid(N, Ho, Wo, sms)
    g = torch.Generator().manual_seed(cout + (path == 'simt') * 7)
    t = TRANSFORMS['one-constant']
    if fmt == 'u8':
        img = torch.randint(0, 256, (N, Hs, Ws), generator=g, dtype=torch.uint8)
        x = DTYPES['bf16'][1]((img.float() - t.mean[0]) * t.scale[0])[..., None]
    else:
        img = torch.randn((N, 1, Hs, Ws), generator=g)
        x = DTYPES['bf16'][1](img.permute(0, 2, 3, 1))
    dz = DTYPES['bf16'][1](torch.randn((N, Ho, Wo, cout), generator=g))
    ws = Workspace('cuda')
    ws.add('dz', dz.to(torch.bfloat16))
    ws.add('ds', shape=(32, cout), dtype=torch.float32)
    ws.add('x27', shape=(N, Ho, Wo, 32), dtype=torch.bfloat16)
    ws.finalize()
    offs = {1: ws.off('dz'), 5: ws.off('ds')}
    if path == 'umma':
        offs[0] = ws.off('x27')
    top = make_top(nat.TOP_WGRAD_STEM, N=N, H=Hs, W=Ws, Cin=1, Ho=Ho, Wo=Wo, Cout=cout, ksize=3, stride=2,
                   impl=nat.WGRAD_SIMT if path == 'simt' else nat.WGRAD_UMMA, off=offs)
    nat.set_input_transform(top, t)
    run_top(top, ws, input=img.cuda().contiguous(), fmt=nat.INPUT_U8_NHWC if fmt == 'u8' else nat.INPUT_F32_NCHW)
    stage = ws.get('ds').cpu()
    assert float(stage[9:].abs().max()) == 0.0
    if path == 'umma':
        assert float(ws.get('x27').float()[..., 9:].abs().max()) == 0.0
    got = stage[:9].reshape(9, 1, cout).permute(2, 1, 0).reshape(cout, 1, 3, 3)
    xd, dzd = x.double().permute(0, 3, 1, 2), dz.double().permute(0, 3, 1, 2)
    ref = torch.nn.grad.conv2d_weight(xd, (cout, 1, 3, 3), dzd, stride=2, padding=1)
    S = torch.nn.grad.conv2d_weight(xd.abs(), (cout, 1, 3, 3), dzd.abs(), stride=2, padding=1)
    K = cdiv(n_seg, blocks) * 64 + blocks if path == 'simt' else N * Ho * Wo + 4 * sms
    assert_within(got, ref, S, K, 'gray stem wgrad %d %s %s' % (cout, path, fmt))


# ------------------------------------------------------------------------------------------------------------------ public paths
def test_predict_for_single_image_takes_a_2d_image():
    """A 2-D uint8 image (cv2.imread(path, IMREAD_UNCHANGED) of a gray file) gives the rows of the host path: model(x) on the float32
    [1,1,H,W] tensor of the normalised image, then the same post-process.  A 3-channel image raises."""
    gray, _ = pair_of('TL_S')
    image = gray_u8(1, 200, 266, seed=3)[0].cpu().numpy()
    rows_fused = gray.predict_for_single_image(image, GRAY_NORM, classification_threshold=0.3)
    m, s = GRAY_NORM.transforms[0].constants()
    xf = torch.from_numpy((image.astype(np.float32) - m) * s)[None, None].cuda()
    with torch.no_grad():
        out = gray(xf)
    dets, labels, _, count, overflow = gray.detect(out, [200], [266], [1.0], 0.3, gray._nms_cfg['iou_thr'], False)
    host = gray._rows(dets, labels, count, overflow, gray.max_detections_per_image)[0]
    assert len(rows_fused) > 0 and rows_fused == host
    assert gray.predict_for_single_image(image[..., None], GRAY_NORM, classification_threshold=0.3) == rows_fused
    with pytest.raises(ValueError):
        gray.predict_for_single_image(np.stack([image] * 3, -1), GRAY_NORM)
    with pytest.raises(ValueError):
        gray.predict_for_single_image(image, Compose([Normalize(mean=(0.4, 0.5, 0.4), std=(0.2,) * 3, max_pixel_value=255.0, p=1.0)]))


@pytest.mark.parametrize('fmt', ['gray', 'nv12'])
def test_streaming_detector_gives_what_the_synchronous_path_gives(fmt):
    from lfd.pipeline import StreamingDetector
    gray, _ = pair_of('TL_S')
    n, h, w = 2, 232, 328
    det = StreamingDetector(gray, n, h, w, 0.3, 0.3, max_out=512, input_pipeline=GRAY_NORM, frame_format=fmt)
    assert det.h2d_bytes == n * h * w * (1 if fmt == 'gray' else 3) // (1 if fmt == 'gray' else 2)
    batches = []
    for s in range(3):
        nv = nv12_frames(n, h, w, seed=s)
        batches.append(torch.from_numpy(nv if fmt == 'nv12' else np.ascontiguousarray(nv[:, :h])).pin_memory())
    gray.set_input_transform(GRAY_NORM)
    try:
        total = 0
        for b in batches:
            d, labels, counts = det.infer(b)
            y = b[:, :h].contiguous().cuda()
            with torch.no_grad():
                out = gray(y)
            dets, lab, _, count, overflow = gray.detect(out, [h] * n, [w] * n, [1.0] * n, 0.3, 0.3)
            for j in range(n):
                k = int(count[j])
                total += k
                assert k == int(counts[j]) and torch.equal(dets[j, :k].cpu(), d[j, :k]) and torch.equal(lab[j, :k].cpu(), labels[j, :k])
        assert total > 0
    finally:
        gray.set_input_transform(None)
    with pytest.raises(ValueError):
        StreamingDetector(gray, n, h, w, 0.3, 0.3, frame_format='bgr')


def test_exported_gray_model_detects_what_predict_gives(tmp_path):
    from lfd.deployment import export_model
    gray, _ = pair_of('TL_S')
    h, w = 184, 248
    path = str(tmp_path / 'gray.lfd')
    export_model(gray, path, 1, h, w, input_pipeline=GRAY_NORM, classification_threshold=0.3, autotune=False)
    eng = Engine(open(path, 'rb').read())
    assert eng.op(0)[0].Cin == 1
    nat.check(eng.bind())
    total = 0
    for seed in range(3):
        image = gray_u8(1, h, w, seed=seed)
        want = gray.predict_for_single_image(image[0].cpu().numpy(), GRAY_NORM, classification_threshold=0.3)
        eng.detect(image, nat.INPUT_U8_NHWC, h, w)
        got = rows(eng.dets, eng.labels, eng.count)[0]
        assert got == want, (seed, len(got), len(want))
        total += len(got)
        nv = torch.from_numpy(nv12_frames(1, h, w, seed=seed)).cuda()
        eng.detect(nv, nat.INPUT_U8_NV12, h, w)
        assert rows(eng.dets, eng.labels, eng.count)[0] == gray.predict_for_single_image(luma(nv)[0].cpu().numpy(), GRAY_NORM,
                                                                                         classification_threshold=0.3)
    assert total > 0


def test_c_program_runs_a_gray_file(tmp_path):
    """examples/lfd_detect.c sizes uint8 frames by op 0's Cin: gray frames (and NV12 ones) of a gray model file print the rows of
    predict_for_single_image."""
    import os
    import subprocess
    from lfd.deployment import export_model
    from test_gpu_engine_file import PROGRAM, _cudart_dir, _program_rows
    gray, _ = pair_of('TL_S')
    h, w = 184, 248
    path = str(tmp_path / 'gray.lfd')
    export_model(gray, path, 1, h, w, input_pipeline=GRAY_NORM, classification_threshold=0.3, autotune=False)
    nv = nv12_frames(3, h, w, seed=7)
    images = [gray_u8(1, h, w, seed=s)[0].cpu().numpy() for s in range(3)] + [f[:h] for f in nv]
    want = [gray.predict_for_single_image(im, GRAY_NORM, classification_threshold=0.3) for im in images]
    assert sum(len(r) for r in want) > 0
    env = dict(os.environ)
    if _cudart_dir():
        env['LD_LIBRARY_PATH'] = _cudart_dir() + os.pathsep + env.get('LD_LIBRARY_PATH', '')
    (tmp_path / 'gray.raw').write_bytes(np.stack(images[:3]).tobytes())
    (tmp_path / 'nv12.raw').write_bytes(nv.tobytes())
    got = []
    for raw, fmt in (('gray.raw', []), ('gray.raw', ['gray']), ('nv12.raw', ['nv12'])):
        r = subprocess.run([PROGRAM, path, str(tmp_path / raw), str(h), str(w)] + fmt, capture_output=True, text=True, env=env, timeout=300)
        assert r.returncode == 0, r.stderr
        got.append(_program_rows(r.stdout))
    assert got[0] == got[1] and got[0] + got[2] == want
    r = subprocess.run([PROGRAM, path, str(tmp_path / 'gray.raw'), str(h), str(w), 'bgr'], capture_output=True, text=True, env=env, timeout=300)
    assert r.returncode != 0


def test_refusals_launch_nothing():
    """A gray image op with in_swap_rb or unequal constants (LFD_ERR_INVALID), a channel count other than 1 and 3 (UNSUPPORTED), NV12 on
    a training op (UNSUPPORTED), and frames of the wrong kind on a gray plan: refused before anything is enqueued."""
    from lfd.data_pipeline.augmentation import InputTransform
    w1, w3, shift, _ = weights(16)
    x = gray_u8(2, 40, 44)
    for tr, cin, want in ((InputTransform(True, (1.0,) * 3, (0.5,) * 3), 1, LFD_ERR_INVALID),
                          (InputTransform(False, (1.0, 2.0, 1.0), (0.5,) * 3), 1, LFD_ERR_INVALID),
                          (InputTransform(False, (1.0,) * 3, (0.5, 0.5, 0.25)), 1, LFD_ERR_INVALID),
                          (None, 2, LFD_ERR_UNSUPPORTED), (None, 4, LFD_ERR_UNSUPPORTED)):
        for impl in (nat.CONV_UMMA, nat.CONV_SIMT):
            rc, ws = run_stem0(x, nat.INPUT_U8_NHWC, w1, shift, cin=cin, transform=tr, impl=impl, raw_rc=True)
            assert rc == want and bool((ws == 0xff).all()), (tr, cin, impl, rc)
            if cin == 2:
                assert '1' in nat.lib().lfd_last_error().decode() and '3' in nat.lib().lfd_last_error().decode()
    # a training op: NV12 stays refused, and WGRAD_STEM takes 1 or 3 channels only
    ws = Workspace('cuda')
    ws.add('dz', shape=(2, 20, 22, 16), dtype=torch.bfloat16)
    ws.add('ds', shape=(32, 16), dtype=torch.float32)
    ws.finalize()
    ws.buf.fill_(0xff)
    for cin, fmt, want in ((1, nat.INPUT_U8_NV12, LFD_ERR_UNSUPPORTED), (2, nat.INPUT_U8_NHWC, LFD_ERR_UNSUPPORTED)):
        top = make_top(nat.TOP_WGRAD_STEM, N=2, H=40, W=44, Cin=cin, Ho=20, Wo=22, Cout=16, ksize=3, stride=2, impl=nat.WGRAD_SIMT,
                       off={1: ws.off('dz'), 5: ws.off('ds')})
        torch.cuda.synchronize()
        rc = nat.lib().lfd_run_top(C.byref(top), nat.ptr(x), fmt, nat.ptr(ws.buf), nat.stream_ptr())
        torch.cuda.synchronize()
        assert rc == want and bool((ws.buf == 0xff).all()), (cin, fmt, rc)
    # a gray plan refuses BGR / 3-plane frames in Python, before any launch
    gray, _ = pair_of('TL_S')
    plan = InferencePlan(gray, 2, 96, 160, torch.device('cuda'))
    plan.workspace.fill_(0xff)
    for bad in (torch.zeros((2, 96, 160, 3), dtype=torch.uint8, device='cuda'), torch.zeros((2, 3, 96, 160), device='cuda'),
                torch.zeros((2, 96, 160, 2), dtype=torch.uint8, device='cuda')):
        with pytest.raises(ValueError):
            plan.forward(bad)
    torch.cuda.synchronize()
    assert bool((plan.workspace == 0xff).all())


# ------------------------------------------------------------------------------------------------------------------ SIMT cross-check
@pytest.mark.parametrize('impl', [nat.CONV_UMMA, nat.CONV_SIMT], ids=['umma', 'simt'])
def test_every_layer_within_one_bf16_ulp_teacher_forced(impl):
    """The gray TL_S plan, on the wgmma kernels and on the SIMT cross-check: each conv layer, evaluated in fp32 on the CPU from the inputs
    the CUDA path itself produced (the gray stem from the bf16-rounded frame [N,1,H,W]), matches the stored output to 1 bf16 ulp (as
    test_gpu_tl_s.py checks the BGR model)."""
    from gpu_ops import assert_bf16_close, bf16r, ref_conv
    from helpers import rel_err
    gray, _ = pair_of('TL_S')
    x = gray_f32(2, 168, 232, seed=2)
    plan = InferencePlan(gray, 2, 168, 232, torch.device('cuda'), impl, reuse=False)
    with torch.no_grad():
        plan.forward(x, use_graph=False)
    torch.cuda.synchronize()
    n_conv = 0
    for op in plan._ops:
        if op['kind'] not in (nat.OP_STEM0, nat.OP_CONV):
            continue
        conv, norm = op['modules']
        scale, shift = InferencePlan._fold(conv, norm)
        src = bf16r(x.cpu()).permute(0, 2, 3, 1) if op['kind'] == nat.OP_STEM0 else plan.tensor(op['inp'])
        res = plan.tensor(op['res']) if op.get('res') is not None else None
        if op['kind'] == nat.OP_STEM0:
            assert op['Cin'] == 1 and conv.in_channels == 1
        n_conv += 1
        if not op.get('tail_cout'):
            ref = ref_conv(src, conv.weight.detach().cpu(), scale, shift, op['stride'], bool(op['relu']), res=res)
            assert_bf16_close(plan.tensor(op['out']), ref, 'conv %s' % op['out'])
            if op.get('ds_cout'):
                sconv, snorm = op['ds_modules']
                sscale, sshift = InferencePlan._fold(sconv, snorm)
                assert_bf16_close(plan.tensor(op['out2']), ref_conv(src, sconv.weight.detach().cpu(), sscale, sshift, 2, False), op['out2'])
        else:
            conv2, norm2 = op['tail_modules']
            scale2, shift2 = InferencePlan._fold(conv2, norm2)
            mid = bf16r(ref_conv(src, conv.weight.detach().cpu(), scale, shift, op['stride'], bool(op['relu'])))
            ref = ref_conv(mid, conv2.weight.detach().cpu(), scale2, shift2, 1, bool(op['tail_relu']), res=res)
            got = plan.tensor(op['out']).float().cpu()
            tol = ref.abs() * 2.0 ** -7 + 2e-3 * float(ref.abs().max())   # 1-ulp flips of the in-kernel intermediate
            assert bool(((got - ref).abs() <= tol).all()), ('fused tail', op['out'], float((got - ref).abs().max()))
            assert rel_err(got, ref)[1] < 3e-3
    assert n_conv > 10
