# -*- coding: utf-8 -*-
"""BGR -> RGB and any Normalize inside the stem kernels' uint8 path.  The defining property: the 16-bit value a loader builds for a
pixel is the rounding of the fp32 number the host pipeline produces, so every op and every plan gives, on a uint8 frame under a
transform, exactly what it gives on the float32 NCHW tensor the host stand-ins make of that frame."""
import ctypes as C
import functools

import numpy as np
import pytest
import torch

import synth
import tl_s
from gpu_ops import DTYPES, conv_out
from helpers import synth_model
from lfd import _native as nat
from lfd._engine import InferencePlan, fold_scale, pack_conv_weight, pack_stem_weight
from lfd.data_pipeline.augmentation import (BGR2RGB, Compose, input_transform_of, simple_widerface_val_pipeline, standard_normalize,
                                            typical_coco_val_pipeline)
from test_input_transform_host import opaque, tl_val_pipeline

pytestmark = pytest.mark.gpu

# name -> (pipeline given to the kernels, pipeline run on the host for the float32 reference)
TRANSFORMS = {
    'zero-fields': (None, simple_widerface_val_pipeline),
    'simple': (simple_widerface_val_pipeline, simple_widerface_val_pipeline),
    'swap-only': (Compose([BGR2RGB()]), Compose([BGR2RGB()])),
    'rgb-standard': (tl_val_pipeline, tl_val_pipeline),
    'caffe': (typical_coco_val_pipeline, typical_coco_val_pipeline),     # mean about 100-120, scale 1: a wrong channel or a normalised
}                                                                         # padding is far outside any rounding


def frames(n, h, w, seed=0):
    """uint8 BGR frames whose border pixels are 0 and 255 in turn and whose channels differ strongly, so that padding and image, and one
    channel and another, cannot be confused."""
    rng = np.random.default_rng(seed + 1000 * h + w)
    x = rng.integers(0, 256, (n, h, w, 3), dtype=np.uint8)
    x[..., 0] //= 3                                   # B dark, R bright
    x[..., 2] = 255 - x[..., 2] // 3
    edge = (np.arange(2 * (h + w)) % 2 * 255).astype(np.uint8)
    x[:, 0, :, :] = edge[:w, None]
    x[:, -1, :, :] = edge[1:w + 1, None]
    x[:, :, 0, :] = edge[None, :h, None]
    x[:, :, -1, :] = edge[None, 1:h + 1, None]
    return x


def host_f32(pipeline, x_u8):
    """What the host pipeline uploads for these frames: float32 NCHW."""
    out = [pipeline({'image': img})['image'] for img in x_u8]
    assert all(o.dtype == np.float32 or pipeline is TRANSFORMS['swap-only'][1] for o in out)      # (a swap alone leaves bytes: exact in float32)
    out = [o.astype(np.float32) for o in out]
    return torch.from_numpy(np.ascontiguousarray(np.stack(out).transpose(0, 3, 1, 2)))


def same_bits(a, b, what):
    bad = a.view(torch.int16) != b.view(torch.int16)
    if bool(bad.any()):
        i = tuple(bad.nonzero()[0].tolist())
        raise AssertionError('%s: %d of %d elements differ, first at %s: %r vs %r' % (what, int(bad.sum()), bad.numel(), i, float(a[i]), float(b[i])))


# ------------------------------------------------------------------------------------------------------------------ single ops
def run_stem0(x, transform, w, shift, tail, dtype, impl=nat.CONV_UMMA, max_ctas=0):
    """LFD_OP_STEM0 through lfd_run_op on uint8 NHWC or float32 NCHW x -> [N, Ho, Wo, Cf]."""
    tdt, code = DTYPES[dtype][0], DTYPES[dtype][3]
    u8 = x.dtype == torch.uint8
    N, H, W = (x.shape[0], x.shape[1], x.shape[2]) if u8 else (x.shape[0], x.shape[2], x.shape[3])
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
    nat.check(nat.lib().lfd_run_op(C.byref(op), nat.ptr(x), nat.INPUT_U8_NHWC if u8 else nat.INPUT_F32_NCHW, nat.ptr(ws), None, None, 0, 0,
                                   impl, nat.stream_ptr()))
    torch.cuda.synchronize()
    return ws[4096:4096 + out_b].view(tdt).view(N, Ho, Wo, Cf).clone()


SIZES = [(37, 40), (38, 41), (39, 42), (40, 43)]           # H and W = 0..3 (mod 4)


@pytest.mark.parametrize('name', sorted(TRANSFORMS))
@pytest.mark.parametrize('dtype', ['bf16', 'fp16'])
@pytest.mark.parametrize('cout', [16, 32, 48, 64])
def test_stem0_on_u8_frames_equals_stem0_on_the_host_normalised_tensor(cout, dtype, name):
    kernel_pipe, host_pipe = TRANSFORMS[name]
    transform = input_transform_of(kernel_pipe)
    g = torch.Generator().manual_seed(cout)
    w = torch.randn((cout, 3, 3, 3), generator=g) * 0.05
    shift = torch.randn(cout, generator=g) * 0.1
    tail = (torch.randn((cout, cout, 1, 1), generator=g) * 0.1, torch.randn(cout, generator=g) * 0.1)
    for h, wd in SIZES:
        x8 = frames(2, h, wd)
        xf = host_f32(host_pipe, x8).cuda()
        x8 = torch.from_numpy(x8).cuda()
        for t in (None, tail):
            for ctas in (0, 3):
                what = 'stem0 Cout=%d%s %s %s %dx%d, max_ctas=%d' % (cout, ' + tail' if t else '', dtype, name, h, wd, ctas)
                same_bits(run_stem0(x8, transform, w, shift, t, dtype, max_ctas=ctas), run_stem0(xf, None, w, shift, t, dtype, max_ctas=ctas), what)
        ref = run_stem0(xf, None, w, shift, None, dtype, impl=nat.CONV_SIMT)
        same_bits(run_stem0(x8, transform, w, shift, None, dtype, impl=nat.CONV_SIMT), ref, 'SIMT stem0 Cout=%d %s %s %dx%d' % (cout, dtype, name, h, wd))
        # the SIMT kernel stays the cross-check of the tensor-core path under every transform (one 16-bit spacing: fp32 summation order)
        tc = run_stem0(x8, transform, w, shift, None, dtype).float()
        assert float((tc - ref.float()).abs().max()) <= DTYPES[dtype][2] * 2 * float(ref.float().abs().max()), (cout, dtype, name)


def test_zero_fields_are_the_simple_constants_and_todays_results():
    g = torch.Generator().manual_seed(1)
    w, shift = torch.randn((64, 3, 3, 3), generator=g) * 0.05, torch.randn(64, generator=g) * 0.1
    x8 = frames(2, 45, 61)
    xf = host_f32(simple_widerface_val_pipeline, x8).cuda()
    x8 = torch.from_numpy(x8).cuda()
    zero = run_stem0(x8, None, w, shift, None, 'bf16')
    same_bits(zero, run_stem0(x8, input_transform_of(simple_widerface_val_pipeline), w, shift, None, 'bf16'), 'zero fields vs explicit constants')
    same_bits(zero, run_stem0(xf, None, w, shift, None, 'bf16'), 'zero fields vs fp32 simple_normalize')
    same_bits(zero, run_stem0(xf, input_transform_of(tl_val_pipeline), w, shift, None, 'bf16'), 'the fp32 input ignores the transform')


# ------------------------------------------------------------------------------------------------------------------ plans
@functools.lru_cache(maxsize=None)
def model_of(name):
    model = tl_s.synth_model()[0] if name == 'TL_S' else synth_model(name)[0]
    return model.cuda().eval()


def misaligned(x):
    raw = torch.empty(x.numel() + 1, dtype=torch.uint8, device='cuda')
    y = raw[1:].view(x.shape)                        # base address 1 (mod 4): the fused stem's per-pixel loader
    y.copy_(x)
    assert y.data_ptr() % 4 == 1
    return y


def run_plan(plan, x, graph=False):
    plan.workspace.fill_(0xff)
    with torch.no_grad():
        for _ in range(3 if graph else 1):
            cls, reg = plan.forward(x, use_graph=graph)
    torch.cuda.synchronize()
    return cls.clone(), reg.clone()


def assert_heads(a, b, exact, what):
    for u, v in zip(a, b):
        if exact:
            assert torch.equal(u, v), '%s: %d head outputs differ, max %g' % (what, int((u != v).sum()), float((u - v).abs().max()))
        else:   # GroupNorm statistics are summed with atomics: the bound of tests/test_gpu_schedule_invariance.py
            d = (u - v).abs()
            assert float(d.max()) <= 2.0 ** -6 * float(v.abs().max()) and float((d > 0).float().mean()) <= 1e-2, (what, float(d.max()))


@pytest.mark.parametrize('name', sorted(TRANSFORMS))
@pytest.mark.parametrize('dtype', ['bf16', 'fp16'])
def test_fused_stem_on_both_loaders(dtype, name):
    """STEM4 (WIDERFACE_S, forced): the word loader (W % 4 == 0, aligned base), the per-pixel loader (other widths, or a base address =
    1 mod 4): the stem3 map bit for bit, the head outputs up to the GroupNorm atomics."""
    kernel_pipe, host_pipe = TRANSFORMS[name]
    model = model_of('WIDERFACE_S')
    for h, w in ((186, 252), (185, 253), (187, 254), (184, 255)):
        plan = InferencePlan(model, 2, h, w, torch.device('cuda'), act_dtype=dtype, fuse_stem=True, input_transform=input_transform_of(kernel_pipe),
                             reuse=False)
        assert plan._ops[0]['kind'] == nat.OP_STEM4
        x8 = frames(2, h, w)
        ref = run_plan(plan, host_f32(host_pipe, x8).cuda())
        ref3 = plan.tensor('stem3').clone()
        x8 = torch.from_numpy(x8).cuda()
        for x in (x8, misaligned(x8)):
            for ctas in (0, 3):
                plan._op_array[0].max_ctas = ctas
                old, plan.handle = plan.handle, plan._create_handle()
                nat.lib().lfd_plan_destroy(old)
                got = run_plan(plan, x)
                what = 'stem4 %s %s %dx%d base %% 4 = %d, max_ctas=%d' % (dtype, name, h, w, x.data_ptr() % 4, ctas)
                same_bits(plan.tensor('stem3'), ref3, what)
                assert_heads(got, ref, False, what)


@pytest.mark.parametrize('name', ['zero-fields', 'rgb-standard', 'caffe'])
@pytest.mark.parametrize('cfg,fuse', [('WIDERFACE_S', True), ('TL_L', None), ('TL_S', None)])
def test_frames_below_the_capacity(cfg, fuse, name):
    """One 2 x 400 x 656 plan, frames of every width mod 4, every buffer pre-filled with 0xff: the frame's outputs on uint8 input are those
    of the same plan on the host-normalised tensor (columns past the width and rows past the height are zero AFTER normalisation)."""
    kernel_pipe, host_pipe = TRANSFORMS[name]
    model = model_of(cfg)
    plan = InferencePlan(model, 2, 400, 656, torch.device('cuda'), fuse_stem=fuse, input_transform=input_transform_of(kernel_pipe))
    assert plan._ops[0]['kind'] == (nat.OP_STEM4 if fuse else nat.OP_STEM0)
    for h, w in ((400, 656), (397, 652), (350, 653), (399, 654), (211, 655), (400, 329)):
        x8 = frames(2, h, w)
        xf = host_f32(host_pipe, x8).cuda()
        for graph in (False, True):
            plan.staging(nat.INPUT_U8_NHWC)
            plan._stage.fill_(0xff)                   # the plan-owned input of frames below the capacity, both formats
            ref = run_plan(plan, xf, graph)
            got = run_plan(plan, torch.from_numpy(x8).cuda(), graph)
            assert got[0].shape == ref[0].shape and got[0].shape[1] == plan.frame_P
            assert_heads(got, ref, cfg != 'WIDERFACE_S', '%s %s %dx%d graph=%d' % (cfg, name, h, w, graph))


# ------------------------------------------------------------------------------------------------------------------ models
MODELS = [('TL_L', tl_val_pipeline), ('TL_S', tl_val_pipeline), ('WIDERFACE_S', typical_coco_val_pipeline)]


@pytest.mark.parametrize('cfg,pipeline', MODELS, ids=[m[0] for m in MODELS])
def test_predict_and_forward_take_the_fused_path_with_the_same_results(cfg, pipeline):
    model, _ = (tl_s.synth_model(cls_bias=-1.0) if cfg == 'TL_S' else synth_model(cfg, cls_bias=-1.0))
    model.cuda().eval()
    image = frames(1, 200, 266, seed=3)[0]             # (fewer points than max_detections_per_image: the synthetic heads saturate)
    seen = []
    forward = model.forward
    model.forward = lambda x: (seen.append(x.dtype), forward(x))[1]
    rows = model.predict_for_single_image(image, pipeline, classification_threshold=0.3)
    host = model.predict_for_single_image(image, opaque(pipeline), classification_threshold=0.3)
    assert seen == [torch.uint8, torch.float32] and model.input_transform is None
    assert len(rows) > 0 and len(rows) == len(host)
    np.testing.assert_allclose(np.asarray(rows), np.asarray(host), rtol=0, atol=0 if cfg != 'WIDERFACE_S' else 2e-2)
    model.predict_for_single_image(image.astype(np.float32), pipeline, classification_threshold=0.3)     # not uint8: the host path, as before
    assert seen[-1] == torch.float32
    model.forward = forward
    x8 = torch.from_numpy(frames(2, 360, 490, seed=4))
    xf = host_f32(pipeline, x8.numpy()).cuda()
    model.set_input_transform(pipeline)
    for graph in (False, True):
        model.use_cuda_graph = graph
        with torch.no_grad():
            for _ in range(3):
                got, ref = model(x8.cuda()), model(xf)
        assert_heads(got, ref, cfg != 'WIDERFACE_S', '%s model(x) graph=%d' % (cfg, graph))
    model.set_input_transform(None)
    with torch.no_grad():
        assert not torch.equal(model(x8.cuda())[0], ref[0])                  # another transform, another plan


@pytest.mark.parametrize('cfg,pipeline', [MODELS[1], ('TL_S', None)], ids=['TL_S-tl', 'TL_S-none'])
def test_streaming_detector_runs_the_pipeline_it_is_given(cfg, pipeline):
    from lfd.pipeline import StreamingDetector
    model, _ = tl_s.synth_model(cls_bias=-1.0)
    model.cuda().eval()
    n, h, w = 2, 232, 328
    det = StreamingDetector(model, n, h, w, 0.3, 0.3, max_out=512, input_pipeline=pipeline)
    assert det.plan.input_transform == input_transform_of(pipeline) and model.input_transform is None
    batches = [torch.from_numpy(frames(n, h, w, seed=s)).pin_memory() for s in range(4)]
    slots = [det.submit(b) for b in batches[:2]]
    got = []
    for i, b in enumerate(batches):
        dets, labels, counts = det.collect(slots[i])
        got.append([(dets[j, :int(counts[j])].clone(), labels[j, :int(counts[j])].clone()) for j in range(n)])
        if i + 2 < len(batches):
            slots.append(det.submit(batches[i + 2]))
    model.set_input_transform(pipeline)        # the synchronous path: forward + detect, one batch at a time
    for b, res in zip(batches, got):
        with torch.no_grad():
            out = model(b.cuda())
        dets, labels, _, count, overflow = model.detect(out, [h] * n, [w] * n, [1.0] * n, 0.3, 0.3)
        assert int(overflow) == 0 and int(count.sum()) > 0
        for j in range(n):
            k = int(count[j])
            assert k == res[j][0].shape[0] and torch.equal(dets[j, :k].cpu(), res[j][0]) and torch.equal(labels[j, :k].cpu(), res[j][1])
    if pipeline is None:                        # None is the detector as it always was: simple_normalize on BGR
        with torch.no_grad():
            assert torch.equal(model(host_f32(simple_widerface_val_pipeline, batches[-1].numpy()).cuda())[0], out[0])


# ------------------------------------------------------------------------------------------------------------------ training
def _step(model, x, ann):
    out = model(x)
    ld = model.get_loss(out, ann)
    model._flat_parameters.grad.zero_()
    ld['loss'].backward()
    torch.cuda.synchronize()
    return float(ld['loss'].detach()), model._flat_parameters.grad.clone()


@pytest.mark.parametrize('cfg,frozen', [('TL_L', None), ('WIDERFACE_L', 1)])
def test_training_step_on_u8_batches_equals_the_step_on_the_host_normalised_batch(cfg, frozen):
    """The stem conv, the im2col of its weight gradient and (fine-tuning) the frozen prefix's stem all read the uint8 batch under the
    transform: their outputs bit for bit, the loss and the flat gradient within the run-to-run tolerance of the fp32 atomics."""
    from test_finetune_plan import finetune_model
    n, h, w = 2, 128, 160
    x8 = frames(n, h, w, seed=9)
    xf = host_f32(tl_val_pipeline, x8).cuda()
    x8 = torch.from_numpy(x8).cuda()
    ann = synth.synth_annotations(n, h, w, 1, seed=5)
    res = []
    for x in (x8, xf):
        model = (finetune_model(cfg, frozen) if frozen else synth_model(cfg, cls_bias=-2.0)[0]).cuda().train()
        model.set_input_transform(tl_val_pipeline)
        loss, grad = _step(model, x, ann)
        plan = model.train_plan_for(n, h, w, x.device)
        if frozen:
            name, (ph, pw, pc) = sorted(plan.prefix_outputs.items())[0]
            kept = [plan.tensor(name, ph, pw, pc).clone()]
        else:
            ho, wo = conv_out(h, 3, 2), conv_out(w, 3, 2)
            kept = [plan.tensor('stem0_z', ho, wo, 64).clone(), plan.tensor('stem_im2col', ho, wo, 32).clone()]
        res.append((loss, grad, kept))
    (l8, g8, k8), (lf, gf, kf) = res
    for a, b in zip(k8, kf):
        same_bits(a, b, '%s: a tensor computed from the image' % cfg)
    assert abs(l8 - lf) <= 1e-3 * abs(lf), (l8, lf)
    assert float((g8 - gf).abs().max()) <= 1e-3 * float(gf.abs().max())


def test_loader_hands_u8_batches_to_a_model_that_normalises(tmp_path):
    import os
    import random
    from lfd.data_pipeline.augmentation import HorizontalFlip, bbox_param
    from lfd.data_pipeline.data_loader import DataLoader
    from lfd.data_pipeline.sampler import RandomBBoxCropRegionSampler, RandomWithNegDatasetSampler
    from lfd.execution.executor import Executor
    from test_gpu_input_pipeline import MemoryDataset
    ds = MemoryDataset(9, n=12, size=(140, 220), num_classes=1)
    region = RandomBBoxCropRegionSampler(crop_size=128, resize_range=(0.5, 1.5), resize_prob=0.5)
    pipe = Compose([HorizontalFlip(p=0.5), BGR2RGB(), standard_normalize], bbox_params=bbox_param)
    first = {}
    for arm in (True, False):
        random.seed(1), np.random.seed(1)
        loader = DataLoader(ds, RandomWithNegDatasetSampler(ds, batch_size=4, neg_ratio=0.25), region, pipe, model_normalizes=arm)
        model, _ = synth_model('TL_L', cls_bias=-2.0)
        opt = torch.optim.SGD(model.parameters(), lr=0.02, momentum=0.9, weight_decay=1e-4)
        cfg = dict(work_dir=os.path.join(str(tmp_path), str(arm)), log_path=None, model=model, optimizer=opt,
                   lr_scheduler=torch.optim.lr_scheduler.MultiStepLR(opt, milestones=[5]), training_epochs=1, gpu_list=[0],
                   train_data_loader=None, val_data_loader=None, evaluator=None, val_interval=0, save_interval=100, display_interval=1,
                   optimizer_grad_clip_cfg=dict(max_norm=10, norm_type=2), resume_path=None, weight_path=None)
        fed, losses = [], []

        class Recording(object):
            input_transform = loader.input_transform

            def __iter__(self):
                for batch in loader:
                    fed.append((batch[0].dtype, tuple(batch[0].shape)))
                    yield batch
                    losses.append(float(cfg['loss'].detach()))

        cfg['train_data_loader'] = Recording()
        Executor(cfg).train()
        first[arm] = losses[0]
        if arm:
            assert all(dt == torch.uint8 and shape[1:] == (128, 128, 3) for dt, shape in fed), fed
            assert cfg['model'].input_transform == input_transform_of(tl_val_pipeline)
        else:
            assert all(dt == torch.float32 and shape[1:] == (3, 128, 128) for dt, shape in fed), fed
            assert cfg['model'].input_transform is None
    assert abs(first[True] - first[False]) <= 1e-3 * abs(first[False]), first
