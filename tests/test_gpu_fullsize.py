# -*- coding: utf-8 -*-
"""BASELINE.json's configurations at their FULL sizes.  The CPU oracle cannot evaluate these batches in test time, so parity
is checked through properties that do not depend on the size (plus one full-resolution frame against the oracle):

  * images of a batch are independent: frame k of the batch-N plan == the same frame through a batch-1 plan
    (bit-exact for the backbone / neck tensors; fp32 head outputs to 1e-5, their GroupNorm statistics are fp64 atomics);
  * a batch of N copies of one frame gives N identical outputs, and a CUDA-graph replay reproduces the eager pass bit for bit;
  * the post-process of the CUDA outputs keeps exactly the (point, class) indices the oracle keeps from the same tensors;
  * one full-resolution frame against the bf16-emulated oracle, inside the end-to-end drift bound of DESIGN.md (gate C).
"""
import numpy as np
import pytest
import torch

import synth
from helpers import assert_same_detections_up_to_margins, rel_err, synth_model, assert_same_detections
from oracle import lfd_oracle as orc

pytestmark = pytest.mark.gpu

FULL = [
    ('WIDERFACE_S', 8, 720, 1280, 0.002, 0.3),     # configs[1]: the bench workload
    ('TT100K_L', 16, 1080, 1920, 0.00005, 0.3),    # configs[3]: 45 classes, softmax / class-offset NMS
    ('WIDERFACE_XS', 2, 2160, 3840, 0.002, 0.3),   # configs[4]: 4K frames (per-GPU shard of the throughput sweep)
    ('WIDERFACE_L', 4, 640, 640, 0.002, 0.3),      # configs[2] geometry (training crops) through the inference plan
]


def _frames(n, h, w, distinct=True):
    base = [synth.synth_image_u8(h, w, seed=11 + (i if distinct else 0)) for i in range(n)]
    return torch.from_numpy(np.stack(base))


@pytest.mark.parametrize('name,n,h,w,frac,iou', FULL, ids=[f[0] for f in FULL])
def test_full_size_batch_independence_and_postprocess(name, n, h, w, frac, iou):
    model, _ = synth_model(name, cls_bias=-2.0)
    model.cuda()
    model.max_detections_per_image = 16384
    x = _frames(n, h, w).cuda()
    with torch.no_grad():
        model.use_cuda_graph = False
        cls_e, reg_e = model(x)
        model.use_cuda_graph = True
        cls_g, reg_g = model(x)
        cls_g2, reg_g2 = model(x)                      # replay of the captured graph
    assert torch.isfinite(cls_e).all() and torch.isfinite(reg_e).all()
    assert rel_err(cls_g, cls_e)[0] < 1e-5 and rel_err(reg_g, reg_e)[0] < 1e-5
    assert rel_err(cls_g2, cls_g)[0] < 1e-5 and rel_err(reg_g2, reg_g)[0] < 1e-5
    sizes = [tuple(model.head_indexes_to_feature_map_sizes[i]) for i in range(len(model.head_indexes_to_feature_map_sizes))]
    assert cls_e.shape[1] == sum(a * b for a, b in sizes)
    # frame k alone == frame k inside the batch
    for k in (0, n - 1):
        with torch.no_grad():
            c1, r1 = model(x[k:k + 1].contiguous())
        assert rel_err(c1[0], cls_e[k])[0] < 1e-5 and rel_err(r1[0], reg_e[k])[0] < 1e-5, (name, k)
    # post-process of the CUDA outputs vs the oracle's decode + NMS of the same tensors
    meta = [dict(resized_height=h, resized_width=w, resize_scale=1.0) for _ in range(n)]
    for i, hw in enumerate(sizes):
        model._head_indexes_to_feature_map_sizes[i] = hw
    # score threshold calibrated so that a fraction `frac` of the (point, class) scores pass (the synthetic weights are not
    # trained), then moved away from every actual score: the CUDA kernel and torch evaluate sigmoid / softmax with different
    # instruction sequences, so a score within a few ulps of the threshold would legitimately pass in one and fail in the other
    scores = cls_e.sigmoid() if cls_e.shape[2] == model._num_classes else cls_e.softmax(-1)[..., :-1]
    flat = scores.flatten().float()
    gen = torch.Generator(device=flat.device).manual_seed(1234)
    sample = flat[torch.randperm(flat.numel(), device=flat.device, generator=gen)[:2000000]] if flat.numel() > 2000000 else flat
    thr = float(torch.quantile(sample, 1.0 - frac))
    for _ in range(50):
        if float((flat - thr).abs().min()) > 2e-5 * thr:
            break
        thr *= 1.0 + 1e-4
    else:
        raise AssertionError('no score-free threshold found')
    dets, labels, src, count, overflow = model.detect((cls_e, reg_e), [h] * n, [w] * n, [1.0] * n, thr, iou)
    assert int(overflow.item()) == 0
    _, osrc = orc.get_results(orc.CONFIGS[name], cls_e.cpu(), reg_e.cpu(), sizes, meta, thr, iou)
    total = 0
    for i in range(n):
        kk = int(count[i].item())
        total += kk
        assert src[i, :kk].cpu().tolist() == osrc[i].tolist(), (name, i)
    print('%s %dx%dx%d: %d detections kept, identical to the oracle' % (name, n, h, w, total))
    assert total > 0


def test_identical_frames_give_identical_outputs():
    model, _ = synth_model('WIDERFACE_S', cls_bias=-2.0)
    model.cuda()
    x = _frames(8, 720, 1280, distinct=False).cuda()
    with torch.no_grad():
        cls, reg = model(x)
    for k in range(1, 8):
        assert rel_err(cls[k], cls[0])[0] < 1e-5 and rel_err(reg[k], reg[0])[0] < 1e-5


def test_one_720p_frame_against_the_oracle():
    model, sd = synth_model('WIDERFACE_S', cls_bias=-2.0)
    model.cuda()
    img = synth.synth_image_u8(720, 1280, seed=5)
    with torch.no_grad():
        cls, reg = model(torch.from_numpy(img)[None].cuda())
    xf = torch.from_numpy(orc.normalize_image_u8(img)).permute(2, 0, 1)[None].contiguous()
    ocls, oreg, sizes = orc.forward(orc.CONFIGS['WIDERFACE_S'], sd, xf, emulate_bf16=True)
    ec, er = rel_err(cls.cpu(), ocls), rel_err(reg.cpu(), oreg)
    print('720p frame vs bf16-emulated oracle: cls max/rms %.2e/%.2e reg %.2e/%.2e' % (ec[0], ec[1], er[0], er[1]))
    assert ec[1] < 2e-2 and er[1] < 2e-2 and ec[0] < 8e-2 and er[0] < 8e-2
    # fp16 storage: the stated 1e-3 at full resolution, and identical kept indices at the predict / evaluation thresholds
    model.act_dtype = 'fp16'
    with torch.no_grad():
        cls, reg = model(torch.from_numpy(img)[None].cuda())
    ocls, oreg, sizes = orc.forward(orc.CONFIGS['WIDERFACE_S'], sd, xf, emulate='fp16')
    ec, er = rel_err(cls.cpu(), ocls), rel_err(reg.cpu(), oreg)
    print('720p frame, fp16 vs fp16-emulated oracle: cls max/rms %.2e/%.2e reg %.2e/%.2e' % (ec[0], ec[1], er[0], er[1]))
    assert ec[1] < 1e-3 and ec[0] < 5e-3 and er[1] < 2e-3 and er[0] < 1e-2, (ec, er)
    meta = [dict(resized_height=720, resized_width=1280, resize_scale=1.0)]
    model.max_detections_per_image = 32768
    osc, obx = orc.decode_image(orc.CONFIGS['WIDERFACE_S'], ocls[0], oreg[0], sizes, 720, 1280, 1.0)
    osc, obx = osc.reshape(-1).numpy(), obx.numpy()
    q999 = float(np.quantile(osc, 0.999))             # a threshold that keeps ~0.1 % of the points whatever the synthetic bias is
    # WIDERFACE_train/predict.py:22 (0.5 / 0.3), evaluation.py:60-61 (0.01 / 0.4: ~10^4 detections per frame)
    for (thr, iou) in ((0.5, 0.3), (q999, 0.3), (0.01, 0.4)):
        dets, labels, src, count, overflow = model.detect((cls, reg), [720], [1280], [1.0], thr, iou)
        assert int(overflow.item()) == 0
        orows, osrc = orc.get_results(orc.CONFIGS['WIDERFACE_S'], ocls, oreg, sizes, meta, thr, iou)
        k = int(count[0].item())
        got = src[0, :k].cpu().tolist()
        # the CUDA post-process on the CUDA outputs is EXACTLY the oracle's post-process on the same outputs ...
        _, same_src = orc.get_results(orc.CONFIGS['WIDERFACE_S'], cls.cpu(), reg.cpu(), sizes, meta, thr, iou)
        assert got == same_src[0].tolist(), ('720p', thr, iou, 'post-process on identical inputs')
        # ... and end to end (two pipelines that agree to 1e-3) the kept sets agree up to provably borderline decisions
        nd = assert_same_detections_up_to_margins(got, osrc[0].tolist(), osc, obx, thr, iou, ('720p', thr, iou))
        print('   thr %.3f / iou %.1f: %d detections, %d borderline decisions differ end to end' % (thr, iou, k, nd))


def test_fp16_activation_range_is_safe():
    """max-abs trace of every stored tensor of the fp16 plan (WIDERFACE-S 720p, TT100K-L 1080p crops): orders of magnitude inside
    the fp16 range (65504) -- the values are post-BatchNorm / ReLU activations; the conversion saturates instead of overflowing."""
    from lfd._engine import InferencePlan
    for name, h, w in (('WIDERFACE_S', 720, 1280), ('TT100K_L', 544, 960)):
        model, _ = synth_model(name, cls_bias=-2.0)
        model.cuda()
        model.act_dtype = 'fp16'
        x = torch.from_numpy(synth.synth_image_u8(h, w, seed=7))[None].cuda()
        # the plan model(x) builds, with reuse=False: every stored tensor stays readable after the forward
        plan = InferencePlan(model, 1, h, w, torch.device('cuda'), model.conv_impl, act_dtype=model.act_dtype,
                             input_transform=model.input_transform, reuse=False)
        cls, reg = plan.forward(x, use_graph=False)
        worst = 0.0
        for op in plan._ops:
            for key in ('out', 'out2'):
                if op.get(key) is not None:
                    worst = max(worst, float(plan.tensor(op[key]).float().abs().max()))
        print('%s fp16 plan: largest stored activation %.1f' % (name, worst))
        assert worst < 2048.0 and torch.isfinite(cls).all() and torch.isfinite(reg).all()
