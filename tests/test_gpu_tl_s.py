# -*- coding: utf-8 -*-
"""TrafficLight LFD-S, the shipped config with 48-channel layers (its stem and stage 0), end to end on the GPU: the wgmma path and the
SIMT cross-check against the emulated oracle with the bounds of test_gpu_forward.py, the post-process against the oracle and the
reference, the input formats, CUDA graphs, batches, capacity plans, and an independent cross-check against the
same weights zero-padded to a 64-channel model that runs on the 64-wide kernels."""
import numpy as np
import pytest
import torch

import synth
import tl_s
from helpers import load_golden, rel_err, assert_same_detections_up_to_margins
from lfd import _native as nat
from oracle import lfd_oracle as orc

pytestmark = pytest.mark.gpu
TOL_E2E_RMS, TOL_E2E_MAX = 2e-2, 6e-2          # the C bound of test_gpu_forward.py (bf16 end to end)
# fp16 gate of test_gpu_forward.py: logits rms / max, raw regressions rms, decoded boxes rms / max (relative)
TOL_FP16_RMS, TOL_FP16_MAX, TOL_FP16_REG_RMS, TOL_FP16_BOX_RMS, TOL_FP16_BOX_MAX = 1e-3, 5e-3, 2e-3, 1e-3, 5e-3
CFG = tl_s.TL_S


def _golden():
    return load_golden('forward_TL_S.pt')


def _model(act_dtype='bf16', impl=nat.CONV_UMMA, graph=False):
    g = _golden()
    model, sd = tl_s.synth_model(cls_bias=g['cls_bias'], seed=g['seed'])
    model.cuda()
    model.act_dtype, model.conv_impl, model.use_cuda_graph = act_dtype, impl, graph
    return g, model, sd


def _forward(model, x):
    with torch.no_grad():
        cls, reg = model(x.cuda())
    torch.cuda.synchronize()
    return cls.cpu(), reg.cpu()


def _plan_convs(model):
    plan = list(model._plans.values())[0]
    return [op for op in plan._ops if op['kind'] in (nat.OP_STEM0, nat.OP_CONV)]


@pytest.mark.parametrize('impl', [nat.CONV_UMMA, nat.CONV_SIMT], ids=['umma', 'simt'])
def test_tl_s_bf16_matches_emulated_oracle(impl):
    g, model, sd = _model('bf16', impl)
    x = synth.synth_input(g['N'], g['H'], g['W'])
    cls, reg = _forward(model, x)
    widths = {op['Cout'] for op in _plan_convs(model)}
    assert 48 in widths, widths
    ocls, oreg, sizes = orc.forward(CFG, sd, x, emulate_bf16=True)
    assert [tuple(s) for s in sizes] == [tuple(s) for s in g['sizes']]
    ec, er = rel_err(cls, ocls), rel_err(reg, oreg)
    print('TL_S bf16 impl=%d vs bf16-emulated oracle: cls max/rms %.2e/%.2e reg %.2e/%.2e' % (impl, ec[0], ec[1], er[0], er[1]))
    assert ec[1] < TOL_E2E_RMS and er[1] < TOL_E2E_RMS and ec[0] < TOL_E2E_MAX and er[0] < TOL_E2E_MAX, (ec, er)
    dc, dr = rel_err(cls, g['cls']), rel_err(reg, g['reg'])
    oc, orr = rel_err(ocls, g['cls']), rel_err(oreg, g['reg'])
    print('   vs reference fp32: cls rms %.2e reg rms %.2e (oracle bf16 emulation: %.2e / %.2e)' % (dc[1], dr[1], oc[1], orr[1]))
    assert dc[1] < 2.5 * max(oc[1], 4e-3) and dr[1] < 2.5 * max(orr[1], 4e-3)


def test_tl_s_fp16_meets_1e3_end_to_end():
    g, model, sd = _model('fp16')
    x = synth.synth_input(g['N'], g['H'], g['W'])
    cls, reg = _forward(model, x)
    ocls, oreg, sizes = orc.forward(CFG, sd, x, emulate='fp16')
    ec, er = rel_err(cls, ocls), rel_err(reg, oreg)
    print('TL_S fp16 vs fp16-emulated oracle: cls max/rms %.2e/%.2e reg %.2e/%.2e' % (ec[0], ec[1], er[0], er[1]))
    # the 1.5x slack test_gpu_forward.py gives the deep TL_L, on the whole TL_L gate: the zero-padded 64-channel model (test below, the
    # pre-existing 64-wide kernels) gives the same outputs bit for bit, so this is the rounding noise of the network, not of the 48-wide
    # kernels
    slack = 1.5
    assert ec[1] < slack * TOL_FP16_RMS and ec[0] < slack * TOL_FP16_MAX, ec
    assert er[1] < slack * TOL_FP16_REG_RMS and er[0] < slack * 2 * TOL_FP16_MAX, er
    worst_box = (0.0, 0.0)
    for i in range(g['N']):
        m = g['meta'][i]
        _, bx = orc.decode_image(CFG, cls[i], reg[i], sizes, m['resized_height'], m['resized_width'], m['resize_scale'])
        _, obx = orc.decode_image(CFG, ocls[i], oreg[i], sizes, m['resized_height'], m['resized_width'], m['resize_scale'])
        eb = rel_err(bx, obx)
        worst_box = (max(worst_box[0], eb[0]), max(worst_box[1], eb[1]))
    print('   decoded boxes: max / rms relative error %.2e / %.2e' % worst_box)
    assert worst_box[1] < slack * TOL_FP16_BOX_RMS and worst_box[0] < slack * TOL_FP16_BOX_MAX, worst_box
    # kept indices: the CUDA post-process on the CUDA outputs equals the oracle's post-process on them, in order; end to end the kept
    # sets match up to provably borderline decisions
    model.max_detections_per_image = 32768
    for (thr, iou) in g['results']:
        _, _, src, count, overflow = model.detect((cls.cuda(), reg.cuda()), [m['resized_height'] for m in g['meta']],
                                                  [m['resized_width'] for m in g['meta']], [m['resize_scale'] for m in g['meta']], thr, iou)
        assert int(overflow.item()) == 0
        _, ssrc = orc.get_results(CFG, cls, reg, sizes, g['meta'], thr, iou)
        _, osrc = orc.get_results(CFG, ocls, oreg, sizes, g['meta'], thr, iou)
        for i in range(g['N']):
            got = src[i, :int(count[i])].cpu().tolist()
            assert got == ssrc[i].tolist(), (thr, iou, i)
            m = g['meta'][i]
            osc, obx = orc.decode_image(CFG, ocls[i], oreg[i], sizes, m['resized_height'], m['resized_width'], m['resize_scale'])
            assert_same_detections_up_to_margins(got, osrc[i].tolist(), osc.reshape(-1).numpy(), obx.numpy(), thr, iou, ('TL_S', thr, iou, i))


def test_tl_s_postprocess_matches_oracle_and_reference():
    g = _golden()
    model, _ = tl_s.synth_model(cls_bias=g['cls_bias'], seed=g['seed'])
    model.cuda()
    model.max_detections_per_image = 32768
    for i, hw in enumerate(g['sizes']):
        model._head_indexes_to_feature_map_sizes[i] = tuple(hw)
    cls, reg = g['cls'].cuda(), g['reg'].cuda()
    for (thr, iou), ref in g['results'].items():
        _, _, src, count, _ = model.detect((cls, reg), [m['resized_height'] for m in g['meta']], [m['resized_width'] for m in g['meta']],
                                           [m['resize_scale'] for m in g['meta']], thr, iou)
        _, osrc = orc.get_results(CFG, g['cls'], g['reg'], g['sizes'], g['meta'], thr, iou)
        model._classification_threshold, model._nms_cfg = thr, dict(type='nms', iou_thr=iou)
        rows = model.get_results((cls, reg), g['meta'])
        for i in range(g['N']):
            assert src[i, :int(count[i])].cpu().tolist() == osrc[i].tolist(), (thr, iou, i)
            a, b = np.asarray(rows[i], np.float64).reshape(-1, 6), ref[i].double().numpy()
            assert a.shape == b.shape
            if a.size:
                assert np.array_equal(a[:, 0], b[:, 0])
                np.testing.assert_allclose(a[:, 1:], b[:, 1:], rtol=2e-5, atol=2e-4)


def test_tl_s_u8_graph_and_batch_frames():
    g, model, sd = _model('bf16', graph=True)
    n, h, w = 3, 200, 264
    img = np.stack([synth.synth_image_u8(h, w, seed=40 + s) for s in range(n)])
    with torch.no_grad():
        c8, r8 = model(torch.from_numpy(img).cuda())
        c8b, r8b = model(torch.from_numpy(img).cuda())            # graph replay
        assert torch.equal(c8, c8b) and torch.equal(r8, r8b)
        xf = torch.from_numpy(np.stack([orc.normalize_image_u8(i) for i in img])).permute(0, 3, 1, 2).contiguous()
        cf, rf = model(xf.cuda())
        assert rel_err(c8.cpu(), cf.cpu())[0] < 1e-6 and rel_err(r8.cpu(), rf.cpu())[0] < 1e-6
        model.use_cuda_graph = False
        ce, re_ = model(torch.from_numpy(img).cuda())
        assert torch.equal(ce, c8) and torch.equal(re_, r8), 'graph replay != eager pass'
        for k in range(n):
            ck, rk = model(torch.from_numpy(img[k:k + 1]).cuda())
            assert torch.equal(ck[0], c8[k]) and torch.equal(rk[0], r8[k]), 'frame %d of the batch != the frame alone' % k


def _plan_forward(plan, x):
    with torch.no_grad():
        cls, reg = plan.forward(x, use_graph=False)
    torch.cuda.synchronize()
    return cls.clone(), reg.clone()


def test_tl_s_every_op_bounded_to_few_ctas_is_bit_identical():
    """Tiles are strided by gridDim and TL heads have no GroupNorm (no order-dependent sums): every op bounded to 1 or 5 CTAs gives
    the same cls / reg bits."""
    from lfd._engine import InferencePlan
    g, model, sd = _model('bf16')
    x = synth.synth_input(g['N'], g['H'], g['W']).cuda()
    plan = InferencePlan(model, g['N'], g['H'], g['W'], torch.device('cuda'))
    assert not any(op['kind'] == nat.OP_GN_APPLY for op in plan._ops)
    cls0, reg0 = _plan_forward(plan, x)
    for m in (1, 5):
        for o in plan._op_array:
            o.max_ctas = m
        old = plan.handle
        plan.handle = plan._create_handle()
        nat.lib().lfd_plan_destroy(old)
        cls, reg = _plan_forward(plan, x)
        assert torch.equal(cls, cls0) and torch.equal(reg, reg0), 'every op bounded to %d CTAs changes the outputs' % m


def test_tl_s_capacity_plan_matches_exact_plans():
    """One 2 x 400 x 656 plan runs frames of every h, w (mod 4) down to 1 x 1 deepest levels, with NaN-filled buffers, bit-identical
    to plans built for each frame."""
    from lfd._engine import InferencePlan
    g, model, sd = _model('bf16')
    cap = InferencePlan(model, 2, 400, 656, torch.device('cuda'))
    cap.workspace.fill_(0xff)            # every 16-bit value NaN: a read of anything not written for this frame shows
    for (h, w) in [(400, 656), (397, 653), (302, 518), (131, 211), (64, 97), (33, 34), (17, 18), (1, 1)]:
        x = synth.synth_input(2, h, w, seed=h * 7 + w).cuda()
        ca, ra = _plan_forward(cap, x)
        exact = InferencePlan(model, 2, h, w, torch.device('cuda'))
        ce, re_ = _plan_forward(exact, x)
        del exact
        assert torch.equal(ca, ce) and torch.equal(ra, re_), 'capacity plan != exact plan at %dx%d' % (h, w)


def test_tl_s_predict_for_single_image():
    g, model, sd = _model('fp16')
    img = synth.synth_image_u8(184, 248, seed=5)
    rows = model.predict_for_single_image(img, None, classification_threshold=0.2, nms_threshold=0.4)
    assert len(rows) > 0
    x = torch.from_numpy(orc.normalize_image_u8(img)).permute(2, 0, 1)[None].contiguous()
    ocls, oreg, sizes = orc.forward(CFG, sd, x, emulate='fp16')
    osc, obx = orc.decode_image(CFG, ocls[0], oreg[0], sizes, 184, 248, 1.0)
    _, osrc = orc.get_results(CFG, ocls, oreg, sizes, [dict(resized_height=184, resized_width=248, resize_scale=1.0)], 0.2, 0.4)
    with torch.no_grad():
        out = model(torch.from_numpy(img)[None].cuda())
    _, _, src, count, _ = model.detect(out, [184], [248], [1.0], 0.2, 0.4)
    got = src[0, :int(count[0])].cpu().tolist()
    assert len(got) == len(rows)
    assert_same_detections_up_to_margins(got, osrc[0].tolist(), osc.reshape(-1).numpy(), obx.numpy(), 0.2, 0.4, 'predict', max_frac=3e-2)
    model._nms_cfg = dict(type='soft_nms', iou_thr=0.4, sigma=0.5, min_score=1e-3, method='gaussian')
    soft = model.predict_for_single_image(img, None, classification_threshold=0.2, nms_threshold=0.4)
    assert len(soft) >= len(rows) > 0


def _padded_model(sd48):
    """The same function as a 64-channel model: the 48-channel layers zero-padded to 64 (conv weights and BatchNorm gamma / beta /
    running mean 0, running variance 1 in the padded channels, and 0 weights on the padded inputs of the next layer)."""
    cfg64 = orc._cfg('fast', 64, [4, 2, 1, 1, 1], [64, 64, 64, 128, 128], CFG['backbone']['out_indices'], 1, CFG['lfd']['regression_ranges'],
                     'QualityFocalLoss', True, 'dist', head_norm=False)
    model = tl_s.build_model(cfg64)
    sd64 = model.state_dict()
    out = {}
    for k, v64 in sd64.items():
        v = sd48[k]
        if v.shape == v64.shape:
            out[k] = v.clone()
            continue
        p = torch.ones_like(v64) if k.endswith('running_var') else torch.zeros_like(v64)
        p[tuple(slice(0, s) for s in v.shape)] = v
        out[k] = p
    model.load_state_dict(out, strict=True)
    model.eval()
    return model


@pytest.mark.parametrize('act_dtype', ['bf16', 'fp16'])
def test_tl_s_agrees_with_its_zero_padded_64_channel_model(act_dtype):
    g, model, sd = _model(act_dtype)
    x = synth.synth_input(g['N'], g['H'], g['W'])
    cls, reg = _forward(model, x)
    pad = _padded_model(sd).cuda()
    pad.act_dtype = act_dtype
    pcls, preg = _forward(pad, x)
    assert 48 not in {op['Cout'] for op in _plan_convs(pad)}
    # Every 48-wide MMA sums the same products in the same order as the 64-wide one over its first 48 columns, and the padded
    # channels are exactly 0: the two models compute the same bits
    assert torch.equal(cls, pcls) and torch.equal(reg, preg), ('%s: TL_S and its zero-padded 64-channel model differ' % act_dtype,
                                                                rel_err(cls, pcls), rel_err(reg, preg))


def test_tl_s_training_is_not_implemented():
    from lfd._train import TrainPlan
    g, model, sd = _model('bf16')
    model.train()
    with pytest.raises(NotImplementedError, match='48-channel'):
        TrainPlan(model, 2, 256, 320, torch.device('cuda', 0))


def test_tl_s_streaming_detector_matches_synchronous_path():
    """lfd.pipeline.StreamingDetector (batches in flight on copy / forward / post-process streams) returns, batch by batch, exactly what
    the synchronous forward + detect returns for TL_S, as test_gpu_forward.py checks for WIDERFACE_XS."""
    from lfd.pipeline import StreamingDetector
    g = _golden()
    model, _ = tl_s.synth_model(cls_bias=g['cls_bias'], seed=g['seed'])
    model.cuda()
    n, h, w, iou = 2, 184, 248, 0.4
    batches = [torch.from_numpy(np.stack([synth.synth_image_u8(h, w, seed=10 * b + i) for i in range(n)])) for b in range(5)]
    with torch.no_grad():
        cls, _ = model(batches[0].cuda())
    thr = float(torch.quantile(cls.sigmoid().flatten().float(), 0.99))
    ref = []
    with torch.no_grad():
        for xb in batches:
            dets, labels, _, count, overflow = model.detect(model(xb.cuda()), [h] * n, [w] * n, [1.0] * n, thr, iou)
            assert int(overflow.item()) == 0
            ref.append((dets.cpu().clone(), labels.cpu().clone(), count.cpu().clone()))
    det = StreamingDetector(model, n, h, w, thr, iou, max_out=512)
    got, pending = [], []
    with torch.no_grad():
        for xb in batches:
            pending.append(det.submit(xb.pin_memory()))
            if len(pending) >= det.depth:
                d, l, c = det.collect(pending.pop(0))
                got.append((d.clone(), l.clone(), c.clone()))
        while pending:
            d, l, c = det.collect(pending.pop(0))
            got.append((d.clone(), l.clone(), c.clone()))
    assert len(got) == len(ref)
    total = 0
    for b, ((rd, rl, rc), (gd, gl, gc)) in enumerate(zip(ref, got)):
        assert rc.tolist() == gc.tolist(), b
        for i in range(n):
            k = int(rc[i])
            total += k
            assert torch.equal(rd[i, :k], gd[i, :k]) and torch.equal(rl[i, :k].int(), gl[i, :k].int()), (b, i)
    assert total > 0
