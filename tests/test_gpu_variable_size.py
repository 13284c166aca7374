# -*- coding: utf-8 -*-
"""Frames below a plan's capacity: one plan of N x H x W runs every frame of h <= H, w <= W on the same kernels, workspace and CUDA
graph, with the results of a plan built for the frame.

Each sub-capacity call is preceded by NaN in the workspace, the plan's input staging and the outputs (0xff bytes: NaN in every float
type, 255 in a uint8 staging), so a bound taken from the capacity instead of the frame shows up as a difference.  Conv outputs that do
not depend on a GroupNorm must be bit-identical in the valid region; the others, and cls / reg of GroupNorm configs, get the allowance of
test_gpu_schedule_invariance.py for cls / reg (the fp64 statistics atomics add in another order on another grid)."""
import random

import numpy as np
import pytest
import torch

import synth
from helpers import close_downstream_of_gn, conv_outputs, downstream_of_gn, poison, synth_model, untouched
from lfd import _native as nat
from lfd._engine import InferencePlan

pytestmark = pytest.mark.gpu

N, H, W = 2, 400, 656
# the capacity; every h mod 4 and w mod 4; deepest levels of 1 x 1 (100 x 120, 37 x 5); the smallest frame; widths with and without the
# stem4 word loader's w % 4 == 0 (the capacity, 656, always has it)
SIZES = [(400, 656), (399, 655), (398, 654), (397, 653), (396, 652), (257, 130), (130, 259), (100, 120), (37, 5), (1, 1)]


def _order(seed):
    """The sizes in a scrambled order, each twice; the capacity first (its graph is captured on the caller's tensor)."""
    rng = random.Random(seed)
    seq = SIZES[1:] * 2
    rng.shuffle(seq)
    return [SIZES[0]] + seq[:9] + [SIZES[0]] + seq[9:]


def _frames(h, w, seed):
    g = torch.Generator().manual_seed(seed)
    u8 = torch.randint(0, 256, (N, h, w, 3), dtype=torch.uint8, generator=g)
    f32 = synth.synth_input(N, h, w, seed=seed)
    return {nat.INPUT_U8_NHWC: u8.cuda(), nat.INPUT_F32_NCHW: f32.cuda().contiguous()}


class _Exact(object):
    """Per frame size: a plan built for it (with the capacity plan's stem choice) and its results per input format."""

    def __init__(self, model, fuse_stem, act_dtype):
        self.model, self.fuse_stem, self.act_dtype, self.cache = model, fuse_stem, act_dtype, {}

    def get(self, h, w, fmt, x):
        key = (h, w, fmt)
        if key not in self.cache:
            plan = InferencePlan(self.model, N, h, w, torch.device('cuda'), act_dtype=self.act_dtype, fuse_stem=self.fuse_stem, reuse=False)
            with torch.no_grad():
                cls, reg = plan.forward(x, use_graph=False)
            torch.cuda.synchronize()
            tensors = {name: plan.tensor(name).clone() for name, _ in conv_outputs(plan)}
            self.cache[key] = (tensors, cls.clone(), reg.clone(), plan.level_sizes, _stats(plan))
            del plan
        return self.cache[key]


def _stats(plan):
    """The GroupNorm statistics of the last forward: (sum, sum of squares) per (statistics slot, image, group), fp64."""
    return plan.workspace[:plan.stats_bytes].view(torch.float64).clone()


def _compare(what, plan, exact, cls, reg, has_gn, tainted):
    tensors, ecls, ereg, level_sizes, estats = exact
    assert plan.frame_level_sizes == level_sizes, what
    # the statistics of the frame's pixels, of convs whose input does not depend on a GroupNorm, summed in another grouping: a pixel
    # counted once too often or too rarely moves the sum of squares by about 1 / (pixels of the level), >= 6e-5 here; the fp32 partial
    # sums of 1x1-conv tiles, which cover 128 consecutive pixels at the capacity's row pitch instead of the frame's, and the fp64
    # atomics' order by ~1e-7
    st, per_slot = _stats(plan), N * 16 * 2
    for op in plan._ops:
        if op['kind'] == nat.OP_CONV and op.get('gn_groups') and op.get('inp') not in tainted and op.get('res') not in tainted:
            k = op['stats']
            s2, es2 = st[k * per_slot + 1:(k + 1) * per_slot:2], estats[k * per_slot + 1:(k + 1) * per_slot:2]
            assert bool(((s2 - es2).abs() <= 1e-5 * es2.abs()).all()), (what, op['out'], 'GroupNorm statistics',
                                                                        float(((s2 - es2).abs() / es2.abs()).max()))
    for name, op in conv_outputs(plan):
        want = tensors[name]
        got = plan.tensor(name)[:, :want.shape[1], :want.shape[2]]
        if name not in tainted:
            assert torch.equal(got.view(torch.int16), want.view(torch.int16)), '%s: %s differs in %d of %d elements' % (
                what, name, int((got.view(torch.int16) != want.view(torch.int16)).sum()), want.numel())
        else:
            close_downstream_of_gn(what + ': ' + name, got.float(), want.float())
    assert cls.shape == ecls.shape and reg.shape == ereg.shape, (what, cls.shape, ecls.shape)
    if not has_gn:
        assert torch.equal(cls, ecls) and torch.equal(reg, ereg), '%s: head outputs differ' % what
    else:
        close_downstream_of_gn(what + ': cls', cls, ecls)
        close_downstream_of_gn(what + ': reg', reg, ereg)


CASES = [('WIDERFACE_S', None, 'bf16'), ('WIDERFACE_S', True, 'bf16'), ('WIDERFACE_L', None, 'bf16'), ('TT100K_L', None, 'bf16'),
         ('TL_L', None, 'bf16'), ('TEST_FAST', None, 'bf16'), ('WIDERFACE_L', None, 'fp16'), ('TL_L', None, 'fp16')]


@pytest.mark.parametrize('name,fuse_stem,act_dtype', CASES)
def test_capacity_plan_matches_exact_plans_tensor_by_tensor(name, fuse_stem, act_dtype):
    model, _ = synth_model(name)
    model.cuda()
    plan = InferencePlan(model, N, H, W, torch.device('cuda'), act_dtype=act_dtype, fuse_stem=fuse_stem, reuse=False)   # intermediates stay readable
    stem4 = plan._ops[0]['kind'] == nat.OP_STEM4
    assert stem4 == bool(fuse_stem)
    # the exact plans are forced to the capacity plan's stem: a small frame alone would not take STEM4 (its stem1 map stays in L2), and
    # the two paths give the same bits (test_gpu_stem_fusion.py)
    exact = _Exact(model, stem4, act_dtype)
    has_gn = any(op['kind'] == nat.OP_GN_APPLY or (op['kind'] == nat.OP_HEAD_FINAL and op.get('gn_groups')) for op in plan._ops)
    assert has_gn == (name != 'TL_L')
    tainted = downstream_of_gn(plan)
    frames = {s: _frames(s[0], s[1], seed=11 + i) for i, s in enumerate(SIZES)}
    graphs = 0
    for fmt in (nat.INPUT_U8_NHWC, nat.INPUT_F32_NCHW):
        held = torch.empty_like(frames[SIZES[0]][fmt])        # capacity frames: one caller tensor, so one graph
        for use_graph in (False, True):
            for (h, w) in _order(fmt * 2 + use_graph):
                x = frames[(h, w)][fmt]
                if (h, w) == (H, W):
                    held.copy_(x)
                    x = held
                else:
                    poison(plan)
                with torch.no_grad():
                    cls, reg = plan.forward(x, use_graph=use_graph)
                torch.cuda.synchronize()
                what = '%s %s fmt=%d graph=%d %dx%d' % (name, act_dtype, fmt, use_graph, h, w)
                _compare(what, plan, exact.get(h, w, fmt, frames[(h, w)][fmt]), cls, reg, has_gn, tainted)
        graphs += 2
        assert plan.num_graphs() == graphs, (name, fmt, plan.num_graphs())   # the caller's tensor at capacity + the staged input


def _images(seed, count, width):
    rng = np.random.RandomState(seed)
    heights = rng.randint(96, 420, size=count)
    return [rng.randint(0, 256, size=(int(h), width, 3)).astype(np.uint8) for h in heights]


def _rows_close(a, b, what):
    assert len(a) == len(b), (what, len(a), len(b))
    if a:
        a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
        assert np.array_equal(a[:, 0], b[:, 0]), what
        assert np.allclose(a[:, 1:], b[:, 1:], rtol=1e-4, atol=1e-3), (what, float(np.abs(a - b).max()))


@pytest.mark.parametrize('nms', ['nms', 'soft_nms'])
def test_predict_for_single_image_one_plan_per_maximum(nms):
    model, _ = synth_model('WIDERFACE_S', cls_bias=-1.0)
    model.cuda()
    model._classification_threshold = 0.3
    model._nms_cfg = dict(type='nms', iou_thr=0.4) if nms == 'nms' else dict(type='soft_nms', iou_thr=0.4, sigma=0.5, min_score=0.3, method='linear')
    images = _images(5, 20, 512)
    got, plans, maxima, top = [], set(), 0, 0
    for im in images:
        if im.shape[0] > top:
            top, maxima = im.shape[0], maxima + 1
        got.append(model.predict_for_single_image(im, None))
        plans |= set(model._plans)           # (n, h, w, device, conv_impl, act_dtype) of the plans built so far
        assert len(model._plans) == 1
    assert len(plans) == maxima, (sorted(plans), maxima)
    for i, im in enumerate(images):
        model.invalidate_plans()
        want = model.predict_for_single_image(im, None)
        _rows_close(got[i], want, '%s image %d (%dx%d)' % (nms, i, im.shape[0], im.shape[1]))


def test_get_results_of_mixed_sizes_match_per_size_post_plans():
    model, _ = synth_model('WIDERFACE_S', cls_bias=-1.0)
    model.cuda()
    model._classification_threshold, model._nms_cfg = 0.3, dict(type='nms', iou_thr=0.4)
    for i, (h, w) in enumerate([(320, 512), (200, 512), (317, 509), (320, 512), (96, 130)]):
        x = torch.from_numpy(_images(30 + i, 1, w)[0][:h]).cuda()[None].repeat(2, 1, 1, 1).contiguous()
        with torch.no_grad():
            cls, reg = model(x)
        sizes = model._sizes()
        meta = [dict(resized_height=h, resized_width=w, resize_scale=1.0)] * 2
        rows = model.get_results((cls, reg), meta)
        pp = model.post_plan(2, sizes, cls.device)
        pp.set_meta([w, w], [h, h], [1.0, 1.0])
        dets, labels, _, count = pp.run(cls.contiguous(), reg.contiguous(), 0.3, 0.4)
        want = model._rows(dets, labels, count[:2], count[2:], model.max_detections_per_image)
        assert rows == want, (h, w)
    assert len(model._plans) == 1


def test_errors_launch_nothing():
    model, _ = synth_model('TEST_FAST')
    model.cuda()
    plan = InferencePlan(model, N, 96, 160, torch.device('cuda'))
    for shape in [(N, 97, 160, 3), (N, 96, 161, 3), (N + 1, 64, 64, 3), (N - 1, 96, 160, 3)]:
        x = torch.zeros(shape, dtype=torch.uint8, device='cuda')
        msg = untouched(plan, lambda: plan.forward(x))
        assert 'capacity' in msg
    # the C entry point checks the frame and the table itself
    lib, stage = nat.lib(), plan.staging(nat.INPUT_U8_NHWC)
    table = plan._extent(64, 100)[0]

    def raw(h, w, t):
        with torch.cuda.device(plan.device):
            nat.check(lib.lfd_plan_forward_extent(plan.handle, nat.ptr(stage), nat.INPUT_U8_NHWC, h, w, t, nat.ptr(plan.workspace),
                                                  nat.ptr(plan.cls_out), nat.ptr(plan.reg_out), 1, nat.stream_ptr()))
    assert 'capacity' in untouched(plan, lambda: raw(97, 160, table))
    assert 'capacity' in untouched(plan, lambda: raw(64, 161, table))
    assert 'frame' in untouched(plan, lambda: raw(64, 96, table))          # a table of another frame
    bad = (nat.Extent * len(table))()
    C_ = __import__('ctypes')
    C_.memmove(bad, table, C_.sizeof(table))
    bad[3].Ho = 10 ** 4
    assert 'outside' in untouched(plan, lambda: raw(64, 100, bad))
    simt = InferencePlan(model, N, 96, 160, torch.device('cuda'), conv_impl=nat.CONV_SIMT)
    x = torch.zeros((N, 64, 100, 3), dtype=torch.uint8, device='cuda')
    assert 'SIMT' in untouched(simt, lambda: simt.forward(x))
    with torch.cuda.device(simt.device):
        rc = lib.lfd_plan_forward_extent(simt.handle, nat.ptr(simt.staging(nat.INPUT_U8_NHWC)), nat.INPUT_U8_NHWC, 64, 100,
                                         simt._extent(64, 100)[0], nat.ptr(simt.workspace), nat.ptr(simt.cls_out), nat.ptr(simt.reg_out),
                                         0, nat.stream_ptr())
    assert rc == 3        # LFD_ERR_UNSUPPORTED
