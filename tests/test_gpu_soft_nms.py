# -*- coding: utf-8 -*-
"""Soft-NMS on the device (soft_nms_kernel behind lfd_multiclass_soft_nms / lfd_postprocess_soft_nms) against the reference's compiled
soft_nms_cpu (linear mode, where oracle/_ref travels with the tree) and the numpy oracle tests/soft_nms_oracle.py (both modes): boxes, scores,
indices and order bit for bit."""
import os

import numpy as np
import pytest
import torch

import soft_nms_oracle as so
import synth
from helpers import synth_model
from oracle import build_ref
from oracle import lfd_oracle as orc

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
SMEM_CAP = 8192   # candidates per image held in shared memory (postprocess.cu kSoftSmem)


def _bits(a):
    """fp32 bit patterns, every NaN as one pattern (the device's NaN and numpy's differ in payload only)"""
    a = np.asarray(a, np.float32)
    return np.ascontiguousarray(np.where(np.isnan(a), np.float32(np.nan), a)).view(np.int32)


def assert_bitexact(dets, inds, ref_dets, ref_inds, what=''):
    dets, ref_dets = np.asarray(dets, np.float32).reshape(-1, 5), np.asarray(ref_dets, np.float32).reshape(-1, 5)
    np.testing.assert_array_equal(np.asarray(inds), np.asarray(ref_inds), err_msg=str(what))
    assert np.array_equal(_bits(dets), _bits(ref_dets)), what


def random_dets(n, rng, span=200.0, wmin=2.0, wmax=60.0):
    d = np.concatenate([rng.uniform(0, span, (n, 2)), rng.uniform(wmin, wmax, (n, 2)), rng.uniform(0.01, 1, (n, 1))], 1).astype(np.float32)
    d[:, 2:4] += d[:, :2]
    return d


def device_soft(d, thr, method, sigma=0.5, min_score=1e-3):
    from lfd.model.utils import soft_nms
    nd, inds = soft_nms(torch.from_numpy(d).cuda(), thr, method, sigma, min_score)
    return nd.cpu().numpy(), inds.cpu().numpy()


def expected(d, thr, method, sigma=0.5, min_score=1e-3):
    """The compiled reference in linear mode when it is available, else (and in gaussian mode) the oracle."""
    ref = build_ref.load_module() if method == 'linear' else None
    if ref is not None:
        r = ref.soft_nms(torch.from_numpy(d), thr, 1, sigma, min_score).numpy()
        return r[:, :5], r[:, 5].astype(np.int64)
    return so.soft_nms(d, thr, method, sigma, min_score)


# ------------------------------------------------------------------------------------------------ 1. docstring, types, empty input
@pytest.mark.parametrize('method', ['linear', 'gaussian'])
def test_docstring_types_and_empty(method):
    from lfd.model.utils import soft_nms
    g = torch.load(os.path.join(HERE, 'golden', 'soft_nms.pt'), weights_only=False)
    d = g['doc']['dets']
    ref_dets, ref_inds = g['doc'][method]
    nd, inds = soft_nms(d, 0.6, method=method, sigma=0.5)        # numpy in -> numpy out, on the current device
    assert isinstance(nd, np.ndarray) and nd.dtype == np.float32 and inds.dtype == np.int64
    assert len(inds) == (5 if method == 'linear' else 6)
    np.testing.assert_array_equal(inds, ref_inds)
    np.testing.assert_array_equal(np.isnan(nd[:, 4]), np.isnan(ref_dets[:, 4]))
    assert_bitexact(nd, inds, *so.soft_nms(d, 0.6, method, 0.5))
    t = torch.from_numpy(d).cuda()
    td, ti = soft_nms(t, 0.6, method=method)
    assert td.is_cuda and td.dtype == torch.float32 and ti.dtype == torch.int64 and ti.device == t.device
    assert_bitexact(td.cpu().numpy(), ti.cpu().numpy(), nd, inds)
    t64 = t.double()
    td64, _ = soft_nms(t64, 0.6, method=method)
    assert td64.dtype == torch.float64
    for x in (np.zeros((0, 5), np.float32), torch.zeros((0, 5), device='cuda')):
        ed, ei = soft_nms(x, 0.6, method=method)
        assert ed.shape == (0, 5) and ei.shape == (0,)
    with pytest.raises(ValueError):
        soft_nms(d, 0.6, method='hard')


# ------------------------------------------------------------------------------------------------ 2. bit-exact on crafted and random sets
def _special_sets(rng):
    sets = {}
    dup = np.tile(np.array([[10, 10, 20, 20, 0.5]], np.float32), (64, 1))
    dup[::3, 4] = 0.7
    dup[5:15, :4] += 3
    sets['duplicates'] = dup
    eq = np.array([[0, 0, 10, 10, 0.9], [0, 0, 10, 5, 0.8], [0, 0, 10, 5, 0.8], [0, 5, 10, 10, 0.7]], np.float32)   # IoU exactly 0.5
    sets['iou_at_threshold'] = eq
    z = random_dets(80, rng, 40.0)
    z[::4, 2] = z[::4, 0]
    z[1::5, 3] = z[1::5, 1]
    sets['zero_area'] = z
    below = random_dets(120, rng, 50.0)
    below[:, 4] = rng.uniform(0, 9e-4, 120).astype(np.float32)
    sets['all_below'] = below
    # cascade: a heavy box, then many near-copies with low scores at the tail, so the element swapped in is removed again
    c = np.tile(np.array([[50, 50, 90, 90, 0.002]], np.float32), (200, 1))
    c[:, :4] += rng.uniform(-0.2, 0.2, (200, 4)).astype(np.float32)
    c[0, 4] = 0.99
    c[::9, 4] = 0.5
    sets['cascade'] = c
    # two holes and two tied survivors above the new count in one iteration: the last live element fills the lowest hole, so the tie
    # between the moved survivors is broken in the reference's order (rows 0, 6, 5, 3, 4)
    sets['hole_order'] = np.array([[0, 0, 10, 10, 0.9], [0, 0, 10, 10, 0.0015], [0, 0, 10, 10, 0.005], [100, 100, 110, 110, 0.4],
                                   [200, 200, 210, 210, 0.4], [300, 300, 310, 310, 0.4], [400, 400, 410, 410, 0.4]], np.float32)
    return sets


@pytest.mark.parametrize('method', ['linear', 'gaussian'])
def test_special_sets_bitexact(method):
    rng = np.random.RandomState(5)
    for name, d in _special_sets(rng).items():
        thr = 0.5 if name == 'iou_at_threshold' else 0.3
        for min_score in (1e-3, 0.0):
            got = device_soft(d, thr, method, 0.5, min_score)
            assert_bitexact(*got, *expected(d, thr, method, 0.5, min_score), what=(name, min_score))
    for method_ in ('linear', 'gaussian'):
        assert device_soft(_special_sets(rng)['hole_order'], 0.3, method_)[1].tolist() == [0, 6, 5, 3, 4]
    # every candidate below min_score: exactly the first selection comes out
    assert len(device_soft(_special_sets(rng)['all_below'], 0.3, method)[1]) == 1


@pytest.mark.parametrize('method', ['linear', 'gaussian'])
@pytest.mark.parametrize('K', [1, 2, 33, 1000, SMEM_CAP - 1, SMEM_CAP, SMEM_CAP + 1, 20000])
def test_random_sets_bitexact(method, K):
    rng = np.random.RandomState(K)
    d = random_dets(K, rng, span=40.0 * np.sqrt(K) + 50)
    d[::13, 4] = d[-1, 4]              # score ties
    got = device_soft(d, 0.3, method)
    assert_bitexact(*got, *expected(d, 0.3, method), what=K)


# ------------------------------------------------------------------------------------------------ 3. batched_nms / multiclass_nms
@pytest.mark.parametrize('method', ['linear', 'gaussian'])
@pytest.mark.parametrize('C', [5, 45])
@pytest.mark.parametrize('class_agnostic', [False, True])
def test_multiclass_and_batched(method, C, class_agnostic):
    from lfd.model.utils import multiclass_nms, batched_nms
    rng = np.random.RandomState(C)
    n = 400
    boxes = random_dets(n, rng)[:, :4]
    scores = (rng.uniform(0, 1, (n, C + 1)).astype(np.float32) ** 4).astype(np.float32)
    cfg = dict(type='soft_nms', iou_thr=0.3, method=method, sigma=0.5, min_score=1e-3, class_agnostic=class_agnostic)
    dets, labels = multiclass_nms(torch.from_numpy(boxes).cuda(), torch.from_numpy(scores).cuda(), 0.05, cfg)
    od, ol, osrc = so.multiclass_soft_nms(boxes, scores[:, :-1], 0.05, 0.3, method, 0.5, 1e-3, class_agnostic)
    np.testing.assert_array_equal(labels.cpu().numpy(), ol)
    assert np.array_equal(_bits(dets.cpu().numpy()), _bits(od))
    d5, l5 = multiclass_nms(torch.from_numpy(boxes).cuda(), torch.from_numpy(scores).cuda(), 0.05, cfg, max_num=17)
    assert torch.equal(d5, dets[:17]) and torch.equal(l5, labels[:17])
    # batched_nms on one label per row, rows in input order
    lab = rng.randint(0, C, n)
    bd, keep = batched_nms(torch.from_numpy(boxes).cuda(), torch.from_numpy(scores[:, 0]).cuda(), torch.from_numpy(lab).cuda(),
                           dict(type='soft_nms', iou_thr=0.3, method=method), class_agnostic=class_agnostic)
    rd, rl, rsrc = so._soft_on_candidates(boxes, scores[:, 0], lab, np.arange(n), 0.3, method, 0.5, 1e-3, class_agnostic)
    np.testing.assert_array_equal(keep.cpu().numpy(), rsrc)
    assert np.array_equal(_bits(bd.cpu().numpy()), _bits(rd))


@pytest.mark.parametrize('method', ['linear', 'gaussian'])
def test_offsets_inexact_near_2_24_over_C(method):
    """Coordinates near 2^24 / C: label * (max + 1) and the added offsets round in fp32, the areas of the offset boxes with them."""
    from lfd.model.utils import multiclass_nms
    C = 45
    rng = np.random.RandomState(11)
    n = 150
    base = float(2 ** 24 / C) - 200.0
    b = np.concatenate([rng.uniform(base, base + 150, (n, 2)), rng.uniform(1, 40, (n, 2))], 1).astype(np.float32)
    b[:, 2:4] += b[:, :2]
    scores = (rng.uniform(0, 1, (n, C + 1)).astype(np.float32) ** 3).astype(np.float32)
    dets, labels = multiclass_nms(torch.from_numpy(b).cuda(), torch.from_numpy(scores).cuda(), 0.1,
                                  dict(type='soft_nms', iou_thr=0.3, method=method))
    od, ol, _ = so.multiclass_soft_nms(b, scores[:, :-1], 0.1, 0.3, method)
    np.testing.assert_array_equal(labels.cpu().numpy(), ol)
    assert np.array_equal(_bits(dets.cpu().numpy()), _bits(od))


def test_cfg_errors():
    from lfd.model.utils import multiclass_nms
    b = torch.rand(4, 4, device='cuda')
    s = torch.rand(4, 3, device='cuda')
    with pytest.raises(TypeError):
        multiclass_nms(b, s, 0.1, dict(type='soft_nms', iou_thr=0.3, bogus=1))
    with pytest.raises(ValueError):
        multiclass_nms(b, s, 0.1, dict(type='soft_nms', iou_thr=0.3, method='hard'))


# ------------------------------------------------------------------------------------------------ 4. the model path
def _device_candidates(model, outputs, hs, ws, scales, thr):
    """Every candidate with its device score and box: hard NMS with iou_thr 1.0 suppresses nothing."""
    saved = model._nms_cfg
    model._nms_cfg = dict(type='nms', iou_thr=1.0)
    dets, labels, src, count, overflow = model.detect(outputs, hs, ws, scales, thr, 1.0, class_agnostic=True)
    model._nms_cfg = saved
    assert int(overflow.item()) == 0
    return [(dets[i, :int(count[i])].cpu().numpy(), src[i, :int(count[i])].cpu().numpy()) for i in range(len(hs))]


@pytest.mark.parametrize('name', ['WIDERFACE_S', 'TT100K_L'])
@pytest.mark.parametrize('method', ['linear', 'gaussian'])
def test_get_results_model_path(name, method):
    g = torch.load(os.path.join(HERE, 'golden', 'forward_%s.pt' % name), weights_only=False)
    gs = torch.load(os.path.join(HERE, 'golden', 'soft_nms.pt'), weights_only=False)['models'][name]
    model, _ = synth_model(name, cls_bias=-1.0)
    model.cuda()
    model.max_detections_per_image = 32768      # TT100K_L at this threshold: more candidates than shared memory holds
    for i, hw in enumerate(g['sizes']):
        model._head_indexes_to_feature_map_sizes[i] = tuple(hw)
    cls, reg = g['cls'].cuda(), g['reg'].cuda()
    thr, C = gs['score_thr'], orc.CONFIGS[name]['lfd']['num_classes']
    meta = g['meta']
    hs, ws, sc = [m['resized_height'] for m in meta], [m['resized_width'] for m in meta], [m['resize_scale'] for m in meta]
    cands = _device_candidates(model, (cls, reg), hs, ws, sc, thr)
    model._classification_threshold = thr
    model._nms_cfg = dict(type='soft_nms', iou_thr=0.3, method=method, sigma=0.5, min_score=1e-3)
    rows = model.get_results((cls, reg), meta)
    for i, (cd, csrc) in enumerate(cands):
        od, ol, _ = so.soft_on_candidates(cd[:, :4], cd[:, 4], csrc, C, 0.3, method)
        want = np.asarray(so.rows_of(od, ol), np.float32).reshape(-1, 6)
        got = np.asarray(rows[i], np.float32).reshape(-1, 6)
        assert np.array_equal(_bits(got), _bits(want)), (name, method, i)
        ref = gs['results'][method][i].numpy()          # the reference's get_results: sigmoid / softmax rounding apart
        assert abs(len(ref) - len(got)) <= max(2, len(ref) // 200), (len(ref), len(got))
        k = min(len(ref), len(got), 50)
        np.testing.assert_array_equal(ref[:k, 0], got[:k, 0])
        np.testing.assert_allclose(got[:k, 1:], ref[:k, 1:], rtol=2e-5, atol=2e-4)


@pytest.mark.parametrize('method', ['linear', 'gaussian'])
def test_predict_for_single_image(method):
    model, _ = synth_model('WIDERFACE_S', cls_bias=-1.0)
    img = synth.synth_image_u8(184, 248, seed=7)
    model._nms_cfg = dict(type='nms', iou_thr=1.0)
    model.predict_for_single_image(img, None, classification_threshold=0.2)      # records the feature-map sizes
    with torch.no_grad():
        out = model(torch.from_numpy(img)[None].cuda())
    (cd, csrc), = _device_candidates(model, out, [184], [248], [1.0], 0.2)
    model._nms_cfg = dict(type='soft_nms', iou_thr=0.3, method=method)
    rows = model.predict_for_single_image(img, None, classification_threshold=0.2)
    od, ol, _ = so.soft_on_candidates(cd[:, :4], cd[:, 4], csrc, 1, 0.3, method)
    assert len(rows) > 0
    assert np.array_equal(_bits(np.asarray(rows, np.float32).reshape(-1, 6)), _bits(np.asarray(so.rows_of(od, ol), np.float32).reshape(-1, 6)))


# ------------------------------------------------------------------------------------------------ 5. mixed batch: empty, shared-memory, global
def test_mixed_batch_and_overflow():
    model, _ = synth_model('WIDERFACE_S', cls_bias=-1.0)
    model.cuda()
    model.max_detections_per_image = 16384
    sizes = [(180, 320), (90, 160), (45, 80), (23, 40), (12, 20)][:len(orc.strides_of(orc.CONFIGS['WIDERFACE_S']))]
    for i, hw in enumerate(sizes):
        model._head_indexes_to_feature_map_sizes[i] = hw
    P = sum(h * w for h, w in sizes)
    g = torch.Generator().manual_seed(0)
    cls = torch.full((3, P, 1), -20.0)
    reg = torch.randn((3, P, 4), generator=g) * 0.5
    counts = (0, 3000, 12000)
    for i, k in enumerate(counts):
        idx = torch.randperm(P, generator=g)[:k]
        cls[i, idx, 0] = torch.randn(k, generator=g)
    cls, reg = cls.cuda(), reg.cuda()
    hs, ws = [720] * 3, [1280] * 3
    cands = _device_candidates(model, (cls, reg), hs, ws, [1.0] * 3, 0.05)
    assert [len(c[1]) for c in cands][0] == 0 and len(cands[1][1]) < SMEM_CAP < len(cands[2][1])
    for method in ('linear', 'gaussian'):
        model._nms_cfg = dict(type='soft_nms', iou_thr=0.3, method=method)
        dets, labels, src, count, overflow = model.detect((cls, reg), hs, ws, [1.0] * 3, 0.05, 0.3)
        assert int(overflow.item()) == 0 and int(count[0]) == 0
        for i in (1, 2):
            cd, csrc = cands[i]
            od, _, osrc = so.soft_on_candidates(cd[:, :4], cd[:, 4], csrc, 1, 0.3, method)
            k = int(count[i])
            np.testing.assert_array_equal(src[i, :k].cpu().numpy(), osrc)
            assert np.array_equal(_bits(dets[i, :k].cpu().numpy()), _bits(od))
    model.max_detections_per_image = 5000
    with pytest.raises(Exception, match='max_detections_per_image'):
        model.get_results((cls, reg), [dict(resized_height=720, resized_width=1280, resize_scale=1.0)] * 3)


# ------------------------------------------------------------------------------------------------ 6. streaming, 7. CUDA graph, 8. unknown type
def test_streaming_detector_soft_nms():
    from lfd.pipeline import StreamingDetector
    model, _ = synth_model('WIDERFACE_XS', cls_bias=-1.0)
    model.cuda()
    model._nms_cfg = dict(type='soft_nms', iou_thr=0.3, method='gaussian', sigma=0.5, min_score=1e-3)
    n, h, w = 2, 184, 248
    batches = [torch.from_numpy(np.stack([synth.synth_image_u8(h, w, seed=100 * b + i) for i in range(n)])) for b in range(5)]
    thr = 0.3
    ref = []
    with torch.no_grad():
        for xb in batches:
            dets, labels, src, count, overflow = model.detect(model(xb.cuda()), [h] * n, [w] * n, [1.0] * n, thr, 0.3)
            ref.append((dets.cpu().clone(), labels.cpu().clone(), count.cpu().clone()))
    det = StreamingDetector(model, n, h, w, thr, 0.3, max_out=512)
    model._nms_cfg = dict(type='nms', iou_thr=0.3)      # read at construction
    total = 0
    with torch.no_grad():
        for b, xb in enumerate(batches):
            gd, gl, gc = det.infer(xb.pin_memory())
            rd, rl, rc = ref[b]
            assert rc.tolist() == gc.tolist(), b
            for i in range(n):
                k = min(int(rc[i]), 512)
                total += k
                assert torch.equal(rd[i, :k], gd[i, :k]) and torch.equal(rl[i, :k].int(), gl[i, :k].int()), (b, i)
    assert total > 0


def test_cuda_graph_replay():
    from lfd.model.utils.nms import _device_nms  # noqa: F401  (library loaded)
    model, _ = synth_model('WIDERFACE_S', cls_bias=-1.0)
    g = torch.load(os.path.join(HERE, 'golden', 'forward_WIDERFACE_S.pt'), weights_only=False)
    model.cuda()
    for i, hw in enumerate(g['sizes']):
        model._head_indexes_to_feature_map_sizes[i] = tuple(hw)
    model._nms_cfg = dict(type='soft_nms', iou_thr=0.3, method='linear')
    cls, reg = g['cls'].cuda().contiguous(), g['reg'].cuda().contiguous()
    meta = g['meta']
    pp = model.post_plan(cls.shape[0], g['sizes'], cls.device)
    pp.set_meta([m['resized_width'] for m in meta], [m['resized_height'] for m in meta], [m['resize_scale'] for m in meta])
    eager = [t.clone() for t in pp.run(cls, reg, 0.05, 0.3)]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        pp.run(cls, reg, 0.05, 0.3)
        torch.cuda.synchronize()
        for t in pp.dets, pp.labels, pp.src, pp.count:
            t.zero_()
        with torch.cuda.graph(graph, stream=s):
            pp.run(cls, reg, 0.05, 0.3)
    torch.cuda.current_stream().wait_stream(s)
    for t in pp.dets, pp.labels, pp.src, pp.count:
        t.zero_()
    graph.replay()
    torch.cuda.synchronize()
    N = cls.shape[0]
    assert torch.equal(eager[3], pp.count)
    for i in range(N):
        k = int(eager[3][i])
        assert k > 0
        assert torch.equal(eager[0][i, :k], pp.dets[i, :k]) and torch.equal(eager[2][i, :k], pp.src[i, :k])


def test_unknown_type_raises():
    model, _ = synth_model('WIDERFACE_XS', cls_bias=-1.0)
    model.cuda()
    x = synth.synth_input(1, 120, 200).cuda()
    with torch.no_grad():
        out = model(x)
    model._nms_cfg = dict(type='nms_match', iou_thr=0.3)
    with pytest.raises(ValueError):
        model.get_results(out, [dict(resized_height=120, resized_width=200, resize_scale=1.0)])
