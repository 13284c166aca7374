# -*- coding: utf-8 -*-
"""The Soft-NMS oracle (tests/soft_nms_oracle.py) against the reference's own results (tests/golden/soft_nms.pt) and, where oracle/_ref has
been built, against the compiled reference directly.  CPU only.

Linear mode is bit-exact.  Gaussian mode selects the same rows in the same order; its scores may differ by an ulp per decay, because the
reference's glibc expf is not correctly rounded and the oracle rounds exp(double)."""
import os

import numpy as np
import pytest
import torch

import soft_nms_oracle as so
from oracle import build_ref
from oracle import lfd_oracle as orc

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope='module')
def golden():
    return torch.load(os.path.join(HERE, 'golden', 'soft_nms.pt'), weights_only=False)


def _np(x):
    return x.numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


def assert_same(ref_dets, ref_inds, dets, inds, method):
    ref_dets, dets = _np(ref_dets).astype(np.float32), _np(dets).astype(np.float32)
    np.testing.assert_array_equal(_np(ref_inds), _np(inds))
    if method == 'linear':
        assert np.array_equal(ref_dets.view(np.int32), dets.view(np.int32))
        return
    assert np.array_equal(ref_dets[:, :4].view(np.int32), dets[:, :4].view(np.int32))
    a, b = ref_dets[:, 4], dets[:, 4]
    nan = np.isnan(a)
    np.testing.assert_array_equal(nan, np.isnan(b))
    # row i has been decayed at most i times, each decay within an ulp of the weight
    bound = np.abs(a[~nan]) * np.float32(2.0 ** -23) * (np.arange(len(a))[~nan] + 2)
    assert np.all(np.abs(a[~nan] - b[~nan]) <= bound)


@pytest.mark.parametrize('method', ['linear', 'gaussian'])
def test_docstring(golden, method):
    d = golden['doc']['dets']
    ref_dets, ref_inds = golden['doc'][method]
    dets, inds = so.soft_nms(d, 0.6, method, sigma=0.5)
    assert len(inds) == (5 if method == 'linear' else 6)
    assert_same(ref_dets, ref_inds, dets, inds, method)
    if method == 'gaussian':   # zero-area pairs: 0 / 0 overlaps
        assert np.isnan(dets[:, 4]).sum() == 4


@pytest.mark.parametrize('method', ['linear', 'gaussian'])
def test_sets(golden, method):
    for key, case in golden['sets'].items():
        ref_dets, ref_inds = case['results'][method]
        dets, inds = so.soft_nms(case['dets'], 0.3, method, 0.5, 1e-3)
        assert_same(ref_dets, ref_inds, dets, inds, method), key
    assert len(golden['sets'][('all_below', 0)]['results'][method][1]) == 1


@pytest.mark.parametrize('method', ['linear', 'gaussian'])
def test_multiclass(golden, method):
    mc = golden['multiclass']
    ref_dets, ref_labels = mc['results'][method]
    sc = mc['scores'].numpy()[:, :-1]
    dets, labels, src = so.multiclass_soft_nms(mc['boxes'].numpy(), sc, mc['score_thr'], 0.3, method, 0.5, 1e-3)
    np.testing.assert_array_equal(ref_labels.numpy(), labels)
    assert_same(ref_dets, src, dets, src, method)


@pytest.mark.parametrize('name', ['WIDERFACE_S', 'TT100K_L'])
@pytest.mark.parametrize('method', ['linear', 'gaussian'])
def test_get_results(golden, name, method):
    g = torch.load(os.path.join(HERE, 'golden', 'forward_%s.pt' % name), weights_only=False)
    case = golden['models'][name]
    rows, _ = so.get_results(orc.CONFIGS[name], g['cls'], g['reg'], g['sizes'], g['meta'], case['score_thr'], 0.3, method, 0.5, 1e-3)
    for ref, got in zip(case['results'][method], rows):
        got = np.asarray(got, np.float32).reshape(-1, 6)
        ref = ref.numpy()
        assert ref.shape == got.shape
        np.testing.assert_array_equal(ref[:, 0], got[:, 0])
        if method == 'linear':
            assert np.array_equal(ref.view(np.int32), got.view(np.int32))
        else:
            assert np.array_equal(ref[:, 2:].view(np.int32), got[:, 2:].view(np.int32))
            np.testing.assert_allclose(got[:, 1], ref[:, 1], rtol=2.0 ** -23 * (len(ref) + 2), atol=0)


def _random(n, rng, span):
    d = np.concatenate([rng.uniform(0, span, (n, 2)), rng.uniform(1, 40, (n, 2)), rng.uniform(0.001, 1, (n, 1))], 1).astype(np.float32)
    d[:, 2:4] += d[:, :2]
    return d


@pytest.mark.parametrize('method', ['linear', 'gaussian'])
def test_against_compiled_reference(method):
    ref = build_ref.load_module()
    if ref is None:
        pytest.skip('oracle/_ref has not been built (python oracle/build_ref.py)')
    rng = np.random.RandomState(99)
    for n, span, thr, sigma, mins in ((3, 20, 0.3, 0.5, 1e-3), (257, 60, 0.5, 0.3, 1e-2), (1500, 300, 0.3, 0.5, 1e-3), (400, 30, 0.1, 1.0, 0.0)):
        d = _random(n, rng, span)
        d[::7, 4] = d[-1, 4]                # score ties
        d[::11, :4] = d[-2, :4]             # duplicate boxes
        r = ref.soft_nms(torch.from_numpy(d), thr, so.METHODS[method], sigma, mins).numpy()
        dets, inds = so.soft_nms(d, thr, method, sigma, mins)
        assert_same(r[:, :5], r[:, 5].astype(np.int64), dets, inds, method)
