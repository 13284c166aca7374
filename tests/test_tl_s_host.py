# -*- coding: utf-8 -*-
"""CPU tests of TrafficLight LFD-S, the shipped config with 48-channel layers: the oracle against the reference's golden, the compiled
48-channel conv kernel (conv_umma_c48_kernel) pipelining its wgmmas, the configurator's plans for the 48-channel cases of
tests/test_gpu_conv48.py, and training refusing the model."""
import os
import subprocess
import tempfile

import numpy as np
import pytest
import torch

import synth
import tl_s
from helpers import load_golden, rel_err
from oracle import lfd_oracle as orc
from test_conv_sass import _build_module, _sass_counts
import re

_C48 = re.compile(r'_ZN3lfd20conv_umma_c48_kernelILi(\d)ELb([01])ELb([01])ELb([01])EEEvNS_14UmmaConvParamsE')
MODES = (0, 1, 2, 3, 4)        # FLAT, 3x3/s1, 3x3/s2, 1x1/s2, STEM
WAITS_C48, WAITS_C48_DS = 2, 1  # main chain + the 48-channel tail; with the shortcut, one


def test_oracle_forward_and_results_equal_the_reference_golden():
    g = load_golden('forward_TL_S.pt')
    model = tl_s.build_model()
    sd = synth.synth_state_dict(model.state_dict(), seed=g['seed'], cls_bias=g['cls_bias'])
    assert [(k, tuple(v.shape)) for k, v in sd.items()] == g['keys']          # the product's state_dict keys == the reference model's
    assert synth.state_checksum(sd) == g['checksum']
    x = synth.synth_input(g['N'], g['H'], g['W'])
    cls, reg, sizes = orc.forward(tl_s.TL_S, sd, x)
    assert [tuple(s) for s in sizes] == [tuple(s) for s in g['sizes']]
    assert cls.shape == g['cls'].shape and cls.shape[-1] == 1
    ec, er = rel_err(cls, g['cls']), rel_err(reg, g['reg'])
    assert ec[0] < 1e-4 and er[0] < 1e-4, (ec, er)
    for (thr, iou), ref in g['results'].items():
        rows, _ = orc.get_results(tl_s.TL_S, g['cls'], g['reg'], g['sizes'], g['meta'], thr, iou)
        for i in range(g['N']):
            a, b = np.asarray(rows[i], np.float64).reshape(-1, 6), ref[i].double().numpy()
            assert a.shape == b.shape, (thr, iou, i)
            if a.size:
                assert np.array_equal(a[:, 0], b[:, 0])
                np.testing.assert_allclose(a[:, 1:], b[:, 1:], rtol=2e-5, atol=2e-4)


@pytest.fixture(scope='module')
def c48_sass():
    b = _build_module()
    cuobjdump = os.path.join(os.path.dirname(b.NVCC), 'cuobjdump')
    if not (os.path.exists(b.NVCC) and os.path.exists(cuobjdump)):
        pytest.skip('nvcc / cuobjdump not found at %s' % os.path.dirname(b.NVCC))
    flags = [f for f in b.FLAGS if f != '-DLFD_B200_TRACE']
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        procs = {}
        for variant, extra in (('plain', []), ('trace', ['-DLFD_B200_TRACE'])):
            obj = os.path.join(tmp, 'conv_umma_%s.o' % variant)
            cmd = [b.NVCC] + flags + extra + ['-Xptxas', '-v', '-c', os.path.join(b.CSRC, 'conv_umma.cu'), '-o', obj]
            procs[variant] = (obj, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT))
        for variant, (obj, p) in procs.items():
            log = p.communicate()[0].decode()
            assert p.returncode == 0, log
            b._check_stack_frames(log)         # no stack frame, no serialised wgmmas
            out[variant] = _sass_counts(obj, cuobjdump)
    return out


@pytest.mark.parametrize('variant', ['plain', 'trace'])
def test_every_c48_instantiation_pipelines_its_wgmmas(c48_sass, variant):
    found = {tuple(int(v) for v in _C48.fullmatch(n).groups()): c for n, c in c48_sass[variant].items() if _C48.fullmatch(n)}
    want = {(m, f16, ext, ds) for m in MODES for f16 in (0, 1) for ext in (0, 1) for ds in ((0, 1) if m == 2 else (0,))}
    assert set(found) == want, set(found) ^ want
    for key, (hgmma, waits) in found.items():
        assert hgmma > 0 and waits <= (WAITS_C48_DS if key[3] else WAITS_C48), ('conv_umma_c48_kernel', key, hgmma, waits)


def test_build_guards_the_c48_kernel():
    b = _build_module()
    name = '_ZN3lfd20conv_umma_c48_kernelILi1ELb0ELb0ELb0EEEvNS_14UmmaConvParamsE'
    with pytest.raises(RuntimeError):
        b._check_stack_frames("ptxas info    : (C7511) Potential Performance Loss: wgmma.mma_async instructions are serialized due to "
                              "insufficient register resources for the wgmma pipeline in the function '%s'" % name)
    with pytest.raises(RuntimeError):
        b._check_stack_frames('ptxas info    : Function properties for %s\n    256 bytes stack frame, 0 bytes spill stores' % name)


# (N, H, W, Cin, Cout, k, s, relu, res, gn, tail, ds) of tests/test_gpu_conv48.py -> (cc, weights_resident, stages)
PLANS = {
    (2, 23, 31, 16, 48, 1, 1, 1, 0, 0, 0, 0): (16, 1, 8),
    (2, 23, 31, 48, 48, 1, 1, 1, 1, 0, 0, 0): (16, 1, 8),
    (2, 23, 31, 64, 48, 1, 1, 0, 1, 0, 0, 0): (64, 1, 4),
    (2, 23, 31, 64, 48, 1, 1, 1, 0, 0, 0, 0): (64, 1, 4),
    (2, 45, 61, 48, 48, 1, 2, 0, 0, 0, 0, 0): (16, 1, 8),
    (2, 44, 62, 64, 48, 1, 2, 0, 1, 0, 0, 0): (64, 1, 4),
    (2, 37, 41, 48, 48, 3, 1, 1, 1, 0, 0, 0): (16, 1, 8),
    (2, 37, 41, 64, 48, 3, 1, 1, 0, 0, 0, 0): (64, 1, 4),
    (2, 45, 61, 48, 48, 3, 2, 1, 0, 0, 0, 0): (16, 1, 4),
    (2, 44, 62, 48, 48, 3, 2, 1, 0, 0, 0, 48): (16, 1, 4),
    (2, 45, 61, 64, 48, 3, 2, 1, 0, 0, 0, 48): (32, 1, 3),
    (2, 44, 80, 64, 48, 3, 2, 1, 0, 0, 0, 0): (32, 1, 3),
}


# (N, H, W, Cin, Cout, k, s) with tail_cout = 48 -> (cc, weights_resident, stages).  (The stem conv itself has no lfd_conv_query
# geometry: its A operand is the fixed 4-channel image patch, one 16-wide K step per filter row; the GPU tests run it with and without
# the tail.)
TAIL_PLANS = {
    (2, 23, 31, 48, 48, 1, 1): (16, 1, 8),
    (2, 23, 31, 64, 48, 1, 1): (64, 1, 4),
    (2, 45, 61, 48, 48, 3, 2): (16, 1, 4),
    (2, 37, 41, 48, 48, 3, 1): (16, 1, 8),
}


def _co(v, k, s):
    return (v + 2 * (k // 2) - k) // s + 1


def test_conv_query_plans_of_the_48_channel_cases():
    from lfd import _native as nat
    import test_gpu_conv48
    assert set(PLANS) == set(test_gpu_conv48.CASES)
    for case, want in PLANS.items():
        N, H, W, Cin, Cout, k, s, relu, res, gn, tail, ds = case
        q = nat.conv_query(N, H, W, Cin, _co(H, k, s), _co(W, k, s), Cout, k, s, tail, ds)
        assert (q['cc'], q['weights_resident'], q['stages']) == want, (case, q)
        assert q['num_tiles'] >= 12, (case, q)             # 3 CTAs with >= 4 tiles each
    # a 48-channel conv with the 48-channel tail (the 'fast' stem's 1x1 48 -> 48 fused behind a 48-wide conv): its plans
    for case, want in TAIL_PLANS.items():
        N, H, W, Cin, Cout, k, s = case
        q = nat.conv_query(N, H, W, Cin, _co(H, k, s), _co(W, k, s), Cout, k, s, 48, 0)
        assert (q['cc'], q['weights_resident'], q['stages']) == want, (case, q)
    # the 48-channel tail belongs to a 48-channel conv only, the shortcut 48 to the 3x3/s2 48 conv only
    for cout, tail in ((64, 48), (48, 64), (48, 16)):
        with pytest.raises(RuntimeError):
            nat.conv_query(2, 23, 31, 64, 23, 31, cout, 1, 1, tail, 0)
    nat.conv_query(2, 23, 31, 64, 23, 31, 48, 1, 1, 48, 0)
    with pytest.raises(RuntimeError):
        nat.conv_query(2, 45, 61, 48, 23, 31, 64, 3, 2, 0, 48)


@pytest.mark.parametrize('frozen', [None, 'backbone'])
def test_training_tl_s_is_not_implemented(frozen):
    from lfd._train import TrainPlan
    model = tl_s.build_model()
    if frozen:
        for p in model.backbone.parameters() if hasattr(model, 'backbone') else model._backbone.parameters():
            p.requires_grad_(False)
    with pytest.raises(NotImplementedError, match='48-channel'):
        TrainPlan(model, 2, 256, 320, 'cpu', create_native=False)
