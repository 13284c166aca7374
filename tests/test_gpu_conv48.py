# -*- coding: utf-8 -*-
"""The 48-channel forward convs (conv_umma_c48_kernel, and the SIMT cross-check kernels) at op level against a float64 CPU evaluation
of the same operation on the same 16-bit operands, with the faithful bound of test_gpu_conv_configs.py: |out - y| <= ulp16(y) +
K 2^-24 S.

A 48-channel tensor has 96-byte pixel rows.  Every tensor the op reads or writes sits in a NaN-filled workspace, with NaN guard bytes
around it (gpu_ops.run_conv, gpu_ops.run_stem0): a store that wrote past channel 47 of a pixel would overwrite the next pixel's channels (or the guard) and a residual load
that read past it would carry a NaN into the sum.  The outputs must be finite, the guards untouched."""
import pytest
import torch

from gpu_ops import (DTYPES, STEM_FMT, assert_faithful, assert_tail_close, conv_reference, ref_conv64, run_conv_case, run_stem0, stem_input,
                     stem_operands)
from helpers import bits
from lfd import _native as nat

pytestmark = pytest.mark.gpu

# (N, H, W, Cin, Cout, k, s, relu, res, gn, tail, ds), as in test_gpu_conv_configs.CASES; the plans are pinned in test_tl_s_host.py
CASES = [
    (2, 23, 31, 16, 48, 1, 1, 1, 0, 0, 0, 0),        # FLAT 48 from Cin 16
    (2, 23, 31, 48, 48, 1, 1, 1, 1, 0, 0, 0),        # from 48 (Cc 16, three chunks), residual
    (2, 23, 31, 64, 48, 1, 1, 0, 1, 0, 0, 0),        # from 64, residual
    (2, 23, 31, 64, 48, 1, 1, 1, 0, 0, 0, 0),
    (2, 45, 61, 48, 48, 1, 2, 0, 0, 0, 0, 0),        # 1x1/s2 48 (the unfused stage-0 shortcut), odd x odd input
    (2, 44, 62, 64, 48, 1, 2, 0, 1, 0, 0, 0),        # even x even, residual
    (2, 37, 41, 48, 48, 3, 1, 1, 1, 0, 0, 0),        # 3x3/s1 48 -> 48 + residual (stage-0 blocks)
    (2, 37, 41, 64, 48, 3, 1, 1, 0, 0, 0, 0),        # 3x3/s1 from 64
    (2, 45, 61, 48, 48, 3, 2, 1, 0, 0, 0, 0),        # 3x3/s2 48 -> 48, odd x odd
    (2, 44, 62, 48, 48, 3, 2, 1, 0, 0, 0, 48),       # with the fused 48 -> 48 shortcut, even x even (stage 0, block 0)
    (2, 45, 61, 64, 48, 3, 2, 1, 0, 0, 0, 48),       # shortcut from 64, odd x odd
    (2, 44, 80, 64, 48, 3, 2, 1, 0, 0, 0, 0),        # 3x3/s2 from 64, even x even
]
# (Cout, tail, fmt, H, W): the 'fast' stem of TL_S with and without its fused 1x1 48 -> 48, H and W = 0..3 (mod 4), large enough for
# interior tiles
STEM_CASES = [(48, 0, 'u8', 100, 124), (48, 48, 'f32', 101, 125), (48, 0, 'f32', 102, 126), (48, 48, 'u8', 103, 127)]


def _id(c):
    return 'N%d_%dx%d_%d-%d_k%ds%d_r%d_res%d_gn%d_tail%d_ds%d' % c


def _stem_id(c):
    return 'c%d_tail%d_%s_%dx%d' % c


def _seed(case):
    return (hash(case) + 48) & 0xffff


def _impls(case):
    # the SIMT cross-check kernels have no fused shortcut: the planner runs that conv on its own there
    return [nat.CONV_UMMA] + ([] if case[11] else [nat.CONV_SIMT])


@pytest.mark.parametrize('max_ctas', [0, 3])
@pytest.mark.parametrize('dtype', ['bf16', 'fp16'])
@pytest.mark.parametrize('case', CASES, ids=_id)
def test_conv48_matches_fp64(case, dtype, max_ctas):
    (ref, S, K), short = conv_reference(case, dtype, _seed(case))
    for impl in _impls(case) if max_ctas == 0 else [nat.CONV_UMMA]:
        out, _, q, out3 = run_conv_case(case, dtype, _seed(case), max_ctas, impl)
        if max_ctas:
            assert q['num_tiles'] // max_ctas >= 4
        what = 'conv48 %s %s impl=%d max_ctas=%d (plan %s)' % (_id(case), dtype, impl, max_ctas, q)
        assert bool(torch.isfinite(out.float()).all()), what + ': NaN read from outside a tensor'
        assert_faithful(out, ref, S, K, dtype, what)
        if out3 is not None:
            assert_faithful(out3, short[0], short[1], short[2], dtype, what + ' shortcut')


@pytest.mark.parametrize('case', CASES, ids=_id)
def test_conv48_grid_does_not_change_the_output(case):
    out0, _, _, sc0 = run_conv_case(case, 'bf16', _seed(case))
    for m in (1, 2, 7):
        out, _, _, sc = run_conv_case(case, 'bf16', _seed(case), m)
        assert torch.equal(bits(out), bits(out0)), 'max_ctas=%d changes %d output elements' % (m, int((out != out0).sum()))
        if sc is not None:
            assert torch.equal(bits(sc), bits(sc0)), 'max_ctas=%d changes the shortcut output' % m


# ------------------------------------------------------------------------------------------------ STEM0 48 (+ the 48 -> 48 tail)
def _stem_seed(case):
    Cout, tail, fmt, H, W = case
    return 4800 + tail * 10 + H + W


def _run_stem(case, dtype, max_ctas, impl=nat.CONV_UMMA):
    img, w, shift, t = stem_operands(case, _stem_seed(case))
    return run_stem0(img.cuda(), STEM_FMT[case[2]], w, shift, tail=t, dtype=dtype, impl=impl, max_ctas=max_ctas)


@pytest.mark.parametrize('max_ctas', [0, 3])
@pytest.mark.parametrize('dtype', ['bf16', 'fp16'])
@pytest.mark.parametrize('case', STEM_CASES, ids=_stem_id)
def test_stem48_matches_fp64(case, dtype, max_ctas):
    Cout, tail, fmt, H, W = case
    img, w, shift, t = stem_operands(case, _stem_seed(case))
    x = stem_input(img, fmt, dtype)
    ones = torch.ones(Cout)
    # the SIMT stem kernel has no fused tail (the planner does not fuse there)
    impls = [nat.CONV_UMMA] + ([nat.CONV_SIMT] if not tail and not max_ctas else [])
    for impl in impls:
        out, num_tiles = _run_stem(case, dtype, max_ctas, impl)
        if max_ctas:
            assert num_tiles // max_ctas >= 4
        what = 'stem48 %s %s impl=%d max_ctas=%d' % (_stem_id(case), dtype, impl, max_ctas)
        assert bool(torch.isfinite(out.float()).all()), what
        if tail:
            mid, _, _ = ref_conv64(x, w, ones, shift, 2, True, dtype=dtype)
            ref, _, _ = ref_conv64(DTYPES[dtype][1](mid.float()), t[0], t[1], t[2], 1, True, dtype=dtype)
            assert_tail_close(out, ref, dtype, what)
        else:
            ref, S, K = ref_conv64(x, w, ones, shift, 2, True, dtype=dtype)
            assert_faithful(out, ref, S, K, dtype, what)


@pytest.mark.parametrize('case', STEM_CASES, ids=_stem_id)
def test_stem48_grid_does_not_change_the_output(case):
    out0 = _run_stem(case, 'bf16', 0)[0]
    for m in (1, 2, 7):
        assert torch.equal(bits(_run_stem(case, 'bf16', m)[0]), bits(out0)), 'stem max_ctas=%d' % m
