# -*- coding: utf-8 -*-
"""The EXT = true kernel builds (frames below a plan's capacity) per configuration against float64: every conv configuration of
test_gpu_conv_configs.py, test_gpu_conv48.py and test_gpu_conv_solo.py, the stem conv from fp32, uint8 BGR and NV12 frames, the fused
four-conv stem with and without its word loader, GroupNorm apply and the head's final 1x1 convs, each launched with a geometry-table row
through lfd_plan_forward_extent (tests/extent_ops.py) at frames chosen to hit the edges of the tile walk.

Per (case, frame, dtype) and at max_ctas 0, 1 and 3:
- the valid region is within the faithful (or fused-tail) bound of a float64 evaluation on the cropped operands with zero padding;
- it is bit-identical to the EXT = false launch (lfd_run_op) of the same op on tensors of the frame's own size, and every grid gives the
  same bits; GroupNorm statistics equal the sums over the valid stored pixels and the full-size launch's up to the order of the fp64
  atomics;
- nothing outside the op's outputs is written, and nothing in them outside the tiles that intersect the valid extent."""
import functools
import random

import pytest
import torch

import extent_ops as X
from gpu_ops import assert_faithful, assert_gn_stats, assert_tail_close, conv_out
from lfd import _native as nat
from train_op_ref import check_within

pytestmark = pytest.mark.gpu

# (N, H, W, Cin, Cout, k, s, relu, res, gn, tail, ds) at the capacity -> (cc, weights_resident, stages, schedule) the configurator picks.
# The configurations of test_gpu_conv_configs.CASES, test_gpu_conv48.CASES and test_gpu_conv_solo.CASES; the 3x3 capacities are at least
# 33 x 17 (stride 1) and 64 x 32 (stride 2) so that a tile's halo can be inside the capacity and one row past the frame.
CONV_CASES = [
    # test_gpu_conv_configs.CASES
    ((2, 23, 31, 16, 16, 1, 1, 1, 0, 0, 0, 0), (16, 1, 8, 'shared')),       # Cout 16, Cc 16
    ((2, 23, 31, 48, 32, 1, 1, 1, 1, 0, 0, 0), (16, 1, 8, 'shared')),       # three chunks, residual
    ((2, 23, 31, 96, 64, 1, 1, 0, 1, 0, 0, 0), (32, 1, 4, 'shared')),       # Cc 32
    ((2, 23, 31, 128, 128, 1, 1, 0, 0, 16, 0, 0), (64, 1, 4, 'shared')),    # GroupNorm statistics of flat tiles
    ((2, 23, 31, 32, 32, 1, 1, 1, 0, 0, 16, 0), (32, 1, 4, 'shared')),      # tail 16
    ((2, 23, 31, 128, 64, 1, 1, 1, 0, 0, 32, 0), (64, 1, 4, 'shared')),     # tail 32
    ((2, 23, 31, 64, 128, 1, 1, 1, 0, 16, 128, 0), (64, 1, 4, 'shared')),   # tail 128 + statistics of the tail output
    ((2, 45, 61, 64, 16, 1, 2, 0, 0, 0, 0, 0), (64, 1, 4, 'shared')),       # 1x1/s2 Cout 16
    ((2, 44, 62, 64, 32, 1, 2, 0, 1, 0, 0, 0), (64, 1, 4, 'shared')),
    ((2, 45, 61, 48, 64, 1, 2, 1, 0, 0, 0, 0), (16, 1, 8, 'shared')),
    ((2, 44, 61, 128, 128, 1, 2, 0, 0, 16, 0, 0), (64, 1, 4, 'shared')),
    ((2, 45, 80, 16, 32, 3, 1, 1, 1, 0, 0, 0), (16, 1, 8, 'shared')),
    ((2, 37, 31, 32, 64, 3, 1, 1, 0, 0, 0, 0), (32, 1, 4, 'shared')),
    ((2, 37, 40, 96, 128, 3, 1, 1, 1, 0, 0, 0), (16, 0, 3, 'shared')),      # streamed weights
    ((2, 37, 40, 128, 128, 3, 1, 0, 0, 16, 0, 0), (16, 0, 3, 'shared')),    # streamed, GroupNorm statistics
    ((2, 37, 29, 64, 64, 3, 1, 1, 1, 0, 128, 0), (64, 1, 3, 'shared')),     # tail 128 with a residual on the tail output
    ((2, 69, 61, 32, 32, 3, 2, 1, 0, 0, 0, 0), (32, 1, 4, 'shared')),
    ((2, 69, 80, 48, 64, 3, 2, 1, 0, 0, 0, 0), (16, 1, 4, 'shared')),
    ((2, 70, 62, 64, 128, 3, 2, 1, 0, 0, 0, 0), (16, 0, 3, 'shared')),
    ((2, 69, 80, 64, 64, 3, 2, 1, 0, 0, 64, 0), (32, 1, 3, 'shared')),      # tail 64
    ((2, 69, 80, 32, 32, 3, 2, 1, 0, 0, 0, 32), (32, 1, 4, 'shared')),      # fused shortcut 32
    ((2, 69, 61, 64, 64, 3, 2, 1, 0, 0, 0, 64), (32, 1, 3, 'shared')),      # shortcut 64
    ((2, 70, 80, 64, 128, 3, 2, 1, 0, 0, 0, 128), (16, 0, 3, 'shared')),    # shortcut 128, streamed
    ((2, 69, 80, 128, 128, 3, 2, 1, 0, 0, 0, 128), (16, 0, 2, 'shared')),   # shortcut 128, 2-stage ring
    # test_gpu_conv48.CASES: conv_umma_c48_kernel
    ((2, 23, 31, 16, 48, 1, 1, 1, 0, 0, 0, 0), (16, 1, 8, 'shared')),
    ((2, 23, 31, 48, 48, 1, 1, 1, 1, 0, 0, 0), (16, 1, 8, 'shared')),
    ((2, 23, 31, 64, 48, 1, 1, 0, 1, 0, 0, 0), (64, 1, 4, 'shared')),
    ((2, 23, 31, 64, 48, 1, 1, 1, 0, 0, 0, 0), (64, 1, 4, 'shared')),
    ((2, 45, 61, 48, 48, 1, 2, 0, 0, 0, 0, 0), (16, 1, 8, 'shared')),
    ((2, 44, 62, 64, 48, 1, 2, 0, 1, 0, 0, 0), (64, 1, 4, 'shared')),
    ((2, 37, 41, 48, 48, 3, 1, 1, 1, 0, 0, 0), (16, 1, 8, 'shared')),
    ((2, 37, 41, 64, 48, 3, 1, 1, 0, 0, 0, 0), (64, 1, 4, 'shared')),
    ((2, 69, 61, 48, 48, 3, 2, 1, 0, 0, 0, 0), (16, 1, 4, 'shared')),
    ((2, 70, 62, 48, 48, 3, 2, 1, 0, 0, 0, 48), (16, 1, 4, 'shared')),
    ((2, 69, 61, 64, 48, 3, 2, 1, 0, 0, 0, 48), (32, 1, 3, 'shared')),
    ((2, 70, 80, 64, 48, 3, 2, 1, 0, 0, 0, 0), (32, 1, 3, 'shared')),
    # test_gpu_conv_solo.CASES: conv_umma_solo_kernel (chosen at the capacity; the frames leave CTAs with one tile or none)
    ((3, 90, 160, 64, 64, 3, 1, 1, 0, 0, 0, 0), (64, 1, 4, 'solo')),
    ((3, 90, 160, 64, 64, 3, 1, 1, 1, 0, 0, 0), (64, 1, 4, 'solo')),
    ((2, 100, 164, 64, 64, 3, 1, 0, 1, 0, 0, 0), (64, 1, 4, 'solo')),
    ((8, 37, 83, 64, 64, 3, 1, 0, 0, 0, 0, 0), (64, 1, 4, 'solo')),
    ((2, 90, 160, 64, 64, 3, 1, 0, 1, 0, 0, 0), (64, 1, 4, 'solo')),
]

# STEM0 (Cout, tail, fmt, transform, N, H, W): every (Cout, tail) of test_gpu_conv_configs.STEM_CASES and test_gpu_conv48.STEM_CASES,
# from fp32, uint8 BGR and NV12 frames, uint8 / NV12 under the zero-field, 'rgb-standard' and 'caffe' transforms
STEM_CASES = [
    (16, 0, 'u8', None, 2, 100, 124), (16, 16, 'f32', None, 2, 101, 125), (16, 32, 'nv12', 'caffe', 2, 100, 126),
    (16, 64, 'u8', 'rgb-standard', 2, 103, 124), (16, 128, 'nv12', None, 2, 102, 124),
    (32, 0, 'nv12', 'rgb-standard', 2, 100, 124), (32, 16, 'u8', 'caffe', 2, 102, 127), (32, 32, 'f32', None, 2, 103, 125),
    (32, 64, 'u8', None, 2, 100, 126), (32, 128, 'f32', None, 2, 102, 127),
    (64, 0, 'f32', None, 2, 103, 126), (64, 16, 'nv12', None, 2, 100, 126), (64, 32, 'u8', 'rgb-standard', 2, 101, 124),
    (64, 64, 'nv12', 'caffe', 2, 102, 126), (64, 128, 'u8', None, 2, 103, 124),
    (48, 0, 'nv12', 'rgb-standard', 2, 100, 124), (48, 48, 'u8', 'caffe', 2, 103, 127),
]

# STEM4 (fmt, aligned, N, H, W): the word loader on (uint8 / NV12, capacity W % 4 == 0, aligned) and off (misaligned uint8, fp32)
STEM4_CASES = [('u8', 1, 2, 132, 256), ('u8', 0, 2, 132, 256), ('f32', 1, 2, 131, 254), ('nv12', 1, 2, 132, 256)]

GN_CASES = [(16, 2, 23, 31), (32, 2, 23, 31), (64, 2, 23, 31), (128, 2, 23, 31)]        # (C, N, H, W), groups = C / 8
# (n_cls, n_reg, groups, N, H, W): one output, the 4 box outputs, a multi-class head; with GroupNorm and without (TL_L's heads)
HEAD_CASES = [(1, 0, 16, 2, 23, 31), (0, 4, 16, 2, 23, 31), (7, 4, 16, 2, 23, 31), (1, 0, 0, 2, 23, 31), (0, 4, 0, 2, 23, 31),
              (7, 4, 0, 2, 23, 31)]

GRIDS = (0, 1, 3)
DTYPE_NAMES = ('bf16', 'fp16')

MODE_FLAT, MODE_3X3S1, MODE_3X3S2, MODE_1X1S2, MODE_STEM = 'flat', '3x3s1', '3x3s2', '1x1s2', 'stem'


def _mode(k, s):
    return {(1, 1): MODE_FLAT, (3, 1): MODE_3X3S1, (3, 2): MODE_3X3S2, (1, 2): MODE_1X1S2}[(k, s)]


def conv_id(c):
    return 'N%d_%dx%d_%d-%d_k%ds%d_r%d_res%d_gn%d_tail%d_ds%d' % c


def stem_id(c):
    return 'c%d_tail%d_%s_%s_N%d_%dx%d' % (c[0], c[1], c[2], c[3] or 'zero', c[4], c[5], c[6])


def stem4_id(c):
    return '%s_%s_N%d_%dx%d' % (c[0], 'aligned' if c[1] else 'misaligned', c[2], c[3], c[4])


def gn_id(c):
    return 'C%d_N%d_%dx%d' % c


def head_id(c):
    return 'cls%d_reg%d_gn%d_N%d_%dx%d' % c


def stem4_extents(H, W, even=False):
    """Frames below a STEM4 capacity of W % 4 == 0: widths with w % 4 = 1, 2, 3 end inside the word loader's last word group"""
    ex = [(H - 1, W - 3, 'partial last tile, w % 4 = 1'), (H - 2, W - 2, 'w % 4 = 2'), (65, W - 1, 'stem3 output 17 rows, w % 4 = 3'),
          (1, 1, '1 x 1'), (3, W, 'full width, one output row'), (H, 7, 'full height, narrow, w % 4 = 3')]
    if even:
        ex = [(max(2, h - h % 2), max(2, w - w % 2), why) for h, w, why in ex]
    return [e for e in ex if (e[0], e[1]) != (H, W)]


def _extents(kind, case):
    if kind == 'conv':
        return X.conv_extents(case)
    if kind == 'stem':
        return X.frame_extents(case[5], case[6], even=case[2] == 'nv12', stem=True)
    if kind == 'stem4':
        return stem4_extents(case[3], case[4], even=case[0] == 'nv12')
    return X.frame_extents(case[-2], case[-1])


SPECS = {'conv': X.ConvSpec, 'stem': X.StemSpec, 'stem4': X.Stem4Spec, 'gn': X.GnSpec, 'head': X.HeadSpec}


@functools.lru_cache(maxsize=None)
def _spec(kind, case, dtype):
    return SPECS[kind](case, dtype)


def _capacity(kind, case):
    if kind == 'conv':
        return case[1], case[2]
    if kind == 'stem4':
        return case[3], case[4]
    return case[-2], case[-1]


def n_cases():
    """(case, frame, dtype, max_ctas) combinations this file checks"""
    tables = [('conv', [c for c, _ in CONV_CASES]), ('stem', STEM_CASES), ('stem4', STEM4_CASES), ('gn', GN_CASES), ('head', HEAD_CASES)]
    return sum(len(_extents(k, c)) for k, t in tables for c in t) * len(DTYPE_NAMES) * len(GRIDS)


def test_case_count():
    """The file's case count: a few hundred (case, frame, dtype, max_ctas) combinations"""
    n = n_cases()
    print('test_gpu_extent_configs: %d (case, frame, dtype, max_ctas) combinations' % n)
    assert n >= 300


# ------------------------------------------------------------------------------------------------------------------ coverage
def _key(case):
    N, H, W, Cin, Cout, k, s, relu, res, gn, tail, ds = case
    return (Cin, Cout, k, s, relu, res, gn, tail, ds)


def test_case_table_covers_every_extent_build():
    """Every conv row pins what the configurator picks at its capacity; the table spans every EXT = true build the launch dispatch of
    conv_umma.cu reaches, and every configuration the full-size files pin."""
    import test_gpu_conv48
    import test_gpu_conv_configs
    import test_gpu_conv_solo
    builds = set()
    keys = []
    for case, want in CONV_CASES:
        N, H, W, Cin, Cout, k, s, relu, res, gn, tail, ds = case
        q = nat.conv_query(N, H, W, Cin, conv_out(H, k, s), conv_out(W, k, s), Cout, k, s, tail, Cout if ds else 0)
        assert (q['cc'], q['weights_resident'], q['stages'], q['schedule']) == want, (case, q)
        keys.append(_key(case) + (want[3],) + (((N, H, W),) if want[3] == 'solo' else ()))   # solo rows: as many tiles as the solo file's
        mode = _mode(k, s)
        if want[3] == 'solo':
            builds.add('conv_umma_solo_kernel<F16, true>')
        elif Cout == 48:
            builds.add('conv_umma_c48_kernel<%s, F16, true, %s>' % (mode, 'true' if ds else 'false'))
        else:
            builds.add('conv_umma_kernel<%s, %d, F16, true, %s>' % (mode, Cout, 'true' if ds else 'false'))
        if k == 3:      # a frame at which a capacity-interior tile's halo reaches past the frame
            X.halo_extent(case)
    assert len(set(keys)) == len(keys), 'two rows of one configuration'
    for c in STEM_CASES:
        builds.add('conv_umma_c48_kernel<stem, F16, true, false>' if c[0] == 48 else 'conv_umma_kernel<stem, %d, F16, true, false>' % c[0])
    want_builds = {'conv_umma_kernel<%s, %d, F16, true, false>' % (m, c) for m in (MODE_FLAT, MODE_1X1S2) for c in (16, 32, 64, 128)}
    want_builds |= {'conv_umma_kernel<%s, %d, F16, true, false>' % (m, c) for m in (MODE_3X3S1, MODE_3X3S2) for c in (32, 64, 128)}
    want_builds |= {'conv_umma_kernel<%s, %d, F16, true, true>' % (MODE_3X3S2, c) for c in (32, 64, 128)}
    want_builds |= {'conv_umma_kernel<stem, %d, F16, true, false>' % c for c in (16, 32, 64)}
    want_builds |= {'conv_umma_c48_kernel<%s, F16, true, false>' % m for m in (MODE_FLAT, MODE_1X1S2, MODE_3X3S1, MODE_3X3S2, MODE_STEM)}
    want_builds |= {'conv_umma_c48_kernel<3x3s2, F16, true, true>', 'conv_umma_solo_kernel<F16, true>'}
    assert builds == want_builds, (sorted(want_builds - builds), sorted(builds - want_builds))
    # every configuration the full-size files pin, once
    full = {_key(c) + ('shared',) for c, _ in test_gpu_conv_configs.CASES} | {_key(c) + ('shared',) for c in test_gpu_conv48.CASES}
    full |= {(64, 64, 3, 1, relu, res, 0, 0, 0, 'solo', (N, H, W)) for N, H, W, relu, res in test_gpu_conv_solo.CASES}
    assert set(keys) == full, (sorted(full - set(keys)), sorted(set(keys) - full))
    pinned = {_key(c): w for c, w in test_gpu_conv_configs.CASES}
    for case, want in CONV_CASES:
        if _key(case) in pinned:
            assert want[:3] == pinned[_key(case)], case
    # STEM0: every (Cout, tail) of the full-size files, once; every input format; a non-trivial transform on uint8 and on NV12
    stems = [(c[0], c[1]) for c in STEM_CASES]
    assert len(set(stems)) == len(stems)
    assert set(stems) == {c[:2] for c in test_gpu_conv_configs.STEM_CASES} | {c[:2] for c in test_gpu_conv48.STEM_CASES}
    assert {c[2] for c in STEM_CASES} == {'f32', 'u8', 'nv12'}
    assert {(c[2], c[3]) for c in STEM_CASES if c[3]} >= {('u8', 'rgb-standard'), ('u8', 'caffe'), ('nv12', 'rgb-standard'), ('nv12', 'caffe')}
    assert all(c[5] >= 64 and c[6] >= 33 for c in STEM_CASES)
    # STEM4: stem4_kernel<F16, true> from uint8 with the word loader on and off, fp32 and NV12
    loaders = {(c[0], c[0] != 'f32' and c[4] % 4 == 0 and bool(c[1])) for c in STEM4_CASES}
    assert len(loaders) == len(STEM4_CASES)
    assert loaders == {('u8', True), ('u8', False), ('f32', False), ('nv12', True)}, loaders
    assert {c[0] for c in GN_CASES} == {16, 32, 64, 128} and len(GN_CASES) == 4
    heads = {(c[0] + c[1], bool(c[2])) for c in HEAD_CASES}
    assert len(heads) == len(HEAD_CASES) and heads == {(n, gn) for n in (1, 4, 11) for gn in (False, True)}


# ------------------------------------------------------------------------------------------------------------------ shared checks
def _launch(kind, case, dtype, h, w, max_ctas=0, full=False):
    """One launch at frame h x w: through the plan with a geometry row (full=False) or on tensors of the frame's size (full=True).
    -> (rig, outputs); the bytes outside the op's outputs are checked."""
    spec = _spec(kind, case, dtype)
    H, W = (h, w) if full else _capacity(kind, case)
    rig = X.Rig(spec, H, W, max_ctas=max_ctas, plan=not full)
    try:
        rig.load(h, w)
        rig.run(h, w)
        rig.assert_untouched('%s %s %s %dx%d max_ctas=%d%s' % (kind, case, dtype, h, w, max_ctas, ' full-size' if full else ''))
        outs = spec.outputs(rig, h, w) if kind == 'head' else spec.outputs(rig)
    finally:
        rig.close()
    return rig, outs


def _same_bits(a, b, what):
    ba, bb = X.bits(a), X.bits(b)
    if not torch.equal(ba, bb):
        bad = ba != bb
        i = tuple(torch.nonzero(bad)[0].tolist())
        raise AssertionError('%s: %d of %d elements differ, first at %s: %r vs %r' % (what, int(bad.sum()), bad.numel(), i, float(a[i]), float(b[i])))


def _stats_equal(a, b, out, what):
    """fp64 statistics equal up to the order of the fp64 atomics"""
    o = out.cpu().double().reshape(out.shape[0], -1, a.shape[1], out.shape[-1] // a.shape[1])
    mag = torch.stack([o.abs().sum(dim=(1, 3)), (o * o).sum(dim=(1, 3))], -1)
    assert bool(((a.cpu() - b.cpu()).abs() <= 1e-12 * mag + 1e-300).all()), what


def _check_spatial(kind, case, dtype):
    """conv / STEM0 / STEM4: values, bits against the full-size launch and across grids, statistics, memory hygiene"""
    spec = _spec(kind, case, dtype)
    for h, w, why in _extents(kind, case):
        ho, wo = spec.out_size(h, w)
        ref = spec.reference(h, w)
        _, want = _launch(kind, case, dtype, h, w, full=True)
        first = None
        for m in GRIDS:
            _, got = _launch(kind, case, dtype, h, w, max_ctas=m)
            what = '%s %s %s frame %dx%d (%s) max_ctas=%d' % (kind, case, dtype, h, w, why, m)
            for name in ('out', 'ds'):
                if name not in got:
                    continue
                valid = got[name][:, :ho, :wo]
                r, S, K = ref[name]
                if S is None:
                    assert_tail_close(valid, r, dtype, what + ' ' + name)
                else:
                    assert_faithful(valid, r, S, K, dtype, what + ' ' + name)
                _same_bits(valid, want[name], what + ' ' + name + ' against the full-size launch')
                X.assert_untouched_beyond_tiles(got[name], ho, wo, spec.flat, what + ' ' + name)
                if first is not None:
                    _same_bits(valid, first[name][:, :ho, :wo], what + ' ' + name + ' against the default grid')
            if 'stats' in got:
                valid = got['out'][:, :ho, :wo]
                assert_gn_stats(got['stats'], valid, case[9], what + ' statistics')
                if spec.flat:
                    # a flat tile's fp32 partial sums cover 128 consecutive pixels at the capacity pitch, a full-size launch's at the
                    # frame's: other groupings of the same terms, within the fp32 bound of assert_gn_stats of each other (~1e-8 here)
                    assert_gn_stats(want['stats'], valid, case[9], what + ' statistics of the full-size launch')
                else:
                    _stats_equal(got['stats'], want['stats'], valid, what + ' statistics against the full-size launch')
                if first is not None:       # the same tiles: only the order of the fp64 atomics differs
                    _stats_equal(got['stats'], first['stats'], valid, what + ' statistics against the default grid')
            if first is None:
                first = got


@pytest.mark.parametrize('dtype', DTYPE_NAMES)
@pytest.mark.parametrize('case', [c for c, _ in CONV_CASES], ids=conv_id)
def test_conv_below_capacity(case, dtype):
    _check_spatial('conv', case, dtype)


@pytest.mark.parametrize('dtype', DTYPE_NAMES)
@pytest.mark.parametrize('case', STEM_CASES, ids=stem_id)
def test_stem0_below_capacity(case, dtype):
    _check_spatial('stem', case, dtype)


@pytest.mark.parametrize('dtype', DTYPE_NAMES)
@pytest.mark.parametrize('case', STEM4_CASES, ids=stem4_id)
def test_stem4_below_capacity(case, dtype):
    _check_spatial('stem4', case, dtype)


@pytest.mark.parametrize('dtype', DTYPE_NAMES)
@pytest.mark.parametrize('case', GN_CASES, ids=gn_id)
def test_gn_apply_below_capacity(case, dtype):
    """The valid region is round16(relu(gamma (x - mean) rstd + beta)) with the statistics counted over h * w pixels (either float rstd
    of head_activation); rows at and below h are never written (GN_APPLY walks the first h rows at the capacity pitch)."""
    spec = _spec('gn', case, dtype)
    for h, w, why in _extents('gn', case):
        a, a_b = spec.reference(h, w)
        _, want = _launch('gn', case, dtype, h, w, full=True)
        first = None
        for m in GRIDS:
            _, got = _launch('gn', case, dtype, h, w, max_ctas=m)
            what = 'gn_apply %s %s frame %dx%d (%s) max_ctas=%d' % (case, dtype, h, w, why, m)
            out = got['out']
            valid = out[:, :h, :w]
            v = valid.cpu().double()
            ok = (v == a) | (v == a_b)
            assert bool(ok.all()), '%s: %d of %d elements off' % (what, int((~ok).sum()), ok.numel())
            _same_bits(valid, want['out'], what + ' against the full-size launch')
            X.assert_poison(out[:, h:], what + ' below the frame')
            if first is not None:
                _same_bits(out, first, what + ' against the default grid')
            else:
                first = out


@pytest.mark.parametrize('dtype', DTYPE_NAMES)
@pytest.mark.parametrize('case', HEAD_CASES, ids=head_id)
def test_head_final_below_capacity(case, dtype):
    """cls / reg of point n P + FRAME_PRE + y w + x against float64 on the activations of the valid pixels; every other point of the
    frame's N P (the other levels) and every point beyond them keeps its NaN."""
    n_cls, n_reg = case[0], case[1]
    spec = _spec('head', case, dtype)
    for h, w, why in _extents('head', case):
        ref, S, K = spec.reference(h, w)
        _, want = _launch('head', case, dtype, h, w, full=True)
        first = None
        lo, hi = X.FRAME_PRE, X.FRAME_PRE + h * w
        for m in GRIDS:
            _, (cls, reg, cls_rest, reg_rest) = _launch('head', case, dtype, h, w, max_ctas=m)
            what = 'head_final %s %s frame %dx%d (%s) max_ctas=%d' % (case, dtype, h, w, why, m)
            if n_cls:
                check_within(cls[:, lo:hi, :n_cls].cpu(), ref[..., :n_cls].cpu(), S[..., :n_cls].cpu(), K, what + ' cls')
                _same_bits(cls[:, lo:hi], want[0][:, lo:hi], what + ' cls against the full-size launch')
            if n_reg:
                check_within(reg[:, lo:hi].cpu(), ref[..., n_cls:].cpu(), S[..., n_cls:].cpu(), K, what + ' reg')
                _same_bits(reg[:, lo:hi], want[1][:, lo:hi], what + ' reg against the full-size launch')
            for name, t, rest in (('cls', cls, cls_rest), ('reg', reg, reg_rest)):
                if (name == 'cls' and n_cls) or (name == 'reg' and n_reg):
                    X.assert_poison(t[:, :lo], what + ' ' + name + ' of the levels before')
                    X.assert_poison(t[:, hi:], what + ' ' + name + ' of the levels after')
                else:
                    X.assert_poison(t, what + ' ' + name + ' (no outputs of this kind)')
                X.assert_poison(rest, what + ' ' + name + ' beyond N P of the frame')
            if first is not None:
                _same_bits(cls, first[0], what + ' cls against the default grid')
                _same_bits(reg, first[1], what + ' reg against the default grid')
            else:
                first = (cls, reg)


# ------------------------------------------------------------------------------------------------------------------ one graph
GRAPH_CASES = [('conv', CONV_CASES[3][0]), ('conv', CONV_CASES[10][0]), ('conv', CONV_CASES[14][0]), ('conv', CONV_CASES[21][0]),
               ('conv', CONV_CASES[36][0]), ('stem', STEM_CASES[2]), ('stem4', STEM4_CASES[0]), ('head', HEAD_CASES[2])]


@pytest.mark.parametrize('kind,case', GRAPH_CASES, ids=['%s-%d' % (k, i) for i, (k, _) in enumerate(GRAPH_CASES)])
def test_graph_replays_every_extent(kind, case):
    """One plan, captured once: replays over a scrambled sequence of frames (each twice) give, bit for bit, what the eager launch of the
    same frame gives.  The table reaches the graph through a fixed device pointer filled from a 4-slot pinned ring."""
    dtype = 'bf16'
    spec = _spec(kind, case, dtype)
    H, W = _capacity(kind, case)
    rig = X.Rig(spec, H, W)
    try:
        frames = [(h, w) for h, w, _ in _extents(kind, case)] * 2
        random.Random(len(frames) + H).shuffle(frames)
        eager = {}
        for h, w in frames:
            if (h, w) not in eager:
                rig.load(h, w)
                rig.run(h, w, use_graph=0)
                eager[(h, w)] = _snapshot(kind, spec, rig, h, w)
        for h, w in frames:
            rig.load(h, w)
            rig.run(h, w, use_graph=1)
            got = _snapshot(kind, spec, rig, h, w)
            for a, b in zip(got, eager[(h, w)]):
                if a.dtype == torch.float64:
                    assert torch.allclose(a, b, rtol=1e-12, atol=0), (kind, case, h, w, 'statistics')
                else:
                    _same_bits(a, b, '%s %s graph replay at %dx%d' % (kind, case, h, w))
        assert nat.lib().lfd_plan_num_graphs(rig.handle) == 1
    finally:
        rig.close()


def _snapshot(kind, spec, rig, h, w):
    if kind == 'head':
        return spec.outputs(rig, h, w)
    o = spec.outputs(rig)
    return [o[k] for k in sorted(o)]
