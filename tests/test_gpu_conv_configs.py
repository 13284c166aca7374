# -*- coding: utf-8 -*-
"""The forward conv kernels at op level, at every configuration the configurator can choose (mode x output width, channel chunk
Cc, resident / streamed weights, ring depth, fused tail width, fused 1x1/s2 shortcut, GroupNorm statistics) and under schedules
that make every CTA walk several tiles, against a float64 CPU evaluation of the same operation on the same 16-bit operands.
Also the stem conv (LFD_OP_STEM0) and the fused four-conv stem (LFD_OP_STEM4) as ops."""
import ctypes as C
import functools

import pytest
import torch

from gpu_ops import (DTYPES, STEM_FMT, assert_faithful, assert_gn_stats, assert_tail_close, conv_out, conv_reference, ref_conv64, run_conv,
                     run_conv_case, run_stem0, stem_input, stem_operands)
from helpers import bits
from lfd import _native as nat

MODE_FLAT, MODE_3X3S1, MODE_3X3S2, MODE_1X1S2, MODE_STEM = 'flat', '3x3s1', '3x3s2', '1x1s2', 'stem'


def _mode(k, s):
    return {(1, 1): MODE_FLAT, (3, 1): MODE_3X3S1, (3, 2): MODE_3X3S2, (1, 2): MODE_1X1S2}[(k, s)]


# (N, H, W, Cin, Cout, k, s, relu, res, gn, tail, ds) -> (cc, weights_resident, stages) the configurator picks
CASES = [
    ((2, 23, 31, 16, 16, 1, 1, 1, 0, 0, 0, 0), (16, 1, 8)),        # Cout 16, Cc 16 from Cin 16
    ((2, 23, 31, 48, 32, 1, 1, 1, 1, 0, 0, 0), (16, 1, 8)),        # Cc 16 from Cin 48 (3 chunks), residual
    ((2, 23, 31, 96, 64, 1, 1, 0, 1, 0, 0, 0), (32, 1, 4)),        # Cc 32, three chunks
    ((2, 23, 31, 128, 128, 1, 1, 0, 0, 16, 0, 0), (64, 1, 4)),     # GroupNorm statistics
    ((2, 23, 31, 32, 32, 1, 1, 1, 0, 0, 16, 0), (32, 1, 4)),       # tail 16
    ((2, 23, 31, 128, 64, 1, 1, 1, 0, 0, 32, 0), (64, 1, 4)),      # tail 32, two chunks
    ((2, 23, 31, 64, 128, 1, 1, 1, 0, 16, 128, 0), (64, 1, 4)),    # tail 128 + GroupNorm statistics of the tail output
    ((2, 45, 61, 64, 16, 1, 2, 0, 0, 0, 0, 0), (64, 1, 4)),        # 1x1/s2, Cout 16, odd x odd input
    ((2, 44, 62, 64, 32, 1, 2, 0, 1, 0, 0, 0), (64, 1, 4)),        # even x even input, residual
    ((2, 45, 61, 48, 64, 1, 2, 1, 0, 0, 0, 0), (16, 1, 8)),
    ((2, 44, 61, 128, 128, 1, 2, 0, 0, 16, 0, 0), (64, 1, 4)),
    ((2, 45, 80, 16, 32, 3, 1, 1, 1, 0, 0, 0), (16, 1, 8)),        # Cc 16 from Cin 16, 60 tiles
    ((2, 23, 31, 32, 64, 3, 1, 1, 0, 0, 0, 0), (32, 1, 4)),
    ((2, 31, 40, 96, 128, 3, 1, 1, 1, 0, 0, 0), (16, 0, 3)),       # streamed weights, 6 chunks per tile
    ((2, 31, 40, 128, 128, 3, 1, 0, 0, 16, 0, 0), (16, 0, 3)),     # streamed, 8 chunks per tile, GroupNorm statistics
    ((2, 37, 29, 64, 64, 3, 1, 1, 1, 0, 128, 0), (64, 1, 3)),      # tail 128 with a residual on the tail output
    ((2, 45, 61, 32, 32, 3, 2, 1, 0, 0, 0, 0), (32, 1, 4)),        # stride 2, odd x odd input
    ((2, 45, 80, 48, 64, 3, 2, 1, 0, 0, 0, 0), (16, 1, 4)),        # Cc 16 from Cin 48
    ((2, 44, 62, 64, 128, 3, 2, 1, 0, 0, 0, 0), (16, 0, 3)),       # even x even input, streamed
    ((2, 45, 80, 64, 64, 3, 2, 1, 0, 0, 64, 0), (32, 1, 3)),       # tail 64 (stem2 + stem3 pattern)
    ((2, 45, 80, 32, 32, 3, 2, 1, 0, 0, 0, 32), (32, 1, 4)),       # fused 1x1/s2 shortcut, Cout 32
    ((2, 45, 61, 64, 64, 3, 2, 1, 0, 0, 0, 64), (32, 1, 3)),       # shortcut 64 -> 64, resident
    ((2, 44, 80, 64, 128, 3, 2, 1, 0, 0, 0, 128), (16, 0, 3)),     # shortcut 64 -> 128, streamed
    ((2, 45, 80, 128, 128, 3, 2, 1, 0, 0, 0, 128), (16, 0, 2)),    # shortcut 128 -> 128, streamed, 2-stage ring
]

# (Cout, tail, fmt, H, W): every output width, without a tail and with every tail width; H and W = 0, 1, 2, 3 (mod 4), tall enough
# for interior tiles (a whole 33 x 18 image patch in range) as well as border tiles
STEM_CASES = [
    (16, 0, 'u8', 100, 124), (16, 16, 'f32', 101, 125), (16, 32, 'u8', 102, 126), (16, 64, 'f32', 103, 127), (16, 128, 'u8', 101, 126),
    (32, 0, 'f32', 101, 127), (32, 16, 'u8', 102, 124), (32, 32, 'f32', 103, 125), (32, 64, 'u8', 100, 126), (32, 128, 'f32', 102, 127),
    (64, 0, 'u8', 103, 126), (64, 16, 'f32', 100, 125), (64, 32, 'u8', 101, 124), (64, 64, 'f32', 102, 126), (64, 128, 'u8', 103, 124),
]


def _id(c):
    c = c[0] if isinstance(c[0], tuple) else c
    N, H, W, Cin, Cout, k, s, relu, res, gn, tail, ds = c
    return 'N%d_%dx%d_%d-%d_k%ds%d_r%d_res%d_gn%d_tail%d_ds%d' % c


def _stem_id(c):
    return 'c%d_tail%d_%s_%dx%d' % c


def _query(case):
    N, H, W, Cin, Cout, k, s, relu, res, gn, tail, ds = case
    return nat.conv_query(N, H, W, Cin, conv_out(H, k, s), conv_out(W, k, s), Cout, k, s, tail, ds)


def test_case_table_covers_every_configuration():
    modes, ccs, residency, stages, tails, shortcuts, gn = set(), set(), set(), set(), set(), {}, set()
    for case, want in CASES:
        N, H, W, Cin, Cout, k, s, relu, res, g, tail, ds = case
        q = _query(case)
        assert (q['cc'], q['weights_resident'], q['stages']) == want, (case, q)
        assert q['num_tiles'] >= 12, (case, q)      # 3 CTAs with >= 4 tiles each
        modes.add((_mode(k, s), Cout))
        ccs.add(q['cc'])
        residency.add(q['weights_resident'])
        stages.add(q['stages'])
        if tail:
            tails.add(tail)
        if ds:
            shortcuts[(Cin, Cout)] = want
        if g:
            gn.add('tail' if tail else 'plain')
    modes |= {(MODE_STEM, c[0]) for c in STEM_CASES}
    launchable = {(m, c) for m in (MODE_FLAT, MODE_1X1S2) for c in (16, 32, 64, 128)} | {(MODE_STEM, c) for c in (16, 32, 64)} | \
                 {(m, c) for m in (MODE_3X3S1, MODE_3X3S2) for c in (32, 64, 128)}
    assert launchable <= modes, launchable - modes
    assert {16, 32, 64} <= ccs and residency == {0, 1} and 2 in stages
    assert {16, 32, 64, 128} <= tails
    assert {c for _, c in shortcuts} >= {32, 64, 128}
    assert shortcuts[(64, 128)] == (16, 0, 3) and shortcuts[(128, 128)] == (16, 0, 2)
    assert gn == {'plain', 'tail'}
    assert {c[1] for c in STEM_CASES} == {0, 16, 32, 64, 128}
    assert {c[3] % 4 for c in STEM_CASES} == {0, 1, 2, 3} and {c[4] % 4 for c in STEM_CASES} == {0, 1, 2, 3}
    # the stem producer skips its bounds checks on interior tiles: tile (1, 1) reads image rows 31..63 and columns 15..32
    assert all(c[3] >= 64 and c[4] >= 33 for c in STEM_CASES)


def _seed(case):
    return hash(case) & 0xffff


@pytest.mark.gpu
@pytest.mark.parametrize('max_ctas', [0, 3])
@pytest.mark.parametrize('dtype', ['bf16', 'fp16'])
@pytest.mark.parametrize('case', [c for c, _ in CASES], ids=_id)
def test_conv_config_matches_fp64(case, dtype, max_ctas):
    N, H, W, Cin, Cout, k, s, relu, use_res, gn, tail, ds = case
    out, stats, q, out3 = run_conv_case(case, dtype, _seed(case), max_ctas)
    if max_ctas:
        assert q['num_tiles'] // max_ctas >= 4
    (ref, S, K), short = conv_reference(case, dtype, _seed(case))
    what = 'conv %s %s max_ctas=%d (plan %s)' % (_id(case), dtype, max_ctas, q)
    if tail:
        assert_tail_close(out, ref, dtype, what)
    else:
        assert_faithful(out, ref, S, K, dtype, what)
    if ds:
        assert_faithful(out3, short[0], short[1], short[2], dtype, what + ' shortcut')
    if gn:
        assert_gn_stats(stats, out, gn, what)


def _assert_stats_equal(a, b, out, what):
    o = out.cpu().double().reshape(out.shape[0], -1, a.shape[1], out.shape[-1] // a.shape[1])
    mag = torch.stack([o.abs().sum(dim=(1, 3)), (o * o).sum(dim=(1, 3))], -1)
    assert bool(((a.cpu() - b.cpu()).abs() <= 1e-12 * mag + 1e-300).all()), what


@pytest.mark.gpu
@pytest.mark.parametrize('case', [c for c, _ in CASES], ids=_id)
def test_grid_does_not_change_the_output(case):
    """Tiles are strided by gridDim: any grid size gives the same stored bits (statistics: the same sums up to the order of the
    fp64 atomics)."""
    runs = [run_conv_case(case, 'bf16', _seed(case), m) for m in (1, 2, 7, 0)]
    out0, st0, _, sc0 = runs[-1]
    for m, (out, st, _, sc) in zip((1, 2, 7), runs[:-1]):
        assert torch.equal(bits(out), bits(out0)), 'max_ctas=%d changes %d output elements' % (m, int((out != out0).sum()))
        if sc is not None:
            assert torch.equal(bits(sc), bits(sc0)), 'max_ctas=%d changes the shortcut output' % m
        if st is not None:
            _assert_stats_equal(st, st0, out0, 'max_ctas=%d statistics' % m)


# ------------------------------------------------------------------------------------------------ GroupNorm statistics + ReLU + residual
@pytest.mark.gpu
@pytest.mark.parametrize('impl,tail', [(nat.CONV_UMMA, False), (nat.CONV_UMMA, True), (nat.CONV_SIMT, False)], ids=['umma', 'umma-tail', 'simt'])
def test_gn_statistics_conv_honours_relu_and_residual(impl, tail):
    """A conv with GroupNorm statistics stores conv + shift + res -> ReLU -> round16, and its statistics are those of that stored
    tensor, whatever the implementation and with or without a fused tail."""
    dtype = 'bf16'
    N, H, W, Cin, Cmid = 2, 23, 31, 64, 128 if not tail else 64
    g = torch.Generator().manual_seed(21)
    x = torch.randn((N, H, W, Cin), generator=g).to(torch.bfloat16)
    w = torch.randn((Cmid, Cin, 3, 3), generator=g) * (2.0 / (Cin * 9)) ** 0.5
    scale, shift = torch.rand((Cmid,), generator=g) + 0.5, torch.randn((Cmid,), generator=g) * 0.2
    res = torch.randn((N, H, W, 128), generator=g).to(torch.bfloat16)
    t = None
    if tail:
        t = (torch.randn((128, Cmid, 1, 1), generator=g) * (2.0 / Cmid) ** 0.5, torch.rand((128,), generator=g) + 0.5,
             torch.randn((128,), generator=g) * 0.2, True)
    out, stats, q = run_conv(x.cuda(), w, scale, shift, 1, True, res=res.cuda(), gn_groups=16, impl=impl, tail=t, dtype=dtype)
    if tail:
        mid, _, _ = ref_conv64(x, w, scale, shift, 1, True, dtype=dtype)
        ref, S, K = ref_conv64(DTYPES[dtype][1](mid.float()), t[0], t[1], t[2], 1, True, res=res, dtype=dtype)
        assert_tail_close(out, ref, dtype, 'GroupNorm conv + tail with ReLU and residual')
    else:
        ref, S, K = ref_conv64(x, w, scale, shift, 1, True, res=res, dtype=dtype)
        assert_faithful(out, ref, S, K, dtype, 'GroupNorm conv with ReLU and residual')
    assert float(out.float().min()) >= 0.0
    assert_gn_stats(stats, out, 16, 'statistics of the stored tensor')


# ------------------------------------------------------------------------------------------------ STEM0 as an op
def _stem_seed(case):
    Cout, tail, fmt, H, W = case
    return Cout * 1000 + tail * 10 + H + W


def _run_stem(case, dtype, max_ctas):
    img, w, shift, t = stem_operands(case, _stem_seed(case))
    return run_stem0(img.cuda(), STEM_FMT[case[2]], w, shift, tail=t, max_ctas=max_ctas, dtype=dtype)


@pytest.mark.gpu
@pytest.mark.parametrize('max_ctas', [0, 3])
@pytest.mark.parametrize('dtype', ['bf16', 'fp16'])
@pytest.mark.parametrize('case', STEM_CASES, ids=_stem_id)
def test_stem0_matches_fp64(case, dtype, max_ctas):
    Cout, tail, fmt, H, W = case
    img, w, shift, t = stem_operands(case, _stem_seed(case))
    out, num_tiles = _run_stem(case, dtype, max_ctas)
    if max_ctas:
        assert num_tiles // max_ctas >= 4
    x = stem_input(img, fmt, dtype)
    ones = torch.ones(Cout)
    what = 'stem0 %s %s max_ctas=%d' % (_stem_id(case), dtype, max_ctas)
    if tail:
        mid, _, _ = ref_conv64(x, w, ones, shift, 2, True, dtype=dtype)
        ref, _, _ = ref_conv64(DTYPES[dtype][1](mid.float()), t[0], t[1], t[2], 1, True, dtype=dtype)
        assert_tail_close(out, ref, dtype, what)
    else:
        ref, S, K = ref_conv64(x, w, ones, shift, 2, True, dtype=dtype)
        assert_faithful(out, ref, S, K, dtype, what)


@pytest.mark.gpu
@pytest.mark.parametrize('case', STEM_CASES, ids=_stem_id)
def test_stem0_grid_does_not_change_the_output(case):
    outs = [_run_stem(case, 'bf16', m)[0] for m in (1, 2, 7, 0)]
    for m, o in zip((1, 2, 7), outs[:-1]):
        assert torch.equal(bits(o), bits(outs[-1])), 'max_ctas=%d changes %d stem elements' % (m, int((o != outs[-1]).sum()))


# ------------------------------------------------------------------------------------------------ STEM4 as an op
STEM4_SIZES = [(60, 127), (61, 126), (62, 125), (63, 124)]      # H and W = 0, 1, 2, 3 (mod 4): every offset of the stem1-map border


@functools.lru_cache(maxsize=None)
def _stem4_plan(h, w, dtype):
    from helpers import synth_model
    from lfd._engine import InferencePlan
    model, _ = synth_model('WIDERFACE_S')
    model.cuda()
    plan = InferencePlan(model, 2, h, w, torch.device('cuda'), act_dtype=dtype, fuse_stem=True)
    assert plan._ops[0]['kind'] == nat.OP_STEM4
    return model, plan


def _run_stem4(plan, img, fmt, max_ctas):
    op = nat.Op.from_buffer_copy(plan._op_array[0])
    op.max_ctas = max_ctas
    out = plan.tensor(plan._ops[0]['out'])
    out.view(torch.int16).fill_(-1)                 # NaN pattern: a tile that is not stored cannot pass
    with torch.cuda.device(plan.workspace.device):
        nat.check(nat.lib().lfd_run_op(C.byref(op), nat.ptr(img), nat.INPUT_U8_NHWC if fmt == 'u8' else nat.INPUT_F32_NCHW,
                                       nat.ptr(plan.workspace), None, None, 0, 0, nat.CONV_UMMA, nat.stream_ptr()))
        torch.cuda.synchronize()
    return out.clone()


@pytest.mark.gpu
@pytest.mark.parametrize('fmt', ['u8', 'f32'])
@pytest.mark.parametrize('h,w', STEM4_SIZES)
def test_stem4_matches_fp64_chain_and_is_grid_invariant(h, w, fmt):
    from lfd._engine import InferencePlan
    dtype = 'bf16'
    model, plan = _stem4_plan(h, w, dtype)
    g = torch.Generator().manual_seed(h * 1000 + w)
    img = torch.randint(0, 256, (2, h, w, 3), generator=g, dtype=torch.uint8) if fmt == 'u8' else torch.randn((2, 3, h, w), generator=g)
    outs = [_run_stem4(plan, img.cuda().contiguous(), fmt, m) for m in (1, 3, 0)]
    q = nat.stem4_query(2, h, w)
    assert q['num_tiles'] >= 3
    for m, o in zip((1, 3), outs[:-1]):
        assert torch.equal(bits(o), bits(outs[-1])), 'stem4 max_ctas=%d changes %d elements' % (m, int((o != outs[-1]).sum()))
    rnd = DTYPES[dtype][1]
    t = stem_input(img, fmt, dtype)
    for conv, norm, relu in model._backbone.stem_layers():
        scale, shift = InferencePlan._fold(conv, norm)
        ref, _, _ = ref_conv64(t, conv.weight.detach().cpu(), scale, shift, conv.stride[0], bool(relu), dtype=dtype)
        t = rnd(ref.float())                         # every intermediate is rounded to 16 bits, as the kernel rounds it
    assert_tail_close(outs[-1], ref, dtype, 'stem4 %dx%d %s' % (h, w, fmt))
