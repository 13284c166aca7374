# -*- coding: utf-8 -*-
"""The 48-channel forward convs (conv_umma_c48_kernel, and the SIMT cross-check kernels) at op level against a float64 CPU evaluation
of the same operation on the same 16-bit operands, with the faithful bound of test_gpu_conv_configs.py: |out - y| <= ulp16(y) +
K 2^-24 S.

A 48-channel tensor has 96-byte pixel rows.  Every tensor the op reads or writes sits in a NaN-filled workspace, with NaN guard bytes
behind it: a store that wrote past channel 47 of a pixel would overwrite the next pixel's channels (or the guard) and a residual load
that read past it would carry a NaN into the sum.  The outputs must be finite, the guards untouched."""
import ctypes as C
import functools

import pytest
import torch

from gpu_ops import DTYPES, assert_faithful, assert_tail_close, conv_out, ref_conv64, stem_input
from lfd import _native as nat
from lfd._engine import fold_scale, pack_conv_weight, pack_stem_weight

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
GUARD = 4096


def _id(c):
    return 'N%d_%dx%d_%d-%d_k%ds%d_r%d_res%d_gn%d_tail%d_ds%d' % c


def _stem_id(c):
    return 'c%d_tail%d_%s_%dx%d' % c


def _bits(t):
    return t.contiguous().view(torch.int16).cpu()


def _nan_ws(total, dtype, dev):
    ws = torch.empty(total // 2, dtype=DTYPES[dtype][0], device=dev)
    ws.fill_(float('nan'))
    return ws.view(torch.uint8)


def _assert_guards(ws, regions, dtype, what):
    """Every byte of ws outside the regions the op owns is still the NaN pattern"""
    v = ws.view(DTYPES[dtype][0])
    mask = torch.ones(v.numel(), dtype=torch.bool, device=ws.device)
    for off, nb in regions:
        mask[off // 2:(off + nb) // 2] = False
    outside = v[mask]
    assert bool(torch.isnan(outside).all()), '%s: %d bytes outside the tensors were written' % (what, 2 * int((~torch.isnan(outside)).sum()))


@functools.lru_cache(maxsize=None)
def _operands(case, dtype):
    N, H, W, Cin, Cout, k, s, relu, use_res, gn, tail, ds = case
    tdt = DTYPES[dtype][0]
    g = torch.Generator().manual_seed((hash(case) + 48) & 0xffff)
    x = torch.randn((N, H, W, Cin), generator=g).to(tdt)
    w = torch.randn((Cout, Cin, k, k), generator=g) * (2.0 / (Cin * k * k)) ** 0.5
    scale, shift = torch.rand((Cout,), generator=g) + 0.5, torch.randn((Cout,), generator=g) * 0.2
    Ho, Wo = conv_out(H, k, s), conv_out(W, k, s)
    res = torch.randn((N, Ho, Wo, Cout), generator=g).to(tdt) if use_res else None
    d = None
    if ds:
        d = (torch.randn((Cout, Cin, 1, 1), generator=g) * (1.0 / Cin) ** 0.5, torch.rand((Cout,), generator=g) + 0.5,
             torch.randn((Cout,), generator=g) * 0.2)
    return x, w, scale, shift, res, d


def _run(case, dtype, max_ctas, impl=nat.CONV_UMMA):
    """-> (out, shortcut out or None, conv_query); the workspace is NaN-filled and its guards are checked"""
    N, H, W, Cin, Cout, k, s, relu, use_res, gn, tail, ds = case
    x, w, scale, shift, res, d = _operands(case, dtype)
    tdt, _, _, code = DTYPES[dtype]
    dev = torch.device('cuda')
    Ho, Wo = conv_out(H, k, s), conv_out(W, k, s)
    q = nat.conv_query(N, H, W, Cin, Ho, Wo, Cout, k, s, 0, Cout if ds else 0)
    wp = pack_conv_weight(fold_scale(w, scale), q['cc'], tdt).to(dev)
    sh = shift.float().to(dev).contiguous()
    in_b, out_b = x.numel() * 2, N * Ho * Wo * Cout * 2
    al = lambda v: (v + 255) & ~255   # noqa: E731
    off_in = GUARD
    off_out = off_in + al(in_b) + GUARD
    off_res = off_out + al(out_b) + GUARD
    off_ds = off_res + al(out_b) + GUARD
    ws = _nan_ws(off_ds + al(out_b) + GUARD, dtype, dev)
    ws[off_in:off_in + in_b] = x.contiguous().view(torch.uint8).reshape(-1).to(dev)
    regions = [(off_in, in_b), (off_out, out_b)]
    if res is not None:
        ws[off_res:off_res + out_b] = res.contiguous().view(torch.uint8).reshape(-1).to(dev)
        regions.append((off_res, out_b))
    op = nat.Op()
    op.kind, op.dtype = nat.OP_CONV, code
    op.N, op.H, op.W, op.Cin, op.Ho, op.Wo, op.Cout = N, H, W, Cin, Ho, Wo, Cout
    op.ksize, op.stride, op.relu, op.gn_groups, op.cc = k, s, int(relu), 0, q['cc']
    op.in_off, op.out_off, op.res_off, op.stats_off = off_in, off_out, (off_res if res is not None else -1), -1
    op.max_ctas = max_ctas
    op.weight, op.shift = wp.data_ptr(), sh.data_ptr()
    if ds:
        w3p = pack_conv_weight(fold_scale(d[0], d[1]), Cin, tdt).to(dev)
        sh3 = d[2].float().to(dev).contiguous()
        op.ds_cout, op.ds_out_off = Cout, off_ds
        op.ds_weight, op.ds_shift = w3p.data_ptr(), sh3.data_ptr()
        regions.append((off_ds, out_b))
    nat.check(nat.lib().lfd_run_op(C.byref(op), None, 0, nat.ptr(ws), None, None, 0, 0, impl, nat.stream_ptr()))
    torch.cuda.synchronize()
    _assert_guards(ws, regions, dtype, 'conv %s' % _id(case))
    out = ws[off_out:off_out + out_b].view(tdt).view(N, Ho, Wo, Cout).clone()
    out3 = ws[off_ds:off_ds + out_b].view(tdt).view(N, Ho, Wo, Cout).clone() if ds else None
    return out, out3, q


@functools.lru_cache(maxsize=None)
def _reference(case, dtype):
    N, H, W, Cin, Cout, k, s, relu, use_res, gn, tail, ds = case
    x, w, scale, shift, res, d = _operands(case, dtype)
    main = ref_conv64(x, w, scale, shift, s, relu, res=res, dtype=dtype)
    short = ref_conv64(x[:, ::2, ::2, :], d[0], d[1], d[2], 1, False, dtype=dtype) if ds else None
    return main, short


def _impls(case):
    # the SIMT cross-check kernels have no fused shortcut: the planner runs that conv on its own there
    return [nat.CONV_UMMA] + ([] if case[11] else [nat.CONV_SIMT])


@pytest.mark.parametrize('max_ctas', [0, 3])
@pytest.mark.parametrize('dtype', ['bf16', 'fp16'])
@pytest.mark.parametrize('case', CASES, ids=_id)
def test_conv48_matches_fp64(case, dtype, max_ctas):
    (ref, S, K), short = _reference(case, dtype)
    for impl in _impls(case) if max_ctas == 0 else [nat.CONV_UMMA]:
        out, out3, q = _run(case, dtype, max_ctas, impl)
        if max_ctas:
            assert q['num_tiles'] // max_ctas >= 4
        what = 'conv48 %s %s impl=%d max_ctas=%d (plan %s)' % (_id(case), dtype, impl, max_ctas, q)
        assert bool(torch.isfinite(out.float()).all()), what + ': NaN read from outside a tensor'
        assert_faithful(out, ref, S, K, dtype, what)
        if out3 is not None:
            assert_faithful(out3, short[0], short[1], short[2], dtype, what + ' shortcut')


@pytest.mark.parametrize('case', CASES, ids=_id)
def test_conv48_grid_does_not_change_the_output(case):
    out0, sc0, _ = _run(case, 'bf16', 0)
    for m in (1, 2, 7):
        out, sc, _ = _run(case, 'bf16', m)
        assert torch.equal(_bits(out), _bits(out0)), 'max_ctas=%d changes %d output elements' % (m, int((out != out0).sum()))
        if sc is not None:
            assert torch.equal(_bits(sc), _bits(sc0)), 'max_ctas=%d changes the shortcut output' % m


# ------------------------------------------------------------------------------------------------ STEM0 48 (+ the 48 -> 48 tail)
@functools.lru_cache(maxsize=None)
def _stem_operands(case):
    Cout, tail, fmt, H, W = case
    N = 2
    g = torch.Generator().manual_seed(4800 + tail * 10 + H + W)
    img = torch.randint(0, 256, (N, H, W, 3), generator=g, dtype=torch.uint8) if fmt == 'u8' else torch.randn((N, 3, H, W), generator=g)
    w = torch.randn((Cout, 3, 3, 3), generator=g) * (2.0 / 27) ** 0.5 * (torch.rand((Cout, 1, 1, 1), generator=g) + 0.5)
    shift = torch.randn((Cout,), generator=g) * 0.2
    t = None
    if tail:
        t = (torch.randn((tail, Cout, 1, 1), generator=g) * (2.0 / Cout) ** 0.5, torch.rand((tail,), generator=g) + 0.5,
             torch.randn((tail,), generator=g) * 0.2, True)
    return img, w, shift, t


def _run_stem(case, dtype, max_ctas, impl=nat.CONV_UMMA):
    Cout, tail, fmt, H, W = case
    img, w, shift, t = _stem_operands(case)
    tdt, _, _, code = DTYPES[dtype]
    dev = torch.device('cuda')
    N = img.shape[0]
    Ho, Wo = conv_out(H, 3, 2), conv_out(W, 3, 2)
    Cf = tail or Cout
    wp = pack_stem_weight(w, tdt).to(dev)
    sh = shift.float().to(dev).contiguous()
    out_b = N * Ho * Wo * Cf * 2
    ws = _nan_ws(GUARD + ((out_b + 255) & ~255) + GUARD, dtype, dev)
    op = nat.Op()
    op.kind, op.dtype = nat.OP_STEM0, code
    op.N, op.H, op.W, op.Cin, op.Ho, op.Wo, op.Cout = N, H, W, 3, Ho, Wo, Cout
    op.ksize, op.stride, op.relu = 3, 2, 1
    op.in_off, op.out_off, op.res_off, op.stats_off = -1, GUARD, -1, -1
    op.max_ctas = max_ctas
    op.weight, op.shift = wp.data_ptr(), sh.data_ptr()
    if t is not None:
        w2p = pack_conv_weight(fold_scale(t[0], t[1]), Cout, tdt).to(dev)
        sh2 = t[2].float().to(dev).contiguous()
        op.tail_cout, op.tail_relu = Cf, 1
        op.tail_weight, op.tail_shift = w2p.data_ptr(), sh2.data_ptr()
    x = img.contiguous().to(dev)
    nat.check(nat.lib().lfd_run_op(C.byref(op), nat.ptr(x), nat.INPUT_U8_NHWC if fmt == 'u8' else nat.INPUT_F32_NCHW, nat.ptr(ws), None,
                                   None, 0, 0, impl, nat.stream_ptr()))
    torch.cuda.synchronize()
    _assert_guards(ws, [(GUARD, out_b)], dtype, 'stem %s' % _stem_id(case))
    return ws[GUARD:GUARD + out_b].view(tdt).view(N, Ho, Wo, Cf).clone(), N * ((Ho + 15) // 16) * ((Wo + 7) // 8)


@pytest.mark.parametrize('max_ctas', [0, 3])
@pytest.mark.parametrize('dtype', ['bf16', 'fp16'])
@pytest.mark.parametrize('case', STEM_CASES, ids=_stem_id)
def test_stem48_matches_fp64(case, dtype, max_ctas):
    Cout, tail, fmt, H, W = case
    img, w, shift, t = _stem_operands(case)
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
        assert torch.equal(_bits(_run_stem(case, 'bf16', m)[0]), _bits(out0)), 'stem max_ctas=%d' % m
