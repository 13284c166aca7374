# -*- coding: utf-8 -*-
"""The 64-channel 3x3/s1 convs on conv_umma_solo_kernel (one consumer warpgroup per tile, the two warpgroups' MMA phases alternating)
at op level against a float64 CPU evaluation of the same operation on the same 16-bit operands, with the faithful bound of
test_gpu_conv_configs.py: |out - y| <= ulp16(y) + K 2^-24 S.

The schedule changes which warpgroup computes a tile, never the sums: every grid gives the same bits.  Tile counts per CTA: 360 tiles
on 132 CTAs are 3 (odd) or 2 (even) per CTA, 240 tiles are 2 or 1 (a CTA whose second warpgroup gets no tile); max_ctas 1, 2, 3 and 7
give long odd and even runs.  Frames below a plan's capacity (the schedule is chosen for the capacity) leave CTAs with one tile or
none.  Every tensor sits in a NaN-filled workspace with NaN guards behind it, as in test_gpu_conv48.py."""
import ctypes as C
import functools

import pytest
import torch

from gpu_ops import DTYPES, assert_faithful, ref_conv64
from helpers import synth_model
from lfd import _native as nat
from lfd._engine import InferencePlan, fold_scale, pack_conv_weight

pytestmark = pytest.mark.gpu

# (N, H, W, relu, res): 64 -> 64 3x3/s1 convs with more tiles than the 132 CTAs
CASES = [
    (3, 90, 160, 1, 0),      # 360 tiles: 3 or 2 per CTA
    (3, 90, 160, 1, 1),
    (2, 100, 164, 0, 1),     # 294 tiles, partial tiles at the right and bottom borders
    (8, 37, 83, 0, 0),       # 264 tiles: 2 per CTA, partial tiles
    (2, 90, 160, 0, 1),      # 240 tiles: 2 or 1 per CTA
]
GRIDS = (1, 2, 3, 7)
GUARD = 4096


def _id(c):
    return 'N%d_%dx%d_r%d_res%d' % c


def _nan_ws(total, dtype, dev):
    ws = torch.empty(total // 2, dtype=DTYPES[dtype][0], device=dev)
    ws.fill_(float('nan'))
    return ws.view(torch.uint8)


@functools.lru_cache(maxsize=None)
def _operands(case, dtype):
    N, H, W, relu, use_res = case
    tdt = DTYPES[dtype][0]
    g = torch.Generator().manual_seed((hash(case) + 64) & 0xffff)
    x = torch.randn((N, H, W, 64), generator=g).to(tdt)
    w = torch.randn((64, 64, 3, 3), generator=g) * (2.0 / (64 * 9)) ** 0.5
    scale, shift = torch.rand((64,), generator=g) + 0.5, torch.randn((64,), generator=g) * 0.2
    res = torch.randn((N, H, W, 64), generator=g).to(tdt) if use_res else None
    return x, w, scale, shift, res


def _run(case, dtype, max_ctas=0, inplace=False):
    """-> (out, conv_query); inplace: the residual is read from the output tensor (out == res)"""
    N, H, W, relu, use_res = case
    x, w, scale, shift, res = _operands(case, dtype)
    tdt, _, _, code = DTYPES[dtype]
    dev = torch.device('cuda')
    q = nat.conv_query(N, H, W, 64, H, W, 64, 3, 1)
    wp = pack_conv_weight(fold_scale(w, scale), q['cc'], tdt).to(dev)
    sh = shift.float().to(dev).contiguous()
    nb = N * H * W * 64 * 2
    al = lambda v: (v + 255) & ~255   # noqa: E731
    off_in = GUARD
    off_out = off_in + al(nb) + GUARD
    off_res = off_out if inplace else off_out + al(nb) + GUARD
    ws = _nan_ws(off_res + al(nb) + GUARD, dtype, dev)
    ws[off_in:off_in + nb] = x.contiguous().view(torch.uint8).reshape(-1).to(dev)
    regions = [(off_in, nb), (off_out, nb)]
    if res is not None:
        ws[off_res:off_res + nb] = res.contiguous().view(torch.uint8).reshape(-1).to(dev)
        regions.append((off_res, nb))
    op = nat.Op()
    op.kind, op.dtype = nat.OP_CONV, code
    op.N, op.H, op.W, op.Cin, op.Ho, op.Wo, op.Cout = N, H, W, 64, H, W, 64
    op.ksize, op.stride, op.relu, op.gn_groups, op.cc = 3, 1, int(relu), 0, q['cc']
    op.in_off, op.out_off, op.res_off, op.stats_off = off_in, off_out, (off_res if res is not None else -1), -1
    op.max_ctas = max_ctas
    op.weight, op.shift = wp.data_ptr(), sh.data_ptr()
    nat.check(nat.lib().lfd_run_op(C.byref(op), None, 0, nat.ptr(ws), None, None, 0, 0, nat.CONV_UMMA, nat.stream_ptr()))
    torch.cuda.synchronize()
    v = ws.view(tdt)
    mask = torch.ones(v.numel(), dtype=torch.bool, device=dev)
    for off, n in regions:
        mask[off // 2:(off + n) // 2] = False
    assert bool(torch.isnan(v[mask]).all()), '%s: bytes outside the tensors were written' % _id(case)
    out = ws[off_out:off_out + nb].view(tdt).view(N, H, W, 64).clone()
    return out, q


@functools.lru_cache(maxsize=None)
def _reference(case, dtype):
    N, H, W, relu, use_res = case
    x, w, scale, shift, res = _operands(case, dtype)
    return ref_conv64(x, w, scale, shift, 1, relu, res=res, dtype=dtype)


@pytest.mark.parametrize('dtype', ['bf16', 'fp16'])
@pytest.mark.parametrize('case', CASES, ids=_id)
def test_solo_conv_matches_fp64_and_every_grid(case, dtype):
    out, q = _run(case, dtype)
    assert q['schedule'] == 'solo' and q['cc'] == 64 and q['weights_resident'] == 1 and q['stages'] >= 3, q
    assert bool(torch.isfinite(out).all())
    y, S, K = _reference(case, dtype)
    assert_faithful(out, y, S, K, dtype, 'solo %s %s' % (_id(case), dtype))
    for g in GRIDS:
        o2, _ = _run(case, dtype, max_ctas=g)
        assert torch.equal(o2.view(torch.int16), out.view(torch.int16)), ('max_ctas', g, _id(case), dtype)


@pytest.mark.parametrize('dtype', ['bf16', 'fp16'])
def test_solo_conv_residual_in_place(dtype):
    case = CASES[1]
    want, _ = _run(case, dtype)
    got, _ = _run(case, dtype, inplace=True)
    assert torch.equal(got.view(torch.int16), want.view(torch.int16)), dtype
    got, _ = _run(case, dtype, max_ctas=3, inplace=True)
    assert torch.equal(got.view(torch.int16), want.view(torch.int16)), dtype


def test_widerface_s_720p_b8_plan_runs_the_90x160_body_convs_solo():
    """The 64 -> 64 3x3/s1 body convs at 90 x 160 (960 tiles) and 45 x 80 (240) take the solo schedule; the ones at 23 x 40 (80 tiles),
    and every other conv, keep both warpgroups on each tile."""
    model, _ = synth_model('WIDERFACE_S')
    model.cuda()
    plan = InferencePlan(model, 8, 720, 1280, torch.device('cuda', 0))
    solo = [(r['H'], r['W']) for r in plan.describe() if r['query'] and r['query'].get('schedule') == 'solo']
    assert solo == [(90, 160)] * 7 + [(45, 80)] * 3, solo
    body = [(r['H'], r['W']) for r in plan.describe() if r['kind'] == 'conv' and (r['Cin'], r['Cout'], r['ksize'], r['stride'], r['tail_cout'])
            == (64, 64, 3, 1, 0)]
    assert sorted(set(body)) == [(23, 40), (45, 80), (90, 160)], body


def test_solo_plan_below_capacity_matches_the_plan_of_the_frame():
    """A capacity plan whose 90 x 160 and 45 x 80 body convs run solo, on frames whose maps give CTAs with one tile (the second warpgroup idle)
    or none: conv outputs bit-identical to a plan built for the frame."""
    model, _ = synth_model('WIDERFACE_S')
    model.cuda()
    cap = InferencePlan(model, 3, 720, 1280, torch.device('cuda', 0), reuse=False)     # 90 x 160 body convs: 360 tiles
    assert any(r['query'] and r['query'].get('schedule') == 'solo' for r in cap.describe())
    # 50 x 80 (120 tiles: one or none per CTA), 25 x 42, 90 x 160 with partial tiles (and their 45 x 80 / 23 x 40 stages)
    for h, w in ((720, 1280), (400, 640), (200, 330), (718, 1274)):
        g = torch.Generator().manual_seed(h * 1000 + w)
        x = torch.randint(0, 256, (3, h, w, 3), dtype=torch.uint8, generator=g).cuda()
        exact = InferencePlan(model, 3, h, w, torch.device('cuda', 0), reuse=False, fuse_stem=cap._ops[0]['kind'] == nat.OP_STEM4)
        cap.workspace.fill_(0xff)
        with torch.no_grad():
            cap.forward(x, use_graph=False)
            exact.forward(x, use_graph=False)
        torch.cuda.synchronize()
        for op in exact._ops:
            if op['kind'] == nat.OP_CONV and (op['Cin'], op['Cout'], op.get('ksize'), op.get('stride')) == (64, 64, 3, 1):
                want = exact.tensor(op['out'])
                got = cap.tensor(op['out'])[:, :want.shape[1], :want.shape[2]]
                assert torch.equal(got.view(torch.int16), want.view(torch.int16)), (h, w, op['out'])
        del exact
