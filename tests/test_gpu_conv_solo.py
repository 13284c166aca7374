# -*- coding: utf-8 -*-
"""The 64-channel 3x3/s1 convs on conv_umma_solo_kernel (one consumer warpgroup per tile, the two warpgroups' MMA phases alternating)
at op level against a float64 CPU evaluation of the same operation on the same 16-bit operands, with the faithful bound of
test_gpu_conv_configs.py: |out - y| <= ulp16(y) + K 2^-24 S.

The schedule changes which warpgroup computes a tile, never the sums: every grid gives the same bits.  Tile counts per CTA: 360 tiles
on 132 CTAs are 3 (odd) or 2 (even) per CTA, 240 tiles are 2 or 1 (a CTA whose second warpgroup gets no tile); max_ctas 1, 2, 3 and 7
give long odd and even runs.  Frames below a plan's capacity (the schedule is chosen for the capacity) leave CTAs with one tile or
none.  Every tensor sits in a NaN-filled workspace with NaN guards around it (gpu_ops.run_conv)."""
import pytest
import torch

from gpu_ops import assert_faithful, conv_reference, run_conv_case
from helpers import synth_model
from lfd import _native as nat
from lfd._engine import InferencePlan

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


def _id(c):
    return 'N%d_%dx%d_r%d_res%d' % c


def _conv(case):
    """The case as a 12-field conv case (test_gpu_conv_configs.py)"""
    N, H, W, relu, use_res = case
    return (N, H, W, 64, 64, 3, 1, relu, use_res, 0, 0, 0)


def _seed(case):
    return (hash(case) + 64) & 0xffff


@pytest.mark.parametrize('dtype', ['bf16', 'fp16'])
@pytest.mark.parametrize('case', CASES, ids=_id)
def test_solo_conv_matches_fp64_and_every_grid(case, dtype):
    out, _, q, _ = run_conv_case(_conv(case), dtype, _seed(case))
    assert q['schedule'] == 'solo' and q['cc'] == 64 and q['weights_resident'] == 1 and q['stages'] >= 3, q
    assert bool(torch.isfinite(out).all())
    (y, S, K), _ = conv_reference(_conv(case), dtype, _seed(case))
    assert_faithful(out, y, S, K, dtype, 'solo %s %s' % (_id(case), dtype))
    for g in GRIDS:
        o2 = run_conv_case(_conv(case), dtype, _seed(case), max_ctas=g)[0]
        assert torch.equal(o2.view(torch.int16), out.view(torch.int16)), ('max_ctas', g, _id(case), dtype)


@pytest.mark.parametrize('dtype', ['bf16', 'fp16'])
def test_solo_conv_residual_in_place(dtype):
    case = CASES[1]
    want = run_conv_case(_conv(case), dtype, _seed(case))[0]
    got = run_conv_case(_conv(case), dtype, _seed(case), inplace=True)[0]     # the residual is read from the output tensor
    assert torch.equal(got.view(torch.int16), want.view(torch.int16)), dtype
    got = run_conv_case(_conv(case), dtype, _seed(case), max_ctas=3, inplace=True)[0]
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
