# -*- coding: utf-8 -*-
"""The fused four-conv 'faster' stem (LFD_OP_STEM4): planner gate (CPU) and bit-identity with the two-kernel path (GPU)."""
import pytest
import torch

import synth
from helpers import synth_model, rel_err
from lfd import _native as nat
from lfd._engine import InferencePlan

CPU = torch.device('cpu')


def _conv_count(plan):
    return [r['kind'] for r in plan.describe()].count('conv')


def test_stem_fusion_follows_the_l2_gate_and_the_fuse_stem_argument():
    model, _ = synth_model('WIDERFACE_S')
    big = InferencePlan(model, 8, 720, 1280, CPU, create_native=False)
    small = InferencePlan(model, 2, 184, 248, CPU, create_native=False)
    row = big.describe()[0]
    assert big._ops[0]['kind'] == nat.OP_STEM4 and row['kind'] == 'stem0' and row['fused_stem'] == 4
    assert (row['H'], row['W'], row['Ho'], row['Wo'], row['Cout'], row['tail_cout']) == (720, 1280, 180, 320, 64, 64)
    assert _conv_count(big) == _conv_count(small) - 1
    # 2.9 MB of stem1 stays in L2: the small plan keeps the two fused pairs
    assert [o['kind'] for o in small._ops[:2]] == [nat.OP_STEM0, nat.OP_CONV] and small._ops[0]['tail_cout'] == 64
    assert all(o['kind'] != nat.OP_STEM4 for o in small._ops)
    # fuse_stem=False restores the two launches; the fused plan needs no stem1 buffer
    unfused = InferencePlan(model, 8, 720, 1280, CPU, create_native=False, fuse_stem=False)
    assert unfused._ops[0]['kind'] == nat.OP_STEM0 and _conv_count(unfused) == _conv_count(small)
    assert big.workspace_bytes < unfused.workspace_bytes
    forced = InferencePlan(model, 2, 184, 248, CPU, create_native=False, fuse_stem=True)
    assert forced._ops[0]['kind'] == nat.OP_STEM4


def test_stem4_query_tiles_the_stem3_map():
    q = nat.stem4_query(8, 720, 1280)
    assert (q['Ho'], q['Wo'], q['num_tiles']) == (180, 320, 8 * 12 * 40)
    assert q['smem_bytes'] <= 227 * 1024
    q = nat.stem4_query(1, 722, 1270)
    assert (q['Ho'], q['Wo'], q['num_tiles']) == (181, 318, 12 * 40)


def _input(fmt, n, h, w):
    if fmt == 'u8':
        return torch.stack([torch.from_numpy(synth.synth_image_u8(h, w, seed=11 + i)) for i in range(n)]).cuda()
    return synth.synth_input(n, h, w, seed=11).cuda()


@pytest.mark.gpu
@pytest.mark.parametrize('fmt', ['u8', 'f32'])
@pytest.mark.parametrize('dtype', ['bf16', 'fp16'])
@pytest.mark.parametrize('n,h,w', [(8, 720, 1280), (2, 186, 250), (1, 722, 1270)])
def test_fused_stem_is_bit_identical_to_the_two_launch_stem(n, h, w, dtype, fmt):
    """Same MMAs in the same order on the same 16-bit values: the stem3 map and the network outputs are bit-identical.
    186 x 250 and 722 x 1270 give stem3 maps that are not multiples of the 16 x 8 tile (border zeros on all four edges)."""
    model, _ = synth_model('WIDERFACE_S')
    model.cuda()
    dev = torch.device('cuda')
    fused = InferencePlan(model, n, h, w, dev, act_dtype=dtype, fuse_stem=True, reuse=False)     # the stem3 map outlives the forward
    pair = InferencePlan(model, n, h, w, dev, act_dtype=dtype, fuse_stem=False, reuse=False)
    assert fused._ops[0]['kind'] == nat.OP_STEM4 and pair._ops[0]['kind'] == nat.OP_STEM0
    x = _input(fmt, n, h, w)
    outs = []
    for plan in (fused, pair):
        with torch.no_grad():
            cls, reg = plan.forward(x, use_graph=False)
        torch.cuda.synchronize()
        outs.append((plan.tensor('stem3').clone(), cls.clone(), reg.clone()))
    (s_f, c_f, r_f), (s_p, c_p, r_p) = outs
    assert torch.equal(s_f.view(torch.int16), s_p.view(torch.int16)), 'stem3 differs: %d elements' % int((s_f != s_p).sum())
    assert torch.equal(c_f, c_p) and torch.equal(r_f, r_p)


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ['bf16', 'fp16'])
def test_fused_stem3_map_matches_the_cpu_chain_of_four_convs(dtype):
    from gpu_ops import ref_conv, DTYPES
    model, _ = synth_model('WIDERFACE_S')
    model.cuda()
    n, h, w = 1, 186, 250
    plan = InferencePlan(model, n, h, w, torch.device('cuda'), act_dtype=dtype, fuse_stem=True, reuse=False)
    x = synth.synth_input(n, h, w, seed=5)
    with torch.no_grad():
        plan.forward(x.cuda(), use_graph=False)
    torch.cuda.synchronize()
    got = plan.tensor('stem3').float().cpu()
    rnd, ulp = DTYPES[dtype][1], DTYPES[dtype][2]
    t = rnd(x).permute(0, 2, 3, 1)                     # rounding point R0
    layers = model._backbone.stem_layers()
    for li, (conv, norm, relu) in enumerate(layers):
        scale, shift = InferencePlan._fold(conv, norm)
        ref = ref_conv(t, conv.weight.detach().cpu(), scale, shift, conv.stride[0], bool(relu), dtype=dtype)
        t = rnd(ref)                                   # every intermediate is stored as 16 bits
    tol = ref.abs() * ulp + 2e-3 * float(ref.abs().max())   # 1-ulp flips of the in-kernel intermediates, as for fused tails
    assert bool(((got - ref).abs() <= tol).all()), float((got - ref).abs().max())
    assert rel_err(got, ref)[1] < 3e-3
