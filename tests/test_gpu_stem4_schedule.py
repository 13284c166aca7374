# -*- coding: utf-8 -*-
"""The fused four-conv stem (LFD_OP_STEM4) under forced grids: every CTA walks a contiguous run of tiles and a tile whose left
neighbour came before it in the run inherits that neighbour's last stem1 column.  Runs of 1, 2, 5, 7 and 131 CTAs start and end
mid-row, at row starts and across images; the stem3 map and the network outputs must stay bit-identical to the two-kernel path.
Also both patch loaders: aligned words (u8, W % 4 == 0, 4-byte aligned base) and per pixel (fp32, W % 4 != 0, a misaligned base)."""
import functools

import pytest
import torch

import synth
from helpers import synth_model
from lfd import _native as nat
from lfd._engine import InferencePlan

GRIDS = (1, 2, 5, 7, 131)
BENCH = (8, 720, 1280)
RAGGED_W4 = (2, 186, 252)     # W % 4 == 0 (word loader), stem3 map 47 x 63: partial tiles on the bottom and right edges
RAGGED = (2, 186, 250)        # W % 4 == 2 (per-pixel loader)


@functools.lru_cache(maxsize=None)
def _model():
    model, _ = synth_model('WIDERFACE_S')
    return model.cuda()


def _input(fmt, n, h, w, misaligned=False):
    if fmt == 'f32':
        return synth.synth_input(n, h, w, seed=23).cuda()
    img = torch.stack([torch.from_numpy(synth.synth_image_u8(h, w, seed=31 + i)) for i in range(n)]).cuda()
    if not misaligned:
        return img
    raw = torch.empty(img.numel() + 1, dtype=torch.uint8, device='cuda')
    x = raw[1:].view(n, h, w, 3)                     # base address 1 (mod 4)
    x.copy_(img)
    assert x.is_contiguous() and x.data_ptr() % 4 == 1
    return x


def _run(plan, x, stem_ctas=None):
    """stem3 map, cls, reg of one eager forward; stem_ctas bounds the fused stem's persistent CTAs."""
    if stem_ctas is not None:
        plan._op_array[0].max_ctas = stem_ctas
        old, plan.handle = plan.handle, plan._create_handle()
        nat.lib().lfd_plan_destroy(old)
    stem3 = plan.tensor('stem3')
    stem3.view(torch.int16).fill_(-1)                # NaN pattern: a tile that is not stored cannot pass
    with torch.no_grad():
        cls, reg = plan.forward(x, use_graph=False)
    torch.cuda.synchronize()
    return stem3.clone(), cls.clone(), reg.clone()


def _check(shape, dtype, fmt, misaligned=False, grids=GRIDS):
    """Both plans are built with reuse=False: the stem3 map must outlive the forward."""
    n, h, w = shape
    model = _model()
    dev = torch.device('cuda')
    fused = InferencePlan(model, n, h, w, dev, act_dtype=dtype, fuse_stem=True, reuse=False)
    pair = InferencePlan(model, n, h, w, dev, act_dtype=dtype, fuse_stem=False, reuse=False)
    assert fused._ops[0]['kind'] == nat.OP_STEM4 and pair._ops[0]['kind'] == nat.OP_STEM0
    x = _input(fmt, n, h, w, misaligned)
    s_p, c_p, r_p = _run(pair, x)
    tiles = nat.stem4_query(n, h, w)['num_tiles']
    for m in grids:
        s_f, c_f, r_f = _run(fused, x, m)
        what = '%s %s %s%s, %d CTAs over %d tiles' % ('x'.join(map(str, shape)), dtype, fmt, ' (misaligned)' if misaligned else '',
                                                      min(m, tiles), tiles)
        bad = s_f.view(torch.int16) != s_p.view(torch.int16)
        if bad.any():
            idx = bad.nonzero()[0].tolist()
            raise AssertionError('%s: stem3 differs in %d elements, first at (n, y, x, c) = %s' % (what, int(bad.sum()), idx))
        assert torch.equal(c_f, c_p) and torch.equal(r_f, r_p), what


@pytest.mark.gpu
@pytest.mark.parametrize('fmt', ['u8', 'f32'])
@pytest.mark.parametrize('dtype', ['bf16', 'fp16'])
@pytest.mark.parametrize('shape', [BENCH, RAGGED_W4, RAGGED], ids=['720p-b8', 'ragged-w4', 'ragged'])
def test_fused_stem_runs_are_bit_identical_to_the_two_launch_stem(shape, dtype, fmt):
    _check(shape, dtype, fmt)


@pytest.mark.gpu
@pytest.mark.parametrize('shape', [BENCH, RAGGED_W4], ids=['720p-b8', 'ragged-w4'])
def test_fused_stem_on_misaligned_u8_input_is_bit_identical(shape):
    """A u8 image at an address that is not a multiple of 4 takes the per-pixel loader."""
    _check(shape, 'bf16', 'u8', misaligned=True, grids=(2, 7, 131))
