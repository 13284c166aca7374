# -*- coding: utf-8 -*-
"""CPU tests of frames below a plan's capacity: the geometry table a capacity plan computes for a frame (lfd_extent rows: H, W, Ho, Wo,
point_off, P, and the level sizes) equals, op by op, the fields of a plan built for that frame -- with the same STEM4 choice, the one
build decision that depends on the size (both paths give the same bits)."""
import pytest
import torch

from helpers import synth_model
from lfd import _native as nat
from lfd._engine import InferencePlan, check_frame
from oracle import lfd_oracle as orc

CAPACITY = (2, 400, 656)
# every h mod 4 and w mod 4, deepest levels of 1 x 1, the smallest frames, the capacity itself
SIZES = [(400, 656), (399, 655), (398, 654), (397, 653), (396, 652), (257, 129), (129, 257), (64, 64), (33, 31), (17, 9), (1, 1),
         (2, 3), (400, 1), (1, 656), (211, 600)]


def _uses_stem4(plan):
    return any(op['kind'] == nat.OP_STEM4 for op in plan._ops)


@pytest.mark.parametrize('name', list(orc.CONFIGS))
def test_geometry_table_matches_an_exact_plan(name):
    model, _ = synth_model(name)
    n, H, W = CAPACITY
    cap = InferencePlan(model, n, H, W, 'cpu', create_native=False)
    for h, w in SIZES:
        rows, level_sizes, P = cap.extent_table(h, w)
        exact = InferencePlan(model, n, h, w, 'cpu', create_native=False, fuse_stem=_uses_stem4(cap))
        assert len(rows) == len(exact._ops) == len(cap._ops)
        for i, (r, op, cop) in enumerate(zip(rows, exact._ops, cap._ops)):
            assert op['kind'] == cop['kind'] and op.get('out') == cop.get('out'), (name, i)
            want = [op['H'], op['W'], op['Ho'], op['Wo']]
            want += [op['point_off'], exact.P] if op['kind'] == nat.OP_HEAD_FINAL else [0, 0]
            assert r == want, (name, h, w, i, r, want)
            assert all(a <= b for a, b in zip(r[:4], [cop['H'], cop['W'], cop['Ho'], cop['Wo']]))
        assert level_sizes == exact.level_sizes and P == exact.P, (name, h, w)
    assert cap.extent_table(H, W)[1:] == (cap.level_sizes, cap.P)


def test_frame_validation():
    x = torch.zeros((2, 40, 64, 3), dtype=torch.uint8)
    with pytest.raises(ValueError):        # not on a CUDA device
        check_frame(x, 2, 40, 64)
    for shape, dtype in [((2, 41, 64, 3), torch.uint8), ((2, 40, 65, 3), torch.uint8), ((3, 40, 64, 3), torch.uint8),
                         ((2, 3, 41, 64), torch.float32), ((2, 40, 64, 4), torch.uint8), ((2, 0, 64, 3), torch.uint8)]:
        with pytest.raises(ValueError):
            check_frame(torch.zeros(shape, dtype=dtype), 2, 40, 64)
    with pytest.raises(TypeError):
        check_frame(torch.zeros((2, 40, 64, 3), dtype=torch.int32), 2, 40, 64)
