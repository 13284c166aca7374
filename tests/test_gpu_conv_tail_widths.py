# -*- coding: utf-8 -*-
"""Fused 1x1 tail at every stored width: the tail GEMM is issued as Cmid / 16 MMAs of N = Cout2, one code path per width, so
Cout2 = 16 / 32 (not used by the shipped networks) get their own cases, plus a layer with two channel chunks per tile and one
with several tiles per CTA."""
import pytest

from test_gpu_conv import test_conv_with_fused_1x1_tail as _check_fused_tail

CASES = [   # (N, H, W, Cin, Cmid, k, stride, Cout2, residual on the tail output, gn on the tail output)
    (2, 45, 80, 64, 64, 3, 2, 16, False, 0),
    (1, 37, 29, 64, 64, 3, 1, 32, True, 0),
    (2, 23, 31, 32, 32, 1, 1, 16, False, 0),
    (1, 30, 50, 128, 64, 3, 1, 32, False, 0),     # two 64-channel chunks per tile
    (3, 180, 320, 64, 64, 3, 2, 64, True, 0),     # 720 tiles: several per CTA
]


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ['bf16', 'fp16'])
@pytest.mark.parametrize('case', CASES, ids=lambda c: 'N%d_%dx%d_%d-%d_k%ds%d_tail%d_res%d_gn%d' % c)
def test_fused_tail_widths(case, dtype):
    _check_fused_tail(case, dtype)
