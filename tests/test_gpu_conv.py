# -*- coding: utf-8 -*-
"""GPU parity (Gate A): the wgmma implicit-GEMM convolution (and its SIMT cross-check) against an fp32 CPU
convolution of the same bf16 operands, through the C-ABI (lfd_run_op)."""
import pytest
import torch

from gpu_ops import bf16r, run_conv, ref_conv, assert_bf16_close, DTYPES
from lfd import _native as nat

pytestmark = pytest.mark.gpu

# (N, H, W, Cin, Cout, k, stride, relu, residual, gn)
CASES = [
    (1, 16, 8, 64, 64, 1, 1, True, False, 0),      # one full flat tile
    (2, 23, 31, 64, 64, 1, 1, True, False, 0),     # ragged flat tiles
    (2, 23, 31, 64, 128, 1, 1, True, False, 0),    # neck shape
    (2, 12, 20, 128, 128, 1, 1, False, False, 16), # head tower + GroupNorm statistics
    (1, 45, 80, 32, 32, 1, 1, True, False, 0),     # XS stem 1x1
    (1, 16, 8, 64, 64, 3, 1, True, False, 0),      # exactly one 16x8 tile
    (2, 23, 40, 64, 64, 3, 1, True, True, 0),      # 720p stage-2 shape, residual
    (1, 37, 29, 64, 64, 3, 1, False, False, 0),
    (2, 12, 20, 128, 128, 3, 1, True, True, 0),    # streamed weights
    (1, 45, 80, 64, 64, 3, 2, True, False, 0),     # stride 2 (odd output size 23x40)
    (2, 23, 40, 64, 128, 3, 2, True, False, 0),    # stage-3 entry
    (1, 46, 62, 32, 32, 3, 2, True, False, 0),     # XS stem 3x3/s2
    (2, 23, 40, 64, 128, 1, 2, False, False, 0),   # downsample path
    (1, 45, 80, 64, 64, 1, 2, False, False, 0),
]


def _make(case, seed=0, dtype='bf16'):
    N, H, W, Cin, Cout, k, s, relu, use_res, gn = case
    tdt, rnd = DTYPES[dtype][0], DTYPES[dtype][1]
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((N, H, W, Cin), generator=g).to(tdt).cuda()
    w = rnd(torch.randn((Cout, Cin, k, k), generator=g) * (2.0 / (Cin * k * k)) ** 0.5)
    scale = torch.rand((Cout,), generator=g) + 0.5
    shift = torch.randn((Cout,), generator=g) * 0.2
    if gn:
        scale, shift = torch.ones(Cout), torch.zeros(Cout)
    Ho, Wo = (H + 2 * (k // 2) - k) // s + 1, (W + 2 * (k // 2) - k) // s + 1
    res = torch.randn((N, Ho, Wo, Cout), generator=g).to(tdt).cuda() if use_res else None
    return x, w, scale, shift, res


@pytest.mark.parametrize('dtype', ['bf16', 'fp16'])
@pytest.mark.parametrize('impl', [nat.CONV_SIMT, nat.CONV_UMMA], ids=['simt', 'umma'])
@pytest.mark.parametrize('case', CASES, ids=lambda c: 'N%d_%dx%d_%d-%d_k%ds%d_r%d_res%d_gn%d' % c)
def test_conv_matches_fp32_reference(case, impl, dtype):
    N, H, W, Cin, Cout, k, s, relu, use_res, gn = case
    x, w, scale, shift, res = _make(case, dtype=dtype)
    out, stats, q = run_conv(x, w, scale, shift, s, relu, res=res, gn_groups=gn, impl=impl, dtype=dtype)
    ref = ref_conv(x, w, scale, shift, s, relu, res=res, dtype=dtype)
    assert_bf16_close(out, ref, 'conv %s %s (plan %s)' % (case, dtype, q), dtype=dtype)
    if gn:
        o = out.float().cpu().reshape(N, -1, gn, Cout // gn).double()
        s1, s2 = o.sum(dim=(1, 3)), (o * o).sum(dim=(1, 3))
        assert torch.allclose(stats[..., 0].cpu(), s1, rtol=1e-6, atol=1e-3)
        assert torch.allclose(stats[..., 1].cpu(), s2, rtol=1e-6, atol=1e-3)


def test_conv_large_grid_persistent_loop():
    """More tiles than SMs: exercises the persistent tile loop, both accumulator stages and ring wrap-around."""
    case = (3, 90, 160, 64, 64, 3, 1, True, True, 0)
    x, w, scale, shift, res = _make(case, seed=3)
    out, _, q = run_conv(x, w, scale, shift, 1, True, res=res)
    assert q['num_tiles'] > 2 * nat.lib().lfd_device_sm_count()
    assert_bf16_close(out, ref_conv(x, w, scale, shift, 1, True, res=res), 'large conv')


TAIL_CASES = [   # (N, H, W, Cin, Cmid, k, stride, Cout2, residual on the tail output, gn on the tail output)
    (2, 45, 80, 64, 64, 3, 2, 64, False, 0),     # stem2 + stem3 pattern
    (1, 37, 29, 64, 64, 3, 1, 128, True, 0),
    (2, 23, 31, 32, 32, 1, 1, 64, False, 0),
    (1, 33, 41, 64, 64, 1, 1, 128, False, 16),
    (2, 45, 80, 64, 128, 1, 1, 128, False, 16),  # neck conv (64 -> 128, BN + ReLU) + first tower conv (128 -> 128, GroupNorm statistics)
    (3, 12, 20, 128, 128, 1, 1, 128, False, 16),
    (1, 23, 40, 32, 128, 1, 1, 128, False, 16),
]


@pytest.mark.parametrize('dtype', ['bf16', 'fp16'])
@pytest.mark.parametrize('case', TAIL_CASES, ids=lambda c: 'N%d_%dx%d_%d-%d_k%ds%d_tail%d_res%d_gn%d' % c)
def test_conv_with_fused_1x1_tail(case, dtype):
    """conv + scale/shift + ReLU -> (bf16) -> 1x1 conv + scale/shift (+res) + ReLU in ONE kernel == the two layers run
    one after the other with the intermediate rounded to bf16."""
    N, H, W, Cin, Cmid, k, s, C2, use_res, gn = case
    tdt, rnd, ulp = DTYPES[dtype][0], DTYPES[dtype][1], DTYPES[dtype][2]
    x, w, scale, shift, _ = _make((N, H, W, Cin, Cmid, k, s, True, False, 0), seed=5, dtype=dtype)
    g = torch.Generator().manual_seed(9)
    w2 = rnd(torch.randn((C2, Cmid, 1, 1), generator=g) * (2.0 / Cmid) ** 0.5)
    sc2, sh2 = torch.rand((C2,), generator=g) + 0.5, torch.randn((C2,), generator=g) * 0.2
    if gn:
        sc2, sh2 = torch.ones(C2), torch.zeros(C2)
    Ho, Wo = (H + 2 * (k // 2) - k) // s + 1, (W + 2 * (k // 2) - k) // s + 1
    res = torch.randn((N, Ho, Wo, C2), generator=g).to(tdt).cuda() if use_res else None
    out, stats, q = run_conv(x, w, scale, shift, s, True, res=res, gn_groups=gn, tail=(w2, sc2, sh2, not gn), dtype=dtype)
    mid = rnd(ref_conv(x, w, scale, shift, s, True, dtype=dtype))
    ref = ref_conv(mid.to(tdt), w2, sc2, sh2, 1, not gn, res=res, dtype=dtype)
    # the intermediate itself may differ from the CPU one by 1 bf16 ulp on isolated elements (fp32 summation order), which
    # moves isolated outputs by more than one output ulp: allow 2e-3 of the output range on top of the 1-ulp bound
    o, r = out.float().cpu(), ref.float()
    tol = r.abs() * ulp + 2e-3 * float(r.abs().max()) * (ulp / 2.0 ** -7)
    assert bool(((o - r).abs() <= tol).all()), 'fused tail %s: max err %g (ref max %g) plan %s' % (case, float((o - r).abs().max()), float(r.abs().max()), q)
    assert float(torch.sqrt(((o - r) ** 2).mean()) / torch.sqrt((r ** 2).mean())) < 3e-3 * (ulp / 2.0 ** -7)
    if gn:
        og = out.float().cpu().reshape(N, -1, gn, C2 // gn).double()
        assert torch.allclose(stats[..., 0].cpu(), og.sum(dim=(1, 3)), rtol=1e-6, atol=1e-3)
