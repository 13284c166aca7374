# -*- coding: utf-8 -*-
"""Weight and data gradients at every shape class of the wgmma kernels, with many tiles per CTA: one CTA per (tap group, channel
chunk) accumulating every tile in registers (persistent split-K over pixels) while its ring wraps many times, against float64
CPU gradients of the same 16-bit operands."""
import pytest
import torch

from gpu_ops import assert_faithful, bf16r, conv_out, ref_conv64
from gpu_train_ops import Workspace, desc_table, make_top, run_top
from lfd import _native as nat

DEV = 'cuda'
MODES = [(1, 1), (3, 1), (3, 2), (1, 2)]          # (ksize, stride)
# input size per mode: 30 tiles of 16 x 8 (or 128 flat) output pixels over N = 2 images, ragged in both directions
SIZES = {(1, 1): (39, 37), (3, 1): (39, 37), (3, 2): (79, 73), (1, 2): (79, 73)}


def wg_plan(N, H, W, Cin, Cout, k, s):
    """Mirror of wg_configure (wgrad_umma.cu): tiles, ring depth, CTAs per tile slice and tap groups."""
    Ho, Wo = conv_out(H, k, s), conv_out(W, k, s)
    flat = (k, s) == (1, 1)
    tiles = N * ((Ho * Wo + 127) // 128 if flat else ((Wo + 7) // 8) * ((Ho + 15) // 16))
    n_px, px_slots = {(1, 1): (128, 128), (3, 1): (180, 180), (3, 2): (561, 594), (1, 2): (128, 128)}[(k, s)]
    a_stage = (8 * (px_slots | 1) * 16 + 127) & ~127
    b_stage = ((Cout // 8) * 129 * 16 + 127) & ~127
    table = 0 if flat else (n_px * 10 + 127) & ~127
    ring_off = (512 + table + 1023) & ~1023
    stages = min(4, (226 * 1024 - ring_off) // (a_stage + b_stage))
    taps = k * k
    per_wg = 1 if taps == 1 else min(256 // Cout, 9)
    n_tapg = (taps + 2 * per_wg - 1) // (2 * per_wg)
    return dict(num_tiles=tiles, stages=stages, per=((Cin + 63) // 64) * n_tapg, n_tapg=n_tapg)


CASES = [(k, s, cout, cin) for (k, s) in MODES for cout in (16, 32, 64, 128) for cin in (32, 64, 128)]


def test_wgrad_shapes_give_many_tiles_per_ring_stage():
    for k, s, cout, cin in CASES:
        H, W = SIZES[(k, s)]
        p = wg_plan(2, H, W, cin, cout, k, s)
        assert 5 * p['stages'] <= p['num_tiles'] <= 50 * p['stages'], (k, s, cout, cin, p)
        if k == 3:
            assert p['n_tapg'] == {16: 1, 32: 1, 64: 2, 128: 3}[cout]      # Cout 64: 5 + 4 taps, 128: 3 x 3


def _wgrad(x, dz, k, s, max_ctas, Cin, Cout):
    N, H, W, _ = x.shape
    Ho, Wo = dz.shape[1], dz.shape[2]
    ws = Workspace(DEV)
    ws.add('x', x.to(torch.bfloat16))
    ws.add('dz', dz.to(torch.bfloat16))
    ws.add('ds', shape=(k * k, Cin, Cout), dtype=torch.float32)
    ws.finalize()
    run_top(make_top(nat.TOP_WGRAD, N=N, H=H, W=W, Cin=Cin, Ho=Ho, Wo=Wo, Cout=Cout, ksize=k, stride=s, impl=nat.WGRAD_UMMA, max_ctas=max_ctas,
                     off={0: ws.off('x'), 1: ws.off('dz'), 5: ws.off('ds')}), ws)
    return ws.get('ds').cpu().permute(2, 1, 0).reshape(Cout, Cin, k, k)


def _assert_wgrad(got, x, dz, k, s, what):
    """|got - ref| <= 1e-5 * S per element, S = the gradient of |x| and |dz|: a tile lost or counted twice moves an element by
    about S / num_tiles."""
    Cout, Cin = got.shape[0], got.shape[1]
    xd, dzd = x.double().permute(0, 3, 1, 2), dz.double().permute(0, 3, 1, 2)
    ref = torch.nn.grad.conv2d_weight(xd, (Cout, Cin, k, k), dzd, stride=s, padding=k // 2)
    S = torch.nn.grad.conv2d_weight(xd.abs(), (Cout, Cin, k, k), dzd.abs(), stride=s, padding=k // 2)
    err = (got.double() - ref).abs()
    bad = err > 1e-5 * S
    if bool(bad.any()):
        i = tuple(torch.nonzero(bad)[0].tolist())
        raise AssertionError('%s: %d / %d elements off; first at %s: got %g want %g (S %g)' % (what, int(bad.sum()), got.numel(), i,
                                                                                             float(got[i]), float(ref[i]), float(S[i])))


@pytest.mark.gpu
@pytest.mark.parametrize('max_ctas', [0, 1])
@pytest.mark.parametrize('k,s,cout,cin', CASES)
def test_wgrad_every_shape_matches_fp64(k, s, cout, cin, max_ctas):
    H, W = SIZES[(k, s)]
    N = 2
    Ho, Wo = conv_out(H, k, s), conv_out(W, k, s)
    g = torch.Generator().manual_seed(k * 1000 + s * 100 + cout + cin)
    x = bf16r(torch.randn((N, H, W, cin), generator=g))
    dz = bf16r(torch.randn((N, Ho, Wo, cout), generator=g))
    got = _wgrad(x, dz, k, s, max_ctas, cin, cout)
    p = wg_plan(N, H, W, cin, cout, k, s)
    _assert_wgrad(got, x, dz, k, s, 'wgrad k%d s%d %d->%d max_ctas=%d (%s)' % (k, s, cin, cout, max_ctas, p))


@pytest.mark.gpu
@pytest.mark.parametrize('fmt', ['f32', 'u8'])
def test_wgrad_stem_with_many_tiles_per_cta(fmt):
    """TOP_WGRAD_STEM, im2col + wgmma: a 1x1 wgrad over the 32-row im2col tensor with > 4 flat tiles per CTA."""
    N, H, W, Cout = 2, 300, 580, 64
    Ho, Wo = conv_out(H, 3, 2), conv_out(W, 3, 2)
    assert N * ((Ho * Wo + 127) // 128) > 4 * nat.lib().lfd_device_sm_count()
    g = torch.Generator().manual_seed(17)
    if fmt == 'u8':
        img = torch.randint(0, 256, (N, H, W, 3), generator=g, dtype=torch.uint8)
        x = bf16r((img.float() - 127.5) * (1.0 / 127.5))
    else:
        img = torch.randn((N, 3, H, W), generator=g)
        x = bf16r(img.permute(0, 2, 3, 1))
    dz = bf16r(torch.randn((N, Ho, Wo, Cout), generator=g))
    ws = Workspace(DEV)
    ws.add('dz', dz.to(torch.bfloat16))
    ws.add('ds', shape=(32, Cout), dtype=torch.float32)
    ws.add('x27', shape=(N, Ho, Wo, 32), dtype=torch.bfloat16)
    ws.finalize()
    run_top(make_top(nat.TOP_WGRAD_STEM, N=N, H=H, W=W, Cin=3, Ho=Ho, Wo=Wo, Cout=Cout, ksize=3, stride=2, impl=nat.WGRAD_UMMA,
                     off={0: ws.off('x27'), 1: ws.off('dz'), 5: ws.off('ds')}), ws,
            input=img.to(DEV).contiguous(), fmt=nat.INPUT_U8_NHWC if fmt == 'u8' else nat.INPUT_F32_NCHW)
    stage = ws.get('ds').cpu()
    assert float(stage[27:].abs().max()) == 0.0
    got = stage[:27].reshape(9, 3, Cout).permute(2, 1, 0).reshape(Cout, 3, 3, 3)
    _assert_wgrad(got, x, dz, 3, 2, 'stem wgrad %s' % fmt)


@pytest.mark.gpu
@pytest.mark.parametrize('case', [(2, 45, 61, 64, 64, 3, 1), (2, 45, 61, 128, 64, 3, 2), (2, 40, 36, 64, 128, 1, 1), (2, 45, 62, 32, 64, 1, 2)],
                         ids=lambda c: 'N%d_%dx%d_%d-%d_k%ds%d' % c)
def test_dgrad_with_many_tiles_per_cta_matches_fp64(case):
    """dx = prev + conv_transpose(dz, W) as the forward kernel runs it in training (TOP_CONV on PACK_CONV_DGRAD weights, the result
    accumulated in place through res = out; stride 2 = a stride-1 conv on the zero-inserted dz), with 3 persistent CTAs."""
    N, H, W, Cin, Cout, k, s = case
    g = torch.Generator().manual_seed(31)
    Ho, Wo = conv_out(H, k, s), conv_out(W, k, s)
    w = bf16r(torch.randn((Cout, Cin, k, k), generator=g) * 0.1)
    dz = bf16r(torch.randn((N, Ho, Wo, Cout), generator=g))
    prev = bf16r(torch.randn((N, H, W, Cin), generator=g))
    up = torch.zeros(N, H, W, Cout)
    up[:, ::s, ::s, :] = dz
    q = nat.conv_query(N, H, W, Cout, H, W, Cin, k, 1)
    assert q['num_tiles'] // 3 >= 4
    wd = w.to(DEV)
    ws = Workspace(DEV)
    ws.add('dzu', up.to(torch.bfloat16))
    ws.add('dx', prev.to(torch.bfloat16))
    ws.add('wp', shape=(w.numel(),), dtype=torch.bfloat16)
    ws.finalize()
    d = nat.PackDesc(kind=nat.PACK_CONV_DGRAD, Cout=Cout, Cin=Cin, k=k, cc=q['cc'], n=w.numel(), src=wd.data_ptr(), dst=ws.buf.data_ptr() + ws.off('wp'))
    table = desc_table([d], DEV)
    run_top(make_top(nat.TOP_PACK, n_desc=1, max_n=w.numel(), ptr={0: table.data_ptr()}), ws)
    run_top(make_top(nat.TOP_CONV, N=N, H=H, W=W, Cin=Cout, Ho=H, Wo=W, Cout=Cin, ksize=k, stride=1, cc=q['cc'], max_ctas=3,
                     off={0: ws.off('dzu'), 1: ws.off('dx'), 2: ws.off('dx'), 4: ws.off('wp')}), ws)
    wt = w.permute(1, 0, 2, 3).flip(2, 3).contiguous()          # the transposed conv's OIHW weights
    ref, S, K = ref_conv64(up, wt, torch.ones(Cin), torch.zeros(Cin), 1, False, res=prev)
    want = torch.nn.grad.conv2d_input((N, Cin, H, W), w.double(), dz.double().permute(0, 3, 1, 2), stride=s, padding=k // 2)
    assert float((ref - (want.permute(0, 2, 3, 1) + prev.double())).abs().max()) < 1e-9      # the reference is the data gradient
    assert_faithful(ws.get('dx'), ref, S, K, 'bf16', 'dgrad %s' % (case,))
