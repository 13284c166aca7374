# -*- coding: utf-8 -*-
"""Helpers that drive single native ops through the C-ABI (lfd_run_op) for the GPU parity tests."""
import ctypes as C

import torch
import torch.nn.functional as F

from lfd import _native as nat
from lfd._engine import pack_conv_weight, pack_stem_weight, fold_scale


def bf16r(t):
    return t.to(torch.bfloat16).float()


def fp16r(t):
    return t.to(torch.float16).float()


# act dtype name -> (torch storage type, rounding function, relative size of one ulp step, native code)
DTYPES = {'bf16': (torch.bfloat16, bf16r, 2.0 ** -7, nat.DTYPE_BF16), 'fp16': (torch.float16, fp16r, 2.0 ** -10, nat.DTYPE_FP16)}


def conv_out(size, k, s):
    return (size + 2 * (k // 2) - k) // s + 1


def run_conv(x_nhwc, weight, scale, shift, stride, relu, res=None, gn_groups=0, impl=nat.CONV_UMMA, tail=None, dtype='bf16', max_ctas=0,
             ds=None):
    """x_nhwc: cuda bf16 / fp16 [N,H,W,Cin]; weight fp32 [Cout,Cin,k,k] (already representable in the 16-bit type).
    max_ctas: lfd_op.max_ctas (0 = one persistent CTA per SM).  ds = (w3 [Cout,Cin,1,1], scale3, shift3): the fused 1x1/s2
    shortcut of a 3x3/s2 conv (lfd_op.ds_cout).
    -> (out [N,Ho,Wo,Cf], stats double [N,groups,2] or None, conv_query dict), plus the shortcut output [N,Ho,Wo,Cout] with ds"""
    tdt, _, _, code = DTYPES[dtype]
    assert x_nhwc.dtype == tdt
    dev = x_nhwc.device
    N, H, W, Cin = x_nhwc.shape
    Cout, _, k, _ = weight.shape
    Ho, Wo = conv_out(H, k, stride), conv_out(W, k, stride)
    Cf = tail[0].shape[0] if tail is not None else Cout
    q = nat.conv_query(N, H, W, Cin, Ho, Wo, Cout, k, stride, Cf if tail is not None else 0, Cout if ds is not None else 0)
    wp = pack_conv_weight(fold_scale(weight, scale), q['cc'], tdt).to(dev)   # BatchNorm scale folded before the bf16 rounding
    sh = shift.float().to(dev).contiguous()
    in_b = x_nhwc.numel() * 2
    out_b = N * Ho * Wo * Cf * 2
    al = lambda v: (v + 255) & ~255
    off_in, off_out = 4096, 4096 + al(in_b)
    off_res = off_out + al(out_b)
    off_ds = off_res + al(out_b)
    total = off_ds + al(out_b) + 256
    ws = torch.zeros(total, dtype=torch.uint8, device=dev)
    ws[off_in:off_in + in_b] = x_nhwc.contiguous().view(torch.uint8).reshape(-1)
    if res is not None:
        ws[off_res:off_res + out_b] = res.contiguous().view(torch.uint8).reshape(-1)
    op = nat.Op()
    op.kind = nat.OP_CONV
    op.dtype = code
    op.N, op.H, op.W, op.Cin, op.Ho, op.Wo, op.Cout = N, H, W, Cin, Ho, Wo, Cout
    op.ksize, op.stride, op.relu, op.gn_groups, op.cc = k, stride, int(relu), gn_groups, q['cc']
    op.in_off, op.out_off, op.res_off = off_in, off_out, (off_res if res is not None else -1)
    op.stats_off = 0 if gn_groups else -1
    op.max_ctas = max_ctas
    op.weight, op.shift = wp.data_ptr(), sh.data_ptr()
    if tail is not None:
        w2, sc2, sh2, relu2 = tail
        w2p = pack_conv_weight(fold_scale(w2, sc2), Cout, tdt).to(dev)
        sh2d = sh2.float().to(dev).contiguous()
        op.tail_cout, op.tail_relu = Cf, int(relu2)
        op.tail_weight, op.tail_shift = w2p.data_ptr(), sh2d.data_ptr()
    if ds is not None:
        w3, sc3, sh3 = ds
        w3p = pack_conv_weight(fold_scale(w3, sc3), Cin, tdt).to(dev)      # [Cin/8][Cout][8]
        sh3d = sh3.float().to(dev).contiguous()
        op.ds_cout, op.ds_out_off = Cout, off_ds
        op.ds_weight, op.ds_shift = w3p.data_ptr(), sh3d.data_ptr()
    with torch.cuda.device(dev):
        nat.check(nat.lib().lfd_run_op(C.byref(op), None, 0, nat.ptr(ws), None, None, 0, 0, impl, nat.stream_ptr()))
        torch.cuda.synchronize()
    out = ws[off_out:off_out + out_b].view(tdt).view(N, Ho, Wo, Cf).clone()
    stats = ws[0:N * gn_groups * 16].view(torch.float64).view(N, gn_groups, 2).clone() if gn_groups else None
    if ds is not None:
        return out, stats, q, ws[off_ds:off_ds + out_b].view(tdt).view(N, Ho, Wo, Cout).clone()
    return out, stats, q


def ref_conv(x_nhwc, weight, scale, shift, stride, relu, res=None, dtype='bf16'):
    """fp32 CPU reference of the fused layer on the operands the kernel sees: weights = round16(weight * scale) (BatchNorm
    fold, rounding point Rw), shift rounded to the 16-bit type; result NOT yet rounded."""
    rnd = DTYPES[dtype][1]
    x = x_nhwc.float().cpu().permute(0, 3, 1, 2)
    k = weight.shape[-1]
    y = F.conv2d(x, rnd(fold_scale(weight, scale)), None, stride=stride, padding=k // 2)
    y = y + rnd(shift.float().cpu())[None, :, None, None]
    if res is not None:
        y = y + res.float().cpu().permute(0, 3, 1, 2)
    if relu:
        y = F.relu(y)
    return y.permute(0, 2, 3, 1).contiguous()


def assert_bf16_close(out_bf16, ref_fp32, what='', dtype='bf16'):
    """out must equal the fp32 reference rounded to the 16-bit type up to 1 ulp (accumulation-order noise next to a rounding
    boundary) -- Gate A of the parity protocol."""
    ulp = DTYPES[dtype][2]
    o = out_bf16.float().cpu()
    r = ref_fp32.float()
    tol = r.abs() * ulp + 2e-3 * float(r.abs().max()) * ulp + 1e-6
    bad = (o - r).abs() > tol
    if bool(bad.any()):
        idx = torch.nonzero(bad)
        i = tuple(idx[0].tolist())
        raise AssertionError('%s: %d / %d elements off; first at %s: got %g want %g; max abs err %g (ref max %g)'
                             % (what, int(bad.sum()), o.numel(), i, float(o[i]), float(r[i]), float((o - r).abs().max()), float(r.abs().max())))


def run_stem0(img, fmt, w, shift, relu, tail=None, max_ctas=0, dtype='bf16'):
    """LFD_OP_STEM0 through lfd_run_op: img = cuda uint8 [N,H,W,3] (fmt 'u8') or float32 [N,3,H,W] (fmt 'f32'); w fp32
    [Cout,3,3,3] with the BatchNorm scale already folded in (rounded to the 16-bit type by the packing); tail as in run_conv.
    -> (out [N,Ho,Wo,Cf], number of 16 x 8 output tiles)"""
    tdt, _, _, code = DTYPES[dtype]
    dev = img.device
    if fmt == 'u8':
        N, H, W, _ = img.shape
    else:
        N, _, H, W = img.shape
    Cout = w.shape[0]
    Ho, Wo = conv_out(H, 3, 2), conv_out(W, 3, 2)
    Cf = tail[0].shape[0] if tail is not None else Cout
    wp = pack_stem_weight(w, tdt).to(dev)
    sh = shift.float().to(dev).contiguous()
    out_b = N * Ho * Wo * Cf * 2
    ws = torch.zeros(4096 + ((out_b + 255) & ~255) + 256, dtype=torch.uint8, device=dev)
    op = nat.Op()
    op.kind = nat.OP_STEM0
    op.dtype = code
    op.N, op.H, op.W, op.Cin, op.Ho, op.Wo, op.Cout = N, H, W, 3, Ho, Wo, Cout
    op.ksize, op.stride, op.relu = 3, 2, int(relu)
    op.in_off, op.out_off, op.res_off, op.stats_off = -1, 4096, -1, -1
    op.max_ctas = max_ctas
    op.weight, op.shift = wp.data_ptr(), sh.data_ptr()
    if tail is not None:
        w2, sc2, sh2, relu2 = tail
        w2p = pack_conv_weight(fold_scale(w2, sc2), Cout, tdt).to(dev)
        sh2d = sh2.float().to(dev).contiguous()
        op.tail_cout, op.tail_relu = Cf, int(relu2)
        op.tail_weight, op.tail_shift = w2p.data_ptr(), sh2d.data_ptr()
    x = img.contiguous()
    with torch.cuda.device(dev):
        nat.check(nat.lib().lfd_run_op(C.byref(op), nat.ptr(x), nat.INPUT_U8_NHWC if fmt == 'u8' else nat.INPUT_F32_NCHW, nat.ptr(ws), None,
                                       None, 0, 0, nat.CONV_UMMA, nat.stream_ptr()))
        torch.cuda.synchronize()
    out = ws[4096:4096 + out_b].view(tdt).view(N, Ho, Wo, Cf).clone()
    return out, N * ((Ho + 15) // 16) * ((Wo + 7) // 8)


def stem_input(img, fmt, dtype='bf16'):
    """The stem's operand as the kernel forms it (rounding point R0): NHWC, normalised in fp32 for u8 input, then rounded to the
    16-bit type."""
    rnd = DTYPES[dtype][1]
    if fmt == 'u8':
        return rnd((img.float() - 127.5) * (1.0 / 127.5))
    return rnd(img.float().permute(0, 2, 3, 1))


def ref_conv64(x_nhwc, weight, scale, shift, stride, relu, res=None, dtype='bf16', device='cpu'):
    """float64 evaluation of the fused layer on exactly the operands the kernel sees: round16(weight * scale), round16(shift),
    the 16-bit input and residual, on `device` (the CPU, or the GPU for whole-network sizes).  -> (y [N,Ho,Wo,Cout] float64, not
    rounded; S = the same sum over |terms| per output; K = the number of terms the kernel adds in fp32 per output)."""
    rnd = DTYPES[dtype][1]
    x = x_nhwc.to(device).double().permute(0, 3, 1, 2)
    w = rnd(fold_scale(weight, scale)).double().to(device)
    b = rnd(shift.float().cpu()).double().to(device)[None, :, None, None]
    k = weight.shape[-1]
    y = F.conv2d(x, w, None, stride=stride, padding=k // 2) + b
    S = F.conv2d(x.abs(), w.abs(), None, stride=stride, padding=k // 2) + b.abs()
    K = weight.shape[1] * k * k + 1
    if res is not None:
        r = res.to(device).double().permute(0, 3, 1, 2)
        y, S, K = y + r, S + r.abs(), K + 1
    if relu:
        y = F.relu(y)
    return y.permute(0, 2, 3, 1).contiguous(), S.permute(0, 2, 3, 1).contiguous(), K


def ulp16(x, dtype='bf16'):
    """Spacing of the 16-bit type at |x| (x float64; 0 at x = 0)."""
    p = 7 if dtype == 'bf16' else 10
    _, e = torch.frexp(x)
    u = torch.ldexp(torch.ones_like(x), e - 1 - p)
    u = u.clamp(min=2.0 ** -133 if dtype == 'bf16' else 2.0 ** -24)
    return torch.where(x == 0, torch.zeros_like(x), u)


def assert_faithful(out, ref64, S, K, dtype='bf16', what=''):
    """Per element |out - ref64| <= ulp16(ref64) + K * 2^-24 * S: out is a faithful 16-bit rounding of the exact value, widened
    only by the worst-case error of an fp32 accumulation of K terms whose magnitudes sum to S."""
    o = out.cpu().double()
    err = (o - ref64).abs()
    tol = ulp16(ref64, dtype) + K * 2.0 ** -24 * S
    bad = ~(err <= tol)
    if bool(bad.any()):
        idx = torch.nonzero(bad)
        i = tuple(idx[0].tolist())
        raise AssertionError('%s: %d / %d elements off; first at %s: got %r want %r (tol %g); max abs err %g (ref max %g)'
                             % (what, int(bad.sum()), o.numel(), i, float(o[i]), float(ref64[i]), float(tol[i]), float(err.max()),
                                float(ref64.abs().max())))


def assert_tail_close(out, ref, dtype='bf16', what=''):
    """Bound for the output of a fused tail: its 16-bit intermediate may differ from the CPU one by 1 ulp on isolated elements
    (fp32 summation order), which moves isolated outputs by more than one output ulp, so 2e-3 of the output range is allowed on
    top of the 1-ulp bound, and the RMS error must stay small.  Compared on ref's device.  -> max err / tol."""
    ulp = DTYPES[dtype][2]
    o, r = out.to(ref.device).double(), ref.double()
    tol = r.abs() * ulp + 2e-3 * float(r.abs().max()) * (ulp / 2.0 ** -7)
    err = (o - r).abs()
    assert bool((err <= tol).all()), '%s: %d elements off, max err %g (ref max %g)' % (what, int((err > tol).sum()), float(err.max()), float(r.abs().max()))
    assert float(torch.sqrt((err ** 2).mean()) / torch.sqrt((r ** 2).mean()).clamp(min=1e-30)) < 3e-3 * (ulp / 2.0 ** -7), what
    return float((err / tol.clamp(min=1e-300)).max())


def assert_gn_stats(stats, out, groups, what=''):
    """Fused GroupNorm statistics against float64 sums of the stored tensor: the kernel adds fp32 partial sums of at most a few
    dozen values before its fp64 atomics, so 1e-5 of the sum of |terms| bounds the difference."""
    N, C = out.shape[0], out.shape[-1]
    o = out.cpu().double().reshape(N, -1, groups, C // groups)
    s1, s2 = o.sum(dim=(1, 3)), (o * o).sum(dim=(1, 3))
    a1 = o.abs().sum(dim=(1, 3))
    st = stats.cpu()
    assert bool(((st[..., 0] - s1).abs() <= 1e-5 * a1 + 1e-30).all()), '%s: sum off by %g' % (what, float((st[..., 0] - s1).abs().max()))
    assert bool(((st[..., 1] - s2).abs() <= 1e-5 * s2 + 1e-30).all()), '%s: sum of squares off by %g' % (what, float((st[..., 1] - s2).abs().max()))
