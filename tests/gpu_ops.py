# -*- coding: utf-8 -*-
"""Helpers that drive single native ops through the C-ABI (lfd_run_op) for the GPU parity tests."""
import ctypes as C
import functools

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


GUARD = 4096          # bytes of poison before and after every tensor of the single-op runners


class Workspace(object):
    """Byte workspace with named, 256-byte aligned regions (what lfd_op / lfd_top offsets index).  By default zero-filled with the regions
    back to back.  guard > 0 keeps that many bytes before and after every region; poison fills the workspace with 0xff bytes (NaN in bf16,
    fp16, fp32 and fp64), so a kernel that reads outside its tensors carries a NaN and one that writes outside them is caught by
    assert_guards().  A region added with zero=True starts at zero (the fused GroupNorm statistics accumulate with atomics)."""

    def __init__(self, device, guard=0, poison=False):
        self.device, self.guard, self.poison = device, guard, poison
        self.top = max(256, guard)
        self.items = {}          # name -> (offset, bytes, dtype, shape)
        self.init = {}
        self.zero = []
        self.buf = None

    def add(self, name, tensor=None, shape=None, dtype=None, zero=False):
        if tensor is not None:
            tensor = tensor.contiguous()
            shape, dtype = tuple(tensor.shape), tensor.dtype
            self.init[name] = tensor
        nbytes = int(torch.empty(0, dtype=dtype).element_size())
        for s in shape:
            nbytes *= s
        off = self.top
        self.items[name] = (off, nbytes, dtype, tuple(shape))
        self.top = ((off + nbytes + 255) & ~255) + self.guard
        if zero:
            self.zero.append(name)
        return off

    def finalize(self):
        self.buf = torch.full((self.top + 256,), 0xff if self.poison else 0, dtype=torch.uint8, device=self.device)
        for name in self.zero:
            off, nbytes, _, _ = self.items[name]
            self.buf[off:off + nbytes] = 0
        for name, t in self.init.items():
            off, nbytes, _, _ = self.items[name]
            self.buf[off:off + nbytes] = t.to(self.device).view(torch.uint8).reshape(-1)
        return self

    def off(self, name):
        return self.items[name][0] if name is not None else -1

    def get(self, name):
        off, nbytes, dtype, shape = self.items[name]
        return self.buf[off:off + nbytes].view(dtype).view(shape).clone()

    def assert_guards(self, what=''):
        """Every byte outside the regions still holds the poison (one reduction on the device; the workspace stays there)."""
        assert self.poison
        outside = torch.ones_like(self.buf, dtype=torch.bool)
        for off, nbytes, _, _ in self.items.values():
            outside[off:off + nbytes] = False
        written = (self.buf != 0xff) & outside
        n = int(written.sum())
        if n:
            first = int(written.nonzero()[0])
            end, name = max([(o + nb, k) for k, (o, nb, _, _) in self.items.items() if o + nb <= first], default=(0, 'the start'))
            raise AssertionError('%s: %d bytes outside the tensors were written, the first at byte %d (%d bytes past the end of %s)'
                                 % (what, n, first, first - end, name))


def make_op(kind, dtype='bf16', transform=None, **fields):
    """An lfd_op (nat.Op) of the 16-bit storage type `dtype`, every tensor offset -1 (none) unless given, the input transform set by
    nat.set_input_transform."""
    op = nat.Op()
    op.kind, op.dtype = kind, DTYPES[dtype][3]
    op.in_off = op.out_off = op.res_off = op.stats_off = op.ds_out_off = -1
    for k, v in fields.items():
        setattr(op, k, v)
    nat.set_input_transform(op, transform)
    return op


def _set_tail(op, tail, cin, tdt, dev):
    """The fused 1x1 tail (w [Cf, cin, 1, 1], scale, shift, relu) of op -> the device operands, to be kept until the launch"""
    w2, sc2, sh2, relu2 = tail
    keep = pack_conv_weight(fold_scale(w2, sc2), cin, tdt).to(dev), sh2.float().to(dev).contiguous()
    op.tail_cout, op.tail_relu = w2.shape[0], int(relu2)
    op.tail_weight, op.tail_shift = keep[0].data_ptr(), keep[1].data_ptr()
    return keep


def _run_op(op, ws, x=None, fmt=0, impl=nat.CONV_UMMA):
    with torch.cuda.device(ws.device):
        rc = nat.lib().lfd_run_op(C.byref(op), nat.ptr(x), fmt, nat.ptr(ws.buf), None, None, 0, 0, impl, nat.stream_ptr())
        torch.cuda.synchronize()
    return rc


def run_conv(x_nhwc, weight, scale, shift, stride, relu, res=None, gn_groups=0, impl=nat.CONV_UMMA, tail=None, dtype='bf16', max_ctas=0,
             ds=None, inplace=False):
    """x_nhwc: cuda bf16 / fp16 [N,H,W,Cin]; weight fp32 [Cout,Cin,k,k] (already representable in the 16-bit type).
    max_ctas: lfd_op.max_ctas (0 = one persistent CTA per SM).  ds = (w3 [Cout,Cin,1,1], scale3, shift3): the fused 1x1/s2
    shortcut of a 3x3/s2 conv (lfd_op.ds_cout).  inplace: the residual is read from the output tensor (out == res).
    Every tensor sits in a guarded, poisoned Workspace whose guards are checked after the launch.
    -> (out [N,Ho,Wo,Cf], stats double [N,groups,2] or None, conv_query dict), plus the shortcut output [N,Ho,Wo,Cout] with ds"""
    tdt = DTYPES[dtype][0]
    assert x_nhwc.dtype == tdt
    dev = x_nhwc.device
    N, H, W, Cin = x_nhwc.shape
    Cout, _, k, _ = weight.shape
    Ho, Wo = conv_out(H, k, stride), conv_out(W, k, stride)
    Cf = tail[0].shape[0] if tail is not None else Cout
    q = nat.conv_query(N, H, W, Cin, Ho, Wo, Cout, k, stride, Cf if tail is not None else 0, Cout if ds is not None else 0)
    wp = pack_conv_weight(fold_scale(weight, scale), q['cc'], tdt).to(dev)   # BatchNorm scale folded before the bf16 rounding
    sh = shift.float().to(dev).contiguous()
    ws = Workspace(dev, guard=GUARD, poison=True)
    ws.add('in', x_nhwc)
    if inplace:
        ws.add('out', res)
    else:
        ws.add('out', shape=(N, Ho, Wo, Cf), dtype=tdt)
        if res is not None:
            ws.add('res', res)
    if gn_groups:
        ws.add('stats', shape=(N, gn_groups, 2), dtype=torch.float64, zero=True)
    if ds is not None:
        ws.add('ds', shape=(N, Ho, Wo, Cout), dtype=tdt)
    ws.finalize()
    op = make_op(nat.OP_CONV, dtype, N=N, H=H, W=W, Cin=Cin, Ho=Ho, Wo=Wo, Cout=Cout, ksize=k, stride=stride, relu=int(relu),
                 gn_groups=gn_groups, cc=q['cc'], max_ctas=max_ctas, in_off=ws.off('in'), out_off=ws.off('out'),
                 res_off=ws.off('out' if inplace else 'res' if res is not None else None), stats_off=ws.off('stats' if gn_groups else None),
                 weight=wp.data_ptr(), shift=sh.data_ptr())
    keep = list(_set_tail(op, tail, Cout, tdt, dev)) if tail is not None else []
    if ds is not None:
        w3, sc3, sh3 = ds
        keep += [pack_conv_weight(fold_scale(w3, sc3), Cin, tdt).to(dev), sh3.float().to(dev).contiguous()]     # [Cin/8][Cout][8]
        op.ds_cout, op.ds_out_off = Cout, ws.off('ds')
        op.ds_weight, op.ds_shift = keep[-2].data_ptr(), keep[-1].data_ptr()
    nat.check(_run_op(op, ws, impl=impl))
    ws.assert_guards('conv N%d %dx%d %d-%d k%ds%d' % (N, H, W, Cin, Cout, k, stride))
    stats = ws.get('stats') if gn_groups else None
    if ds is not None:
        return ws.get('out'), stats, q, ws.get('ds')
    return ws.get('out'), stats, q


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


def run_stem0(x, fmt, w, shift, *, cin=3, relu=True, tail=None, transform=None, dtype='bf16', impl=nat.CONV_UMMA, max_ctas=0, raw_rc=False):
    """LFD_OP_STEM0 with Cin = cin through lfd_run_op.  x (fmt, a nat.INPUT_* code): float32 [N,cin,H,W], uint8 [N,H,W,cin] or gray
    [N,H,W], NV12 [N,3H/2,W]; w fp32 [Cout,cin,3,3] with the BatchNorm scale already folded in (rounded to the 16-bit type by the
    packing); tail as in run_conv.  The output sits in a guarded, poisoned Workspace whose guards are checked after the launch.
    -> (out [N,Ho,Wo,Cf], number of 16 x 8 output tiles); raw_rc: -> (lfd_run_op's return code, the workspace bytes), unchecked"""
    tdt = DTYPES[dtype][0]
    dev = x.device
    N = x.shape[0]
    if fmt == nat.INPUT_F32_NCHW:
        H, W = x.shape[2], x.shape[3]
    elif fmt == nat.INPUT_U8_NV12:
        H, W = x.shape[1] * 2 // 3, x.shape[2]
    else:
        H, W = x.shape[1], x.shape[2]
    Cout = w.shape[0]
    Ho, Wo = conv_out(H, 3, 2), conv_out(W, 3, 2)
    Cf = tail[0].shape[0] if tail is not None else Cout
    wp, sh = pack_stem_weight(w, tdt).to(dev), shift.float().to(dev).contiguous()
    ws = Workspace(dev, guard=GUARD, poison=True)
    ws.add('out', shape=(N, Ho, Wo, Cf), dtype=tdt)
    ws.finalize()
    op = make_op(nat.OP_STEM0, dtype, transform, N=N, H=H, W=W, Cin=cin, Ho=Ho, Wo=Wo, Cout=Cout, ksize=3, stride=2, relu=int(relu),
                 max_ctas=max_ctas, out_off=ws.off('out'), weight=wp.data_ptr(), shift=sh.data_ptr())
    keep = _set_tail(op, tail, Cout, tdt, dev) if tail is not None else None    # noqa: F841  (alive until the launch)
    rc = _run_op(op, ws, x.contiguous(), fmt, impl)
    if raw_rc:
        return rc, ws.buf
    nat.check(rc)
    ws.assert_guards('stem0 N%d %dx%d Cin %d Cout %d tail %d' % (N, H, W, cin, Cout, Cf if tail is not None else 0))
    return ws.get('out'), N * ((Ho + 15) // 16) * ((Wo + 7) // 8)


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


# ------------------------------------------------------------------------------------------------ op-level conv and stem cases
# conv case: (N, H, W, Cin, Cout, k, s, relu, res, gn, tail, ds); stem case: (Cout, tail, fmt 'u8' / 'f32', H, W).  Each test module
# passes its own seed, so its operands stay what they have always been.
STEM_FMT = {'u8': nat.INPUT_U8_NHWC, 'f32': nat.INPUT_F32_NCHW}


@functools.lru_cache(maxsize=None)
def conv_operands(case, dtype, seed):
    """-> (x, w, scale, shift, res or None, tail (w2, scale2, shift2, relu) or None, shortcut (w3, scale3, shift3) or None), drawn in
    that order"""
    N, H, W, Cin, Cout, k, s, relu, use_res, gn, tail, ds = case
    tdt = DTYPES[dtype][0]
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((N, H, W, Cin), generator=g).to(tdt)
    w = torch.randn((Cout, Cin, k, k), generator=g) * (2.0 / (Cin * k * k)) ** 0.5
    scale, shift = torch.rand((Cout,), generator=g) + 0.5, torch.randn((Cout,), generator=g) * 0.2
    Cf = tail or Cout
    Ho, Wo = conv_out(H, k, s), conv_out(W, k, s)
    res = torch.randn((N, Ho, Wo, Cf), generator=g).to(tdt) if use_res else None
    t = None
    if tail:
        t = (torch.randn((tail, Cout, 1, 1), generator=g) * (2.0 / Cout) ** 0.5, torch.rand((tail,), generator=g) + 0.5,
             torch.randn((tail,), generator=g) * 0.2, bool(relu))
    d = None
    if ds:
        d = (torch.randn((Cout, Cin, 1, 1), generator=g) * (1.0 / Cin) ** 0.5, torch.rand((Cout,), generator=g) + 0.5,
             torch.randn((Cout,), generator=g) * 0.2)
    return x, w, scale, shift, res, t, d


@functools.lru_cache(maxsize=None)
def conv_reference(case, dtype, seed):
    """(ref64, S, K) of the stored output (tail: the two-layer chain with the 16-bit intermediate) and of the shortcut output (or None)."""
    N, H, W, Cin, Cout, k, s, relu, use_res, gn, tail, ds = case
    x, w, scale, shift, res, t, d = conv_operands(case, dtype, seed)
    rnd = DTYPES[dtype][1]
    if tail:
        mid, _, _ = ref_conv64(x, w, scale, shift, s, relu, dtype=dtype)
        main = ref_conv64(rnd(mid.float()), t[0], t[1], t[2], 1, t[3], res=res, dtype=dtype)
    else:
        main = ref_conv64(x, w, scale, shift, s, relu, res=res, dtype=dtype)
    # the shortcut reads the conv's centre tap: a 1x1/s2 conv of the same input, stored without ReLU
    short = ref_conv64(x[:, ::2, ::2, :], d[0], d[1], d[2], 1, False, dtype=dtype) if ds else None
    return main, short


def run_conv_case(case, dtype, seed, max_ctas=0, impl=nat.CONV_UMMA, inplace=False):
    """run_conv on conv_operands(case, dtype, seed) -> (out, stats or None, conv_query, shortcut output or None)"""
    N, H, W, Cin, Cout, k, s, relu, use_res, gn, tail, ds = case
    x, w, scale, shift, res, t, d = conv_operands(case, dtype, seed)
    r = run_conv(x.cuda(), w, scale, shift, s, bool(relu), res=None if res is None else res.cuda(), gn_groups=gn, impl=impl, tail=t,
                 dtype=dtype, max_ctas=max_ctas, ds=d, inplace=inplace)
    return r if ds else r + (None,)


@functools.lru_cache(maxsize=None)
def stem_operands(case, seed):
    """-> (image, w with the BatchNorm scale folded in, shift, tail (w2, scale2, shift2, True) or None)"""
    Cout, tail, fmt, H, W = case
    N = 2
    g = torch.Generator().manual_seed(seed)
    if fmt == 'u8':
        img = torch.randint(0, 256, (N, H, W, 3), generator=g, dtype=torch.uint8)
    else:
        img = torch.randn((N, 3, H, W), generator=g)
    w = torch.randn((Cout, 3, 3, 3), generator=g) * (2.0 / 27) ** 0.5 * (torch.rand((Cout, 1, 1, 1), generator=g) + 0.5)
    shift = torch.randn((Cout,), generator=g) * 0.2
    t = None
    if tail:
        t = (torch.randn((tail, Cout, 1, 1), generator=g) * (2.0 / Cout) ** 0.5, torch.rand((tail,), generator=g) + 0.5,
             torch.randn((tail,), generator=g) * 0.2, True)
    return img, w, shift, t
