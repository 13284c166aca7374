# -*- coding: utf-8 -*-
"""One op launched on a frame below its capacity through the production entry points: lfd_plan_create on a hand-built op list, then
lfd_plan_forward_extent with a hand-built geometry table (lfd_extent), so the op runs its EXT = true kernel build.  The same op on
tensors of the frame's own size runs through lfd_run_op (the EXT = false build).

lfd_plan_forward_extent needs op 0 to read the image and takes the table only for a frame below the image op's capacity.  So an op that
does not read the image (CONV, GN_APPLY, HEAD_FINAL) runs behind a small dummy STEM0 (16 x 16 capacity, 8 x 8 frame) that writes its own
workspace region; a STEM0 / STEM4 under test is the plan's only op.

Operands lie in the capacity layout (row pitch = the capacity width) with the frame in the top-left corner, and every byte outside the
frame is poison: 0xff in the workspace (NaN in bf16 and fp16), NaN in fp32 images, 255 in uint8 BGR and NV12 bytes.  Every region has
NaN guard bytes behind it.  After a launch, every byte outside the regions the op may write must be what it was before."""
import ctypes as C
import functools

import torch

from gpu_ops import DTYPES, conv_out, ref_conv64, stem_operand
from helpers import bits  # noqa: F401  (X.bits of test_gpu_extent_configs.py)
from lfd import _native as nat
from lfd._engine import fold_scale, pack_conv_weight, pack_stem_weight
from nv12_oracle import nv12_frames, nv12_oracle

GUARD = 4096
STEM_CAP, STEM_FRAME = 16, 8           # the dummy image op: capacity and frame
EPS = 1e-5


def al(v):
    return (v + 255) & ~255


def roundup(v, m):
    return (v + m - 1) // m * m


def _dev(t):
    return t.contiguous().cuda()


def poisoned(shape, dtype):
    """A tensor of poison: NaN for floating types, 255 for uint8."""
    if dtype == torch.uint8:
        return torch.full(shape, 255, dtype=torch.uint8)
    return torch.full(shape, float('nan'), dtype=dtype)


class Rig(object):
    """One op in a poisoned workspace at tensor geometry H x W.  plan=True: the op runs through a plan and lfd_plan_forward_extent
    (the tensors are the capacity's, frames below it); plan=False: through lfd_run_op on tensors of the frame's own size (H x W = the
    frame).  spec supplies the op, its regions and its operands."""

    def __init__(self, spec, H, W, max_ctas=0, plan=True):
        self.spec, self.H, self.W, self.max_ctas, self.use_plan = spec, H, W, max_ctas, plan
        regions = list(spec.regions(H, W))
        if plan and not spec.reads_image:
            regions.append(('stem', spec.N * (STEM_CAP // 2) ** 2 * 16 * 2))
        self.off, self.nb, top = {}, {}, 0
        for name, nb in regions:              # 'stats' first: the statistics sit at workspace offset 0
            self.off[name], self.nb[name] = top, nb
            top += al(nb) + GUARD
        self.ws = torch.full((top,), 0xff, dtype=torch.uint8, device='cuda')
        self.keep = []
        self.op = spec.op(self, H, W)
        self.op.max_ctas = max_ctas
        self.cls, self.reg = spec.head_buffers(H, W)
        self.image = None
        self.handle = None
        if plan:
            ops = []
            if not spec.reads_image:
                ops.append(self._dummy_stem())
            ops.append(self.op)
            self.ops = (nat.Op * len(ops))(*ops)
            self.index = len(ops) - 1
            stats_bytes = self.nb.get('stats', 0) if spec.clear_stats else 0
            h = C.c_void_p()
            with torch.cuda.device(self.ws.device):
                nat.check(nat.lib().lfd_plan_create(self.ops, len(ops), spec.N, spec.P(H, W), spec.cls_channels, 0, stats_bytes,
                                                    self.ws.numel(), nat.CONV_UMMA, C.byref(h)))
            self.handle = h
            if not spec.reads_image:
                self.image = torch.zeros((spec.N, STEM_CAP, STEM_CAP, 3), dtype=torch.uint8, device='cuda')

    def _dummy_stem(self):
        o = nat.Op()
        tdt, code = DTYPES[self.spec.dtype][0], DTYPES[self.spec.dtype][3]
        w, sh = pack_stem_weight(torch.zeros(16, 3, 3, 3), tdt).cuda(), torch.zeros(16, device='cuda')
        self.keep += [w, sh]
        o.kind, o.dtype = nat.OP_STEM0, code
        o.N, o.H, o.W, o.Cin, o.Ho, o.Wo, o.Cout = self.spec.N, STEM_CAP, STEM_CAP, 3, STEM_CAP // 2, STEM_CAP // 2, 16
        o.ksize, o.stride, o.relu = 3, 2, 1
        o.in_off, o.out_off, o.res_off, o.stats_off, o.ds_out_off = -1, self.off['stem'], -1, -1, -1
        o.weight, o.shift = w.data_ptr(), sh.data_ptr()
        return o

    def close(self):
        if self.handle is not None:
            nat.check(nat.lib().lfd_plan_destroy(self.handle))
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def view(self, name, dtype, shape):
        off, nb = self.off[name], self.nb[name]
        return self.ws[off:off + nb].view(dtype).view(shape)

    def load(self, h, w):
        """Poison the workspace and the head outputs, then write the frame's operands."""
        self.ws.fill_(0xff)
        for b in (self.cls, self.reg):
            if b is not None:
                b.view(torch.uint8).fill_(0xff)
        self.spec.load(self, h, w)
        if 'stats' in self.nb and self.spec.clear_stats and not self.use_plan:
            self.ws[:self.nb['stats']].zero_()            # lfd_run_op does not clear them; a plan's clear region does
        self.before = self.ws.clone()

    def run(self, h, w, use_graph=0):
        spec = self.spec
        cls = self.cls if self.cls is not None else _scratch()
        reg = self.reg if self.reg is not None else _scratch()
        with torch.cuda.device(self.ws.device):
            if self.use_plan:
                assert (h, w) != (self.H, self.W) or not spec.reads_image
                ext = (nat.Extent * len(self.ops))()
                if not spec.reads_image:
                    ext[0].H, ext[0].W, ext[0].Ho, ext[0].Wo = STEM_FRAME, STEM_FRAME, STEM_FRAME // 2, STEM_FRAME // 2
                    fh, fw, fmt = STEM_FRAME, STEM_FRAME, nat.INPUT_U8_NHWC
                else:
                    fh, fw, fmt = h, w, spec.fmt_code
                ext[self.index].H, ext[self.index].W, ext[self.index].Ho, ext[self.index].Wo, ext[self.index].point_off, \
                    ext[self.index].P = spec.row(h, w)
                nat.check(nat.lib().lfd_plan_forward_extent(self.handle, nat.ptr(self.image), fmt, fh, fw, ext, nat.ptr(self.ws), nat.ptr(cls),
                                                             nat.ptr(reg), use_graph, nat.stream_ptr()))
            else:
                assert (h, w) == (self.H, self.W)
                P, cs = spec.row(h, w)[5] or 1, spec.cls_channels
                nat.check(nat.lib().lfd_run_op(C.byref(self.op), nat.ptr(self.image) if spec.reads_image else None,
                                               spec.fmt_code if spec.reads_image else 0, nat.ptr(self.ws), nat.ptr(cls), nat.ptr(reg), P, cs,
                                               nat.CONV_UMMA, nat.stream_ptr()))
            torch.cuda.synchronize()

    def assert_untouched(self, what):
        """Every byte outside the regions the op may write (and the dummy stem's output) is what it was before the launch: guards,
        inputs, residuals."""
        mask = torch.ones(self.ws.numel(), dtype=torch.bool, device=self.ws.device)
        for name in self.spec.writable + ('stem',):
            if name in self.off:
                mask[self.off[name]:self.off[name] + self.nb[name]] = False
        bad = (self.ws != self.before) & mask
        if bool(bad.any()):
            i = int(torch.nonzero(bad)[0])
            where = [n for n in self.off if self.off[n] <= i < self.off[n] + al(self.nb[n]) + GUARD]
            raise AssertionError('%s: %d bytes outside the op\'s outputs were written, first at byte %d (after region %s)'
                                 % (what, int(bad.sum()), i, where))


@functools.lru_cache(maxsize=1)
def _scratch_buf():
    return torch.full((64,), float('nan'), device='cuda')


def _scratch():
    return _scratch_buf()


def assert_poison(t, what):
    """Every element of t (a view of a poisoned buffer) still holds the poison bytes."""
    b = t.contiguous().view(torch.uint8)
    if not bool((b == 0xff).all()):
        raise AssertionError('%s: %d bytes written' % (what, int((b != 0xff).sum())))


def assert_untouched_beyond_tiles(out, ho, wo, flat, what):
    """out: an output in the capacity layout [N, Ho, Wo, C].  Spatial tiles are 16 rows x 8 columns of the valid extent's tile grid, so
    nothing beyond roundup(ho, 16) rows or roundup(wo, 8) columns may be written; flat tiles are 128 consecutive pixels at the capacity
    pitch over the first ho rows, so nothing past the last of them may be."""
    N, Ho, Wo, Cf = out.shape
    if flat:
        assert_poison(out.reshape(N, Ho * Wo, Cf)[:, roundup(ho * Wo, 128):], what + ' beyond the last flat tile')
    else:
        assert_poison(out[:, roundup(ho, 16):], what + ' below the last tile row')
        assert_poison(out[:, :, roundup(wo, 8):], what + ' right of the last tile column')


# ------------------------------------------------------------------------------------------------------------------ CONV
class ConvSpec(object):
    """LFD_OP_CONV (N, H, W, Cin, Cout, k, s, relu, res, gn, tail, ds) as in test_gpu_conv_configs.CASES, at the capacity H x W."""
    reads_image, clear_stats, cls_channels = False, True, 1
    writable = ('stats', 'out', 'ds')

    def __init__(self, case, dtype):
        self.case, self.dtype = case, dtype
        N, H, W, Cin, Cout, k, s, relu, use_res, gn, tail, ds = case
        self.N, self.k, self.s, self.Cf = N, k, s, tail or Cout
        self.flat = (k, s) == (1, 1)
        tdt = DTYPES[dtype][0]
        g = torch.Generator().manual_seed(hash(case) & 0xffff)
        self.x = torch.randn((N, H, W, Cin), generator=g).to(tdt)
        self.w = torch.randn((Cout, Cin, k, k), generator=g) * (2.0 / (Cin * k * k)) ** 0.5
        self.scale, self.shift = torch.rand((Cout,), generator=g) + 0.5, torch.randn((Cout,), generator=g) * 0.2
        Ho, Wo = conv_out(H, k, s), conv_out(W, k, s)
        self.res = torch.randn((N, Ho, Wo, self.Cf), generator=g).to(tdt) if use_res else None
        self.t = self.d = None
        if tail:
            self.t = (torch.randn((tail, Cout, 1, 1), generator=g) * (2.0 / Cout) ** 0.5, torch.rand((tail,), generator=g) + 0.5,
                      torch.randn((tail,), generator=g) * 0.2, bool(relu))
        if ds:
            self.d = (torch.randn((Cout, Cin, 1, 1), generator=g) * (1.0 / Cin) ** 0.5, torch.rand((Cout,), generator=g) + 0.5,
                      torch.randn((Cout,), generator=g) * 0.2)
        self.q = nat.conv_query(N, H, W, Cin, Ho, Wo, Cout, k, s, tail, Cout if ds else 0)
        self.wp = pack_conv_weight(fold_scale(self.w, self.scale), self.q['cc'], tdt).cuda()
        self.sh = _dev(self.shift.float())
        if tail:
            self.w2p, self.sh2 = pack_conv_weight(fold_scale(self.t[0], self.t[1]), Cout, tdt).cuda(), _dev(self.t[2].float())
        if ds:
            self.w3p, self.sh3 = pack_conv_weight(fold_scale(self.d[0], self.d[1]), Cin, tdt).cuda(), _dev(self.d[2].float())

    def out_size(self, h, w):
        return conv_out(h, self.k, self.s), conv_out(w, self.k, self.s)

    def P(self, H, W):
        return 1

    def head_buffers(self, H, W):
        return None, None

    def row(self, h, w):
        return (h, w) + self.out_size(h, w) + (0, 0)

    def regions(self, H, W):
        N, _, _, Cin, Cout, k, s, relu, use_res, gn, tail, ds = self.case
        Ho, Wo = self.out_size(H, W)
        r = [('stats', N * gn * 16)] if gn else []
        r += [('in', N * H * W * Cin * 2), ('out', N * Ho * Wo * self.Cf * 2)]
        if use_res:
            r.append(('res', N * Ho * Wo * self.Cf * 2))
        if ds:
            r.append(('ds', N * Ho * Wo * Cout * 2))
        return r

    def op(self, rig, H, W):
        N, _, _, Cin, Cout, k, s, relu, use_res, gn, tail, ds = self.case
        Ho, Wo = self.out_size(H, W)
        o = nat.Op()
        o.kind, o.dtype = nat.OP_CONV, DTYPES[self.dtype][3]
        o.N, o.H, o.W, o.Cin, o.Ho, o.Wo, o.Cout = N, H, W, Cin, Ho, Wo, Cout
        o.ksize, o.stride, o.relu, o.gn_groups, o.cc = k, s, int(relu), gn, self.q['cc']
        o.in_off, o.out_off = rig.off['in'], rig.off['out']
        o.res_off = rig.off['res'] if use_res else -1
        o.stats_off = 0 if gn else -1
        o.ds_out_off = -1
        o.weight, o.shift = self.wp.data_ptr(), self.sh.data_ptr()
        if tail:
            o.tail_cout, o.tail_relu, o.tail_weight, o.tail_shift = tail, int(self.t[3]), self.w2p.data_ptr(), self.sh2.data_ptr()
        if ds:
            o.ds_cout, o.ds_out_off, o.ds_weight, o.ds_shift = Cout, rig.off['ds'], self.w3p.data_ptr(), self.sh3.data_ptr()
        return o

    def load(self, rig, h, w):
        N, Cin = self.N, self.case[3]
        tdt = DTYPES[self.dtype][0]
        rig.view('in', tdt, (N, rig.H, rig.W, Cin))[:, :h, :w] = self.x[:, :h, :w].cuda()
        if self.res is not None:
            ho, wo = self.out_size(h, w)
            Ho, Wo = self.out_size(rig.H, rig.W)
            rig.view('res', tdt, (N, Ho, Wo, self.Cf))[:, :ho, :wo] = self.res[:, :ho, :wo].cuda()

    def outputs(self, rig):
        """-> {'out': [N, Ho, Wo, Cf], 'ds': [N, Ho, Wo, Cout], 'stats': double [N, 16, 2]} of the tensor geometry, cloned"""
        N, tdt = self.N, DTYPES[self.dtype][0]
        Ho, Wo = self.out_size(rig.H, rig.W)
        r = {'out': rig.view('out', tdt, (N, Ho, Wo, self.Cf)).clone()}
        if self.d is not None:
            r['ds'] = rig.view('ds', tdt, (N, Ho, Wo, self.case[4])).clone()
        if self.case[9]:
            r['stats'] = rig.view('stats', torch.float64, (N, self.case[9], 2)).clone()
        return r

    @functools.lru_cache(maxsize=None)
    def reference(self, h, w):
        """float64 on the cropped operands with zero padding, on the GPU: {'out': (ref, S, K), 'ds': (ref, S, K)}; a fused tail's is the
        two-layer chain with the 16-bit intermediate (S, K None)."""
        rnd = DTYPES[self.dtype][1]
        ho, wo = self.out_size(h, w)
        x = self.x[:, :h, :w]
        res = self.res[:, :ho, :wo] if self.res is not None else None
        s, relu, dt = self.s, bool(self.case[7]), self.dtype
        if self.t is not None:
            mid, _, _ = ref_conv64(x, self.w, self.scale, self.shift, s, relu, dtype=dt, device='cuda')
            ref, _, _ = ref_conv64(rnd(mid.float()), self.t[0], self.t[1], self.t[2], 1, self.t[3], res=res, dtype=dt, device='cuda')
            r = {'out': (ref.cpu(), None, None)}
        else:
            ref, S, K = ref_conv64(x, self.w, self.scale, self.shift, s, relu, res=res, dtype=dt, device='cuda')
            r = {'out': (ref.cpu(), S.cpu(), K)}
        if self.d is not None:
            ref, S, K = ref_conv64(x[:, ::2, ::2, :], self.d[0], self.d[1], self.d[2], 1, False, dtype=dt, device='cuda')
            r['ds'] = (ref.cpu(), S.cpu(), K)
        return r


def conv_extents(case):
    """Frames (h, w, property) below the capacity of a conv case, chosen by the output tile walk they hit.  Stride 2 takes both
    parities of h and w."""
    N, H, W, Cin, Cout, k, s = case[:7]
    Ho, Wo = conv_out(H, k, s), conv_out(W, k, s)

    def inp(o, full, odd):               # an input size whose output size is o
        if s == 1:
            return o
        v = 2 * o - 1 if odd else 2 * o
        return v if v <= full else 2 * o - 1

    ho1, wo1 = max(v for v in range(1, Ho) if v % 16 == 1), max(v for v in range(1, Wo) if v % 8 == 1)
    ex = [(inp(Ho - 1, H, False), inp(Wo - 3, W, True), 'partial last tile in both directions'),
          (inp(ho1, H, True), inp(wo1, W, False), 'ho = 1 (mod 16), wo = 1 (mod 8): one-row and one-column border tiles'),
          (inp(1, H, s == 1), inp(1, W, True), '1 x 1 output'),
          (inp(1, H, False), W, 'full width, one output row: fewer tiles than CTAs'),
          (H, inp(5, W, True), 'full height, 5 output columns (flat: 128-pixel tiles straddle valid and invalid columns)')]
    if k == 3:
        ex.append(halo_extent(case) + ('the last tile\'s halo is in range at the capacity, one row / column past the frame',))
    return ex


def halo_extent(case):
    """3x3 convs: the largest frame (h, w) at which a tile whose halo (iy0 + kDyMax, ix0 + kDxMax) lies inside the capacity reaches
    exactly the first row and column outside the frame, so a capacity-based interior-tile test would read them."""
    H, W, s = case[1], case[2], case[6]
    if s == 1:           # tile origin iy0 = 16 ty (ty >= 1), halo rows iy0 - 1 .. iy0 + 16; columns ix0 - 1 .. ix0 + 8
        hs, ws = range(32, H, 16), range(16, W, 8)
    else:                # iy0 = 32 ty, rows iy0 - 1 .. iy0 + 31; ix0 = 16 tx, columns ix0 - 1 .. ix0 + 15
        hs, ws = range(63, H, 32), range(31, W, 16)
    return max(hs), max(ws)


# ------------------------------------------------------------------------------------------------------------------ STEM0 / STEM4
FMT_CODES = {'f32': nat.INPUT_F32_NCHW, 'u8': nat.INPUT_U8_NHWC, 'nv12': nat.INPUT_U8_NV12}


def transform_of(name):
    """None (zero fields: simple_normalize on BGR) or the InputTransform of a pipeline of test_gpu_input_transform.py"""
    if name is None:
        return None
    from lfd.data_pipeline.augmentation import input_transform_of, typical_coco_val_pipeline
    from test_input_transform_host import tl_val_pipeline
    return input_transform_of({'rgb-standard': tl_val_pipeline, 'caffe': typical_coco_val_pipeline}[name])


class _ImageSpec(object):
    """The image handling shared by STEM0 and STEM4: frames in the capacity layout, poison around them."""
    reads_image, clear_stats, cls_channels = True, False, 1
    writable = ('out',)

    def P(self, H, W):
        return 1

    def head_buffers(self, H, W):
        return None, None

    def frame(self, h, w):
        """The frame's image (CPU): the capacity image's corner for f32 / u8, NV12 frames of the frame's size"""
        if self.fmt == 'nv12':
            return torch.from_numpy(nv12_frames(self.N, h, w, seed=self.seed))
        if self.fmt == 'f32':
            return self.img[:, :, :h, :w].contiguous()
        return self.img[:, :h, :w].contiguous()

    def load(self, rig, h, w):
        N, H, W = self.N, rig.H, rig.W
        f = self.frame(h, w)
        if self.fmt == 'f32':
            img = poisoned((N, 3, H, W), torch.float32)
            img[:, :, :h, :w] = f
        elif self.fmt == 'u8':
            img = poisoned((N, H, W, 3), torch.uint8)
            img[:, :h, :w] = f
        else:
            img = poisoned((N, H * 3 // 2, W), torch.uint8)
            img[:, :h, :w] = f[:, :h]
            img[:, H:H + h // 2, :w] = f[:, h:]
        if rig.image is None:                # one buffer per rig: a captured graph keeps its input pointer
            raw = torch.empty(img.numel() * img.element_size() + 4, dtype=torch.uint8, device='cuda')
            skip = 1 if self.misaligned else 0   # base address 1 (mod 4): the fused stem's per-pixel loader
            rig.image = raw[skip:skip + img.numel() * img.element_size()].view(img.dtype).view(img.shape)
        rig.image.copy_(img)

    def operand(self, h, w):
        return stem_operand(self.frame(h, w), self.fmt, self.xf, self.dtype)

    def outputs(self, rig):
        Ho, Wo = self.out_size(rig.H, rig.W)
        return {'out': rig.view('out', DTYPES[self.dtype][0], (self.N, Ho, Wo, self.Cf)).clone()}

    def regions(self, H, W):
        Ho, Wo = self.out_size(H, W)
        return [('out', self.N * Ho * Wo * self.Cf * 2)]

    def row(self, h, w):
        return (h, w) + self.out_size(h, w) + (0, 0)


class StemSpec(_ImageSpec):
    """LFD_OP_STEM0 (Cout, tail, fmt, transform, N, H, W) at the capacity H x W"""
    flat = False

    def __init__(self, case, dtype):
        self.case, self.dtype = case, dtype
        Cout, tail, fmt, xname, N, H, W = case
        self.fmt, self.fmt_code, self.xf, self.misaligned = fmt, FMT_CODES[fmt], transform_of(xname), False
        self.N, self.H, self.W, self.Cf, self.seed = N, H, W, tail or Cout, Cout * 10 + tail
        g = torch.Generator().manual_seed(Cout * 1000 + tail * 10 + H + W)
        self.img = (torch.randint(0, 256, (N, H, W, 3), generator=g, dtype=torch.uint8) if fmt == 'u8' else
                    torch.randn((N, 3, H, W), generator=g) if fmt == 'f32' else None)
        # caffe-style transforms leave inputs of about +-120: smaller weights keep the outputs in a range where fp16 does not overflow
        gain = 0.01 if xname == 'caffe' else 1.0
        self.w = torch.randn((Cout, 3, 3, 3), generator=g) * (2.0 / 27) ** 0.5 * (torch.rand((Cout, 1, 1, 1), generator=g) + 0.5) * gain
        self.shift = torch.randn((Cout,), generator=g) * 0.2
        self.t = None
        tdt = DTYPES[dtype][0]
        self.wp, self.sh = pack_stem_weight(self.w, tdt).cuda(), _dev(self.shift.float())
        if tail:
            self.t = (torch.randn((tail, Cout, 1, 1), generator=g) * (2.0 / Cout) ** 0.5, torch.rand((tail,), generator=g) + 0.5,
                      torch.randn((tail,), generator=g) * 0.2, True)
            self.w2p, self.sh2 = pack_conv_weight(fold_scale(self.t[0], self.t[1]), Cout, tdt).cuda(), _dev(self.t[2].float())

    def out_size(self, h, w):
        return conv_out(h, 3, 2), conv_out(w, 3, 2)

    def op(self, rig, H, W):
        Cout, tail = self.case[0], self.case[1]
        Ho, Wo = self.out_size(H, W)
        o = nat.Op()
        o.kind, o.dtype = nat.OP_STEM0, DTYPES[self.dtype][3]
        o.N, o.H, o.W, o.Cin, o.Ho, o.Wo, o.Cout = self.N, H, W, 3, Ho, Wo, Cout
        o.ksize, o.stride, o.relu = 3, 2, 1
        o.in_off, o.out_off, o.res_off, o.stats_off, o.ds_out_off = -1, rig.off['out'], -1, -1, -1
        o.weight, o.shift = self.wp.data_ptr(), self.sh.data_ptr()
        if tail:
            o.tail_cout, o.tail_relu, o.tail_weight, o.tail_shift = tail, 1, self.w2p.data_ptr(), self.sh2.data_ptr()
        nat.set_input_transform(o, self.xf)
        return o

    @functools.lru_cache(maxsize=None)
    def reference(self, h, w):
        x, ones, rnd = self.operand(h, w), torch.ones(self.case[0]), DTYPES[self.dtype][1]
        if self.t is not None:
            mid, _, _ = ref_conv64(x, self.w, ones, self.shift, 2, True, dtype=self.dtype, device='cuda')
            ref, _, _ = ref_conv64(rnd(mid.float()), self.t[0], self.t[1], self.t[2], 1, True, dtype=self.dtype, device='cuda')
            return {'out': (ref.cpu(), None, None)}
        ref, S, K = ref_conv64(x, self.w, ones, self.shift, 2, True, dtype=self.dtype, device='cuda')
        return {'out': (ref.cpu(), S.cpu(), K)}


class Stem4Spec(_ImageSpec):
    """LFD_OP_STEM4 (fmt, aligned, N, H, W): the 'faster' stem 3x3/s2 3->64, 1x1 64->64, 3x3/s2 64->64, 1x1 64->64 as one kernel.
    The word loader runs for u8 / NV12 images of capacity W % 4 == 0 at a 4-byte aligned address (aligned = 0: one byte past)."""
    flat = False

    def __init__(self, case, dtype):
        self.case, self.dtype = case, dtype
        fmt, aligned, N, H, W = case
        self.fmt, self.fmt_code, self.xf, self.misaligned = fmt, FMT_CODES[fmt], None, not aligned
        self.N, self.H, self.W, self.Cf, self.seed = N, H, W, 64, 4 + aligned
        g = torch.Generator().manual_seed(H * 1000 + W + aligned)
        self.img = (torch.randint(0, 256, (N, H, W, 3), generator=g, dtype=torch.uint8) if fmt == 'u8' else
                    torch.randn((N, 3, H, W), generator=g) if fmt == 'f32' else None)
        tdt = DTYPES[dtype][0]
        self.layers = []                     # (weight [Cout, Cin, k, k], shift, stride): every conv with ReLU
        for cin, k, s in ((3, 3, 2), (64, 1, 1), (64, 3, 2), (64, 1, 1)):
            w = torch.randn((64, cin, k, k), generator=g) * (2.0 / (cin * k * k)) ** 0.5
            self.layers.append((w, torch.randn((64,), generator=g) * 0.2, s))
        self.packed = [pack_stem_weight(self.layers[0][0], tdt).cuda()] + [pack_conv_weight(w, 64, tdt).cuda() for w, _, _ in self.layers[1:]]
        self.shifts = [_dev(sh.float()) for _, sh, _ in self.layers]

    def out_size(self, h, w):
        return conv_out(conv_out(h, 3, 2), 3, 2), conv_out(conv_out(w, 3, 2), 3, 2)

    def word_loader(self):
        return self.fmt != 'f32' and self.W % 4 == 0 and not self.misaligned

    def op(self, rig, H, W):
        Ho, Wo = self.out_size(H, W)
        o = nat.Op()
        o.kind, o.dtype = nat.OP_STEM4, DTYPES[self.dtype][3]
        o.N, o.H, o.W, o.Cin, o.Ho, o.Wo, o.Cout = self.N, H, W, 3, Ho, Wo, 64
        o.ksize, o.stride, o.relu = 3, 2, 1
        o.in_off, o.out_off, o.res_off, o.stats_off, o.ds_out_off = -1, rig.off['out'], -1, -1, -1
        o.weight, o.shift = self.packed[0].data_ptr(), self.shifts[0].data_ptr()
        o.tail_cout, o.tail_relu, o.tail_weight, o.tail_shift = 64, 1, self.packed[1].data_ptr(), self.shifts[1].data_ptr()
        o.s2_relu, o.s2_weight, o.s2_shift = 1, self.packed[2].data_ptr(), self.shifts[2].data_ptr()
        o.s3_relu, o.s3_weight, o.s3_shift = 1, self.packed[3].data_ptr(), self.shifts[3].data_ptr()
        return o

    @functools.lru_cache(maxsize=None)
    def reference(self, h, w):
        """The four-conv chain with every intermediate rounded to 16 bits, as the kernel rounds it (bound of a fused tail)"""
        t, rnd = self.operand(h, w), DTYPES[self.dtype][1]
        for wt, sh, s in self.layers:
            ref, _, _ = ref_conv64(t, wt, torch.ones(64), sh, s, True, dtype=self.dtype, device='cuda')
            t = rnd(ref.float())
        return {'out': (ref.cpu(), None, None)}


# ------------------------------------------------------------------------------------------------------------------ GN_APPLY / HEAD_FINAL
def _write_stats(rig, x, groups):
    """The GroupNorm statistics of x [N, h, w, C] (the valid pixels of the 16-bit input), fp64, into the statistics region"""
    N, C = x.shape[0], x.shape[-1]
    v = x.double().reshape(N, -1, groups, C // groups)
    st = torch.stack([v.sum(dim=(1, 3)), (v * v).sum(dim=(1, 3))], -1)
    rig.view('stats', torch.float64, (N, groups, 2)).copy_(st.cuda())
    return st


class GnSpec(object):
    """LFD_OP_GN_APPLY (C, N, H, W), groups = C / 8: the test writes the statistics of the frame's pixels"""
    reads_image, clear_stats, cls_channels, flat = False, False, 1, False
    writable = ('out',)

    def __init__(self, case, dtype):
        self.case, self.dtype = case, dtype
        C_, N, H, W = case
        self.C, self.N, self.G = C_, N, C_ // 8
        g = torch.Generator().manual_seed(C_ * 7 + H + W)
        self.x = (torch.randn((N, H, W, C_), generator=g) * 1.5 + 0.3).to(DTYPES[dtype][0])
        self.gamma, self.beta = torch.rand((C_,), generator=g) + 0.5, torch.randn((C_,), generator=g) * 0.3
        self.gd, self.bd = _dev(self.gamma), _dev(self.beta)

    def P(self, H, W):
        return 1

    def head_buffers(self, H, W):
        return None, None

    def out_size(self, h, w):
        return h, w

    def row(self, h, w):
        return (h, w, h, w, 0, 0)

    def regions(self, H, W):
        nb = self.N * H * W * self.C * 2
        return [('stats', self.N * self.G * 16), ('in', nb), ('out', nb)]

    def op(self, rig, H, W):
        o = nat.Op()
        o.kind, o.dtype = nat.OP_GN_APPLY, DTYPES[self.dtype][3]
        o.N, o.H, o.W, o.Cin, o.Ho, o.Wo, o.Cout = self.N, H, W, self.C, H, W, self.C
        o.gn_groups, o.relu = self.G, 1
        o.in_off, o.out_off, o.res_off, o.stats_off, o.ds_out_off = rig.off['in'], rig.off['out'], -1, 0, -1
        o.gamma, o.beta = self.gd.data_ptr(), self.bd.data_ptr()
        return o

    def load(self, rig, h, w):
        x = self.x[:, :h, :w]
        rig.view('in', DTYPES[self.dtype][0], (self.N, rig.H, rig.W, self.C))[:, :h, :w] = x.cuda()
        rig.stats = _write_stats(rig, x, self.G)

    def outputs(self, rig):
        return {'out': rig.view('out', DTYPES[self.dtype][0], (self.N, rig.H, rig.W, self.C)).clone()}

    @functools.lru_cache(maxsize=None)
    def reference(self, h, w):
        from train_op_ref import head_activation
        x = self.x[:, :h, :w]
        v = x.double().reshape(self.N, -1, self.G, 8)
        st = torch.stack([v.sum(dim=(1, 3)), (v * v).sum(dim=(1, 3))], -1)
        a, a_b, _ = head_activation(x.double().reshape(self.N, h * w, self.C), self.gamma, self.beta, st, self.G, EPS, self.dtype)
        return a.reshape(x.shape), a_b.reshape(x.shape)


HEAD_PRE, HEAD_POST = 50, 20          # points of the other levels before / after the head's level at the capacity
FRAME_PRE, FRAME_POST = 13, 5         # ... and for the frame


class HeadSpec(object):
    """LFD_OP_HEAD_FINAL (n_cls, n_reg, gn, N, H, W) on 128 channels (the only width head_final_kernel takes), gn = 16 groups or 0 (a
    tower without norm layers).  The level starts at point HEAD_PRE of the capacity's P and at FRAME_PRE of the frame's."""
    reads_image, clear_stats, flat = False, False, False
    writable = ()                     # cls / reg are outside the workspace

    def __init__(self, case, dtype):
        self.case, self.dtype = case, dtype
        n_cls, n_reg, gn, N, H, W = case
        self.n_cls, self.n_reg, self.G, self.N, self.C = n_cls, n_reg, gn, N, 128
        self.cls_channels = max(n_cls, 1)
        n_out = n_cls + n_reg
        g = torch.Generator().manual_seed(n_cls * 100 + n_reg * 10 + gn + H + W)
        raw = torch.randn((N, H, W, 128), generator=g) * 1.5 + 0.3
        self.x = (raw if gn else raw.clamp(min=-0.5)).to(DTYPES[dtype][0])
        self.gamma, self.beta = torch.rand((128,), generator=g) + 0.5, torch.randn((128,), generator=g) * 0.3
        self.w = torch.randn((n_out, 128), generator=g) * (1.0 / 128) ** 0.5
        self.scale, self.shift = torch.rand((n_out,), generator=g) + 0.5, torch.randn((n_out,), generator=g) * 0.2
        self.dev = [_dev(t.float()) for t in (self.gamma, self.beta, self.w, self.scale, self.shift)]

    def P(self, H, W):
        return HEAD_PRE + H * W + HEAD_POST

    def frame_P(self, h, w):
        return FRAME_PRE + h * w + FRAME_POST

    def head_buffers(self, H, W):
        P = self.P(H, W)
        return (torch.full((self.N * P * self.cls_channels,), float('nan'), device='cuda'),
                torch.full((self.N * P * 4,), float('nan'), device='cuda'))

    def out_size(self, h, w):
        return h, w

    def row(self, h, w):
        return (h, w, h, w, FRAME_PRE, self.frame_P(h, w))

    def regions(self, H, W):
        r = [('stats', self.N * self.G * 16)] if self.G else []
        return r + [('in', self.N * H * W * 256)]

    def op(self, rig, H, W):
        o = nat.Op()
        o.kind, o.dtype = nat.OP_HEAD_FINAL, DTYPES[self.dtype][3]
        o.N, o.H, o.W, o.Cin, o.Ho, o.Wo, o.Cout = self.N, H, W, 128, H, W, self.n_cls + self.n_reg
        o.gn_groups, o.n_cls, o.n_reg = self.G, self.n_cls, self.n_reg
        # a full-size launch takes the frame's level start from the op; a launch with a geometry row must take the row's
        o.point_off = HEAD_PRE if rig.use_plan else FRAME_PRE
        o.in_off, o.out_off, o.res_off, o.stats_off, o.ds_out_off = rig.off['in'], -1, -1, 0 if self.G else -1, -1
        o.gamma, o.beta, o.weight, o.scale, o.shift = [t.data_ptr() for t in self.dev]
        return o

    def load(self, rig, h, w):
        x = self.x[:, :h, :w]
        rig.view('in', DTYPES[self.dtype][0], (self.N, rig.H, rig.W, 128))[:, :h, :w] = x.cuda()
        if self.G:
            _write_stats(rig, x, self.G)

    def outputs(self, rig, h, w):
        """-> cls [N, P_frame, cls_channels], reg [N, P_frame, 4] (the frame's layout at the start of the buffers) and the rest of
        each buffer"""
        P = self.frame_P(h, w)
        n = self.N * P
        return (rig.cls[:n * self.cls_channels].view(self.N, P, self.cls_channels).clone(), rig.reg[:n * 4].view(self.N, P, 4).clone(),
                rig.cls[n * self.cls_channels:].clone(), rig.reg[n * 4:].clone())

    @functools.lru_cache(maxsize=None)
    def reference(self, h, w):
        from train_op_ref import head_activation, head_forward_ref
        x = self.x[:, :h, :w]
        st = None
        if self.G:
            v = x.double().reshape(self.N, -1, self.G, 8)
            st = torch.stack([v.sum(dim=(1, 3)), (v * v).sum(dim=(1, 3))], -1)
        a, a_b, _ = head_activation(x.double().reshape(self.N, h * w, 128), self.gamma, self.beta, st, self.G, EPS, self.dtype)
        return head_forward_ref(a, a_b, self.w, self.scale, self.shift)


def frame_extents(H, W, even=False, stem=False):
    """Frames below an H x W capacity for STEM0, GN_APPLY and HEAD_FINAL: a partial last tile, ho = 1 (mod 16) and wo = 1 (mod 8)
    of the stride-2 stem, 1 x 1, full width with one output row, full height at a narrow width; stem: the frame at which the stem tile
    (1, 1), whose 33 x 18 image patch lies inside a capacity of at least 64 x 33, reaches the first row and column past the frame.
    even: NV12 frames (even h and w)."""
    ex = [(H - 1, W - 3, 'partial last tile in both directions'),
          (33, 17, 'stem output 17 x 9: ho = 1 (mod 16), wo = 1 (mod 8)') if stem else (17, 9, 'h = 1 (mod 16), w = 1 (mod 8)'),
          (1, 1, '1 x 1'),
          (2, W, 'full width, one stem output row: fewer tiles than CTAs'),
          (H, 9, 'full height, narrow')]
    if stem:
        assert H >= 64 and W >= 33
        ex.append((63, 32, 'stem patch rows 31..63, columns 15..32: in range at the capacity, one past the frame'))
    if even:
        ex = [(max(2, h - h % 2), max(2, w - w % 2), why) for h, w, why in ex]
    return ex
