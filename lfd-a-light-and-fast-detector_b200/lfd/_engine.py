# -*- coding: utf-8 -*-
"""Layer-plan builder: walks an lfd.model.LFD module tree once per (batch, height, width), folds BatchNorm
into per-channel scale/shift, packs conv weights into the wgmma kernel's operand order, lays the bf16 NHWC
activations out in one workspace with liveness-based reuse, and hands the op list to liblfd_b200.so
(lfd_plan_create / lfd_plan_forward).

Replaces the module-by-module execution of LFD.forward (reference lfd/model/lfd.py:511-542).

Rounding points of the bf16 pipeline (mirrored by oracle/lfd_oracle.py forward(emulate_bf16=True)):
  R0  the input image is rounded to bf16 when the stem kernel loads it;
  Rw  backbone / neck / tower conv weights are multiplied by the folded BatchNorm scale in fp32 and THEN rounded to bf16;
      the folded shift (bias) is rounded to bf16 and added on the tensor core (an extra K = 16 MMA against a constant
      operand), so the accumulator already holds conv*scale + shift; the final head convs keep fp32 bias / Scale;
  Ra  every fused layer output (after scale/shift, residual add, ReLU) is stored as bf16;
  Rg  GroupNorm statistics are taken over the stored (bf16) tensor, the normalised+ReLU'd value is rounded
      to bf16 again; the final cls / reg outputs are fp32.
"""
import ctypes as C
import struct
import time
import zlib

import torch
import torch.nn as nn

from . import _native as nat

BN_TYPES = (nn.BatchNorm2d,)


def conv_out(size, k, s):
    return (size + 2 * (k // 2) - k) // s + 1


def level_geometry(backbone, head, h, w):
    """Sizes of the head levels for a stem output of h x w (every stage starts with a stride-2 block) -> (level_sizes, P, offset of
    each level's first point)."""
    taps = list(backbone._out_indices)
    if len(taps) != head._num_heads:
        raise ValueError('backbone taps (%d) and head levels (%d) differ' % (len(taps), head._num_heads))
    sizes = {}
    for si, stage in enumerate(backbone.stages()):
        h, w = conv_out(h, 3, 2), conv_out(w, 3, 2)
        for bi in range(len(stage)):
            if (si, bi) in taps:
                sizes[(si, bi)] = (h, w)
    level_sizes = [sizes[t] for t in taps]
    offs, acc = [], 0
    for fh, fw in level_sizes:
        offs.append(acc)
        acc += fh * fw
    return level_sizes, acc, offs


def image_channels(model):
    """Channels of the image a model reads: its stem conv's in_channels (3: BGR, 1: gray)."""
    return model._backbone.stem_layers()[0][0].in_channels


def _u8_shape_ok(shape, N, h, w, channels):
    """uint8 frames: [N,h,w,3] for BGR; [N,h,w] or [N,h,w,1] for gray."""
    return shape == (N, h, w, channels) or (channels == 1 and shape == (N, h, w))


def check_input(x, N, H, W, contiguous, channels=3):
    """x: float32 [N,C,H,W] or uint8 [N,H,W,3] (gray, C = 1: [N,H,W] or [N,H,W,1]) on a CUDA device -> its nat.INPUT_* format."""
    if x.dtype == torch.float32:
        fmt, ok = nat.INPUT_F32_NCHW, tuple(x.shape) == (N, channels, H, W)
    elif x.dtype == torch.uint8:
        fmt, ok = nat.INPUT_U8_NHWC, _u8_shape_ok(tuple(x.shape), N, H, W, channels)
    else:
        raise TypeError('input must be float32 NCHW or uint8 NHWC, got %s' % (x.dtype,))
    if not ok or not x.is_cuda or (contiguous and not x.is_contiguous()):
        raise ValueError('input must be a%s CUDA tensor matching the plan shape N=%d H=%d W=%d (got %s)'
                         % (' contiguous' if contiguous else '', N, H, W, tuple(x.shape)))
    return fmt


def check_frame(x, N, H, W, channels=3):
    """x: float32 [N,C,h,w] or uint8 [N,h,w,3] (gray, C = 1: [N,h,w] or [N,h,w,1]), contiguous, on a CUDA device, with h <= H and w <= W
    -> (its nat.INPUT_* format, h, w)."""
    if x.dtype == torch.float32:
        fmt, ok = nat.INPUT_F32_NCHW, x.dim() == 4 and x.shape[1] == channels
        h, w = (x.shape[2], x.shape[3]) if ok else (0, 0)
    elif x.dtype == torch.uint8:
        fmt, ok = nat.INPUT_U8_NHWC, x.dim() >= 3 and _u8_shape_ok(tuple(x.shape), x.shape[0], x.shape[1], x.shape[2], channels)
        h, w = (x.shape[1], x.shape[2]) if ok else (0, 0)
    else:
        raise TypeError('input must be float32 NCHW or uint8 NHWC, got %s' % (x.dtype,))
    if not ok or not x.is_cuda or not x.is_contiguous() or x.shape[0] != N or not (1 <= h <= H and 1 <= w <= W):
        raise ValueError('input must be a contiguous CUDA tensor of N=%d frames of at most H=%d x W=%d (the plan\'s capacity), got %s'
                         % (N, H, W, tuple(x.shape)))
    return fmt, int(h), int(w)


def check_nv12_frame(x, N, H, W):
    """x: NV12 frames, uint8 [N, 3h/2, w] (each image a Y plane of h rows x w bytes, then an interleaved UV plane of h/2 rows x w bytes),
    contiguous, on a CUDA device, h and w even, h <= H and w <= W, on a capacity H x W that is even too -> (h, w)."""
    if H % 2 or W % 2:
        raise ValueError('NV12 frames need a plan of even height and width, this plan\'s capacity is %dx%d' % (H, W))
    if x.dtype != torch.uint8 or x.dim() != 3:
        raise ValueError('NV12 frames are a uint8 [N, 3h/2, w] tensor, got %s %s' % (x.dtype, tuple(x.shape)))
    n, rows, w = (int(s) for s in x.shape)
    if rows % 3 or w % 2:
        raise ValueError('NV12 frames have an even height and width: %d rows x %d columns is not [3h/2, w] of an even h and w' % (rows, w))
    h = rows // 3 * 2
    if n != N or not (1 <= h <= H and 1 <= w <= W):
        raise ValueError('input must be N=%d NV12 frames of at most H=%d x W=%d (the plan\'s capacity), got %d frames of %dx%d' % (N, H, W, n, h, w))
    if not x.is_cuda or not x.is_contiguous():
        raise ValueError('NV12 frames must be a contiguous CUDA tensor')
    return h, w


def check_source(x, N, channels, nv12):
    """x: N source frames of any size for a resized forward -- uint8 [N,h,w,3] (BGR), [N,h,w] or [N,h,w,1] (gray, channels = 1), or with nv12
    NV12 frames uint8 [N,3h/2,w] of even h and w -- contiguous, on a CUDA device -> (its nat.INPUT_* format, h, w).  float32 frames are
    refused: the resize reads uint8."""
    if x.dtype != torch.uint8:
        raise ValueError('resized frames are uint8 (BGR, gray or NV12), got %s' % (x.dtype,))
    if nv12:
        ok = x.dim() == 3 and x.shape[1] % 3 == 0 and x.shape[2] % 2 == 0     # 3h/2 rows of an even h
        fmt, h, w = nat.INPUT_U8_NV12, (int(x.shape[1]) // 3 * 2 if ok else 0), (int(x.shape[2]) if ok else 0)
    else:
        ok = x.dim() >= 3 and _u8_shape_ok(tuple(x.shape), x.shape[0], x.shape[1], x.shape[2], channels)
        fmt, h, w = nat.INPUT_U8_NHWC, (int(x.shape[1]) if ok else 0), (int(x.shape[2]) if ok else 0)
    if not ok or x.shape[0] != N or h < 1 or w < 1 or not x.is_cuda or not x.is_contiguous():
        want = 'NV12 frames uint8 [N, 3h/2, w] of even h and w' if nv12 else ('uint8 [N, h, w, 3]' if channels == 3 else 'uint8 [N, h, w]')
        raise ValueError('resized input must be N=%d contiguous CUDA frames, %s; got %s' % (N, want, tuple(x.shape)))
    return fmt, h, w


# the packed camera-frame formats of InferencePlan.forward / StreamingDetector: name -> (nat.INPUT_* code, bytes per pixel)
PACKED_FORMATS = {'yuy2': (nat.INPUT_U8_YUY2, 2), 'uyvy': (nat.INPUT_U8_UYVY, 2), 'bgra': (nat.INPUT_U8_BGRA, 4), 'rgba': (nat.INPUT_U8_RGBA, 4)}


def check_packed(x, frame_format, N, channels, H=None, W=None):
    """x: packed camera frames (include/lfd_b200.h), contiguous, on a CUDA device -- 'yuy2' / 'uyvy': YUV 4:2:2 uint8 [N,h,w,2] of an
    even w; 'bgra' / 'rgba': uint8 [N,h,w,4] -- for a model that reads `channels` image channels (a gray model takes 4:2:2 only, of
    which it reads the Y bytes); with a capacity H x W, h <= H and w <= W on an even W for 4:2:2 -> (its nat.INPUT_* format, h, w)."""
    fmt, bpp = PACKED_FORMATS[frame_format]
    if channels == 1 and bpp == 4:
        raise ValueError("a gray model reads 4:2:2 frames ('yuy2' / 'uyvy'); %r frames are colour, got frame_format %r" % (frame_format, frame_format))
    if bpp == 2 and W is not None and W % 2:
        raise ValueError('4:2:2 frames need a plan of even width, this plan\'s capacity is %dx%d' % (H, W))
    if x.dtype != torch.uint8 or x.dim() != 4 or x.shape[3] != bpp:
        raise ValueError('%s frames are a uint8 [N, h, w, %d] tensor, got %s %s' % (frame_format.upper(), bpp, x.dtype, tuple(x.shape)))
    n, h, w = (int(v) for v in x.shape[:3])
    if bpp == 2 and w % 2:
        raise ValueError('4:2:2 frames have an even width, got %dx%d' % (h, w))
    if n != N or h < 1 or w < 1 or (H is not None and not (h <= H and w <= W)):
        cap = ' of at most H=%d x W=%d (the plan\'s capacity)' % (H, W) if H is not None else ''
        raise ValueError('input must be N=%d %s frames%s, got %d frames of %dx%d' % (N, frame_format.upper(), cap, n, h, w))
    if not x.is_cuda or not x.is_contiguous():
        raise ValueError('%s frames must be a contiguous CUDA tensor' % (frame_format.upper(),))
    return fmt, h, w


def stage_nv12(stage, x, h, w):
    """Copies NV12 frames x [N, 3h/2, w] into the capacity layout stage [N, 3H/2, W]: the Y rows into the top-left corner of the H x W Y
    plane, the UV rows into the top-left corner of the H/2 x W UV plane."""
    H = stage.shape[1] // 3 * 2
    stage[:, :h, :w].copy_(x[:, :h])
    stage[:, H:H + h // 2, :w].copy_(x[:, h:])


def tune_branch_bounds(work, measure, candidates, budget_s, max_branches=None):
    """Coordinate descent over per-branch bounds on the persistent CTAs of side-branch kernels.  work: {branch: amount of work};
    measure(caps) -> time of the plan with caps = {branch: bound} (0 = unbounded).  The branches with the most work come first (at most
    max_branches of them); each candidate bound is tried on top of the best caps so far and kept only when it is measurably faster
    (below 0.995x the best time).  No trial starts after budget_s seconds.  -> (caps, [(label, time), ...])."""
    t_end = time.time() + budget_s
    caps = {b: 0 for b in work}
    best = measure(caps)
    log = [('all SMs', best)]
    for b in sorted(work, key=lambda k: -work[k])[:max_branches]:
        for c in candidates:
            if time.time() > t_end:
                break
            trial = dict(caps)
            trial[b] = c
            t = measure(trial)
            log.append(('branch %d <= %d CTAs' % (b, c), t))
            if t < best * 0.995:
                best, caps = t, trial
    return caps, log


ACT_DTYPES = {'bf16': (torch.bfloat16, nat.DTYPE_BF16), 'fp16': (torch.float16, nat.DTYPE_FP16)}


def pack_conv_weight(weight, cc, dtype=torch.bfloat16):
    """[Cout, Cin, k, k] float -> 16-bit [Cin/cc][k*k][cc/8][Cout][8], the B-operand order of conv_umma.cu
    (K-major, no-swizzle core matrices; one contiguous slice per channel chunk so that it can be bulk-copied)."""
    cout, cin, k, _ = weight.shape
    wt = weight.detach().float().cpu().permute(2, 3, 1, 0).reshape(k * k, cin // cc, cc // 8, 8, cout)
    return wt.permute(1, 0, 2, 4, 3).contiguous().to(dtype)


def fold_scale(weight, scale):
    """BatchNorm folding: per-output-channel scale multiplied into the fp32 weights (they are rounded to bf16 afterwards)."""
    return weight.detach().float().cpu() * scale.float().reshape(-1, 1, 1, 1)


def pack_stem_weight(weight, dtype=torch.bfloat16):
    """[Cout, Cin, 3, 3] float (Cin = 3, or 1 for a gray image) -> bf16 [kh][2][Cout][8]: element (kh, kc, n, j) is the weight of output n
    for input channel j % 4 and filter column kw = 2*kc + j // 4 (zero for kw = 3 and for channels >= Cin) -- the B operand of the stem
    conv, whose K runs over the 4 pixels x 4 channels that follow a filter row's first input pixel (conv_umma.cu, kStem*)."""
    cout, cin = weight.shape[0], weight.shape[1]
    w = weight.detach().float().cpu()                      # [n, ci, kh, kw]
    full = torch.zeros(3, 4, 4, cout)                      # [kh, pixel, channel, n]
    full[:, :3, :cin, :] = w.permute(2, 3, 1, 0)
    return full.reshape(3, 2, 8, cout).permute(0, 1, 3, 2).contiguous().to(dtype)


_AUX_BRANCH = 7      # graph branch of the residual blocks' shortcut convs (LFD_MAX_BRANCHES - 1)

# model files (include/lfd_b200.h): a pointer field of an op record holds ((blob + 1) << 56) | byte offset, blob 0 = fp32, 1 = 16-bit
MODEL_MAGIC = b'LFDMODEL'
MODEL_FORMAT_VERSION = 1
MODEL_BLOB_F32, MODEL_BLOB_16 = 1 << 56, 2 << 56


class _Arena(object):
    """First-fit allocator with coalescing free list over one workspace (byte offsets, 256 B aligned)."""

    def __init__(self, base=0):
        self.top = base
        self.free = []  # (off, size)

    def alloc(self, size):
        size = (size + 255) & ~255
        best = None
        for i, (o, s) in enumerate(self.free):
            if s >= size and (best is None or s < self.free[best][1]):
                best = i
        if best is not None:
            o, s = self.free.pop(best)
            if s > size:
                self.free.append((o + size, s - size))
            return o
        o = self.top
        self.top += size
        return o

    def release(self, off, size):
        size = (size + 255) & ~255
        self.free.append((off, size))
        self.free.sort()
        merged = []
        for o, s in self.free:
            if merged and merged[-1][0] + merged[-1][1] == o:
                merged[-1] = (merged[-1][0], merged[-1][1] + s)
            else:
                merged.append((o, s))
        self.free = merged


def place_tensors(ops, sizes, arenas, hold=(), skip=()):
    """Liveness placement: a tensor an op writes ('out', 'out2') is allocated in the arena of the op's branch when the op runs and
    released after the last op that reads it ('inp', 'res').  Tensors in `hold` are never released, tensors in `skip` are placed
    elsewhere by the caller.  -> {name: offset inside its arena}"""
    last = {op[k]: i for i, op in enumerate(ops) for k in ('inp', 'res') if op.get(k) is not None and op[k] not in skip}
    placed = {}                                  # name -> (arena, offset)
    for i, op in enumerate(ops):
        arena = arenas[op.get('branch', 0)]
        for k in ('out', 'out2'):
            if op.get(k) is not None and op[k] not in skip:
                placed[op[k]] = (arena, arena.alloc(sizes[op[k]]))
        for name, lu in last.items():
            if lu == i and name not in hold:
                placed[name][0].release(placed[name][1], sizes[name])
    return {name: off for name, (_, off) in placed.items()}


class InferencePlan(object):
    """One native forward plan for a fixed input shape."""

    # the per-level neck + head chains and the unfused residual shortcut convs run on side branches (graph branches / side streams)
    side_branches = True

    def __init__(self, model, N, H, W, device, conv_impl=nat.CONV_UMMA, create_native=True, act_dtype='bf16', fuse_stem=None,
                 input_transform=None, reuse=True):
        """fuse_stem: run a four-conv 'faster' stem as one kernel (LFD_OP_STEM4) -- None: when its stem1 map would not stay in
        L2 (see _use_stem4), True / False: always / never (tests).
        input_transform: what the stem op makes of uint8 frames -- None: simple_normalize on BGR, else an InputTransform
        (lfd/data_pipeline/augmentation.py).  float32 NCHW input is taken as it is.
        reuse: False gives every tensor its own workspace region, so that tensor() can read any intermediate after a forward (tests)."""
        self._configure(N, H, W, device, conv_impl, create_native, act_dtype, fuse_stem)
        self.input_transform = input_transform
        self._build(model)
        self._finalize(reuse)

    def _configure(self, N, H, W, device, conv_impl, create_native, act_dtype, fuse_stem):
        self.N, self.H, self.W = N, H, W
        if act_dtype not in ACT_DTYPES:
            raise ValueError("act_dtype must be 'bf16' or 'fp16' (got %r)" % (act_dtype,))
        self.act_dtype = act_dtype
        self.tdtype, self.dtype_code = ACT_DTYPES[act_dtype]   # 16-bit storage type of activations and packed weights
        self.create_native = create_native   # False: host-side planning only (CPU tests of the planner)
        self.device = device
        self.conv_impl = conv_impl
        self._f32, self._bf16 = [], []      # parameter staging (host tensors, concatenated at the end)
        self._f32_n, self._bf16_n = 0, 0
        self._ops = []                       # dicts; tensors referenced by name
        self._tensors = {}                   # name -> bytes
        self._branch = 0                     # branch id given to the ops being emitted (0 = main stream)
        # conv -> 1x1 conv pairs and 1x1/s2 shortcuts run inside the conv they follow / share their input with (tensor-core kernels
        # only; the SIMT cross-check runs them unfused)
        self.fuse = conv_impl == nat.CONV_UMMA
        self.fuse_stem = fuse_stem
        self.input_transform = None

    # ------------------------------------------------------------------ parameter staging
    def _add_f32(self, t):
        t = t.detach().float().reshape(-1).cpu()
        off = self._f32_n
        self._f32.append(t)
        self._f32_n += (t.numel() + 3) // 4 * 4
        if t.numel() % 4:
            self._f32.append(torch.zeros(4 - t.numel() % 4))
        return off

    def _add_bf16(self, t):
        """16-bit parameter staging (bf16 or fp16 bit patterns, kept as int16 so that one buffer serves both types)."""
        t = t.detach().to(self.tdtype).reshape(-1).cpu().view(torch.int16)
        off = self._bf16_n
        self._bf16.append(t)
        self._bf16_n += (t.numel() + 7) // 8 * 8
        if t.numel() % 8:
            self._bf16.append(torch.zeros(8 - t.numel() % 8, dtype=torch.int16))
        return off

    @staticmethod
    def _fold(conv, norm):
        """-> per-output-channel (scale, shift) fp32 such that y = conv_nobias(x) * scale + shift."""
        cout = conv.out_channels
        bias = conv.bias.detach().float().cpu() if conv.bias is not None else torch.zeros(cout)
        if norm is None:
            return torch.ones(cout), bias
        if not isinstance(norm, BN_TYPES):
            raise NotImplementedError('only BatchNorm2d can be folded into a conv epilogue (got %s)' % type(norm).__name__)
        if norm.training and norm.track_running_stats is False:
            raise NotImplementedError('BatchNorm2d without running statistics is not supported by the inference plan')
        g = norm.weight.detach().float().cpu() if norm.weight is not None else torch.ones(cout)
        b = norm.bias.detach().float().cpu() if norm.bias is not None else torch.zeros(cout)
        scale = g / torch.sqrt(norm.running_var.detach().float().cpu() + norm.eps)
        shift = b - norm.running_mean.detach().float().cpu() * scale + bias * scale
        return scale, shift

    def _tensor(self, name, n, h, w, c):
        self._tensors[name] = n * h * w * c * 2
        return name

    # ------------------------------------------------------------------ op emitters
    def _tail_fields(self, tail, cmid):
        """tail = (conv1x1, norm, relu) fused behind a layer with cmid output channels -> op fields."""
        conv2, norm2, relu2 = tail
        scale2, shift2 = self._fold(conv2, norm2)
        return dict(tail_cout=conv2.out_channels, tail_relu=int(relu2),
                    tail_w=self._add_bf16(pack_conv_weight(fold_scale(conv2.weight, scale2), cmid, self.tdtype)),
                    tail_shift=self._add_f32(shift2), tail_modules=(conv2, norm2))

    @staticmethod
    def _can_fuse_shortcut(block, pairs):
        """The block's 1x1/s2 shortcut conv reads the same tensor as its first conv; when that is a 3x3/s2 conv with the same
        number of output channels (every shipped block) the shortcut's input pixel is the 3x3 conv's centre tap."""
        ds = list(block._downsample)
        c0, sc = pairs[0][0], ds[0]
        return (len(pairs) >= 2 and c0.kernel_size == (3, 3) and c0.stride == (2, 2) and sc.kernel_size == (1, 1) and sc.stride == (2, 2)
                and sc.in_channels == c0.in_channels and sc.out_channels == c0.out_channels and c0.out_channels in (32, 48, 64, 128)
                and sc.groups == 1 and c0.groups == 1)

    @staticmethod
    def _can_tail(conv, nxt):
        """nxt = (conv, norm, relu): a bias-free-or-not 1x1/s1 conv directly consuming `conv`'s output.  A 48-channel conv takes a
        48-channel tail only (the 'fast' stem of TrafficLight LFD-S)."""
        c2 = nxt[0]
        return (c2.kernel_size == (1, 1) and c2.stride == (1, 1) and c2.groups == 1 and c2.in_channels == conv.out_channels
                and ((conv.out_channels in (32, 64) and c2.out_channels in (32, 64, 128)) or (conv.out_channels == 48 and c2.out_channels == 48)))

    def _emit_stem0(self, conv, norm, relu, out_name, h, w, tail=None):
        if conv.in_channels not in (1, 3) or conv.kernel_size != (3, 3) or conv.stride != (2, 2):
            raise NotImplementedError('the H100 stem kernel handles the 3x3/s2 conv on a 3-channel (BGR) or 1-channel (gray) image only')
        ho, wo = conv_out(h, 3, 2), conv_out(w, 3, 2)
        scale, shift = self._fold(conv, norm)
        wt = pack_stem_weight(fold_scale(conv.weight, scale), self.tdtype)
        op = dict(kind=nat.OP_STEM0, H=h, W=w, Cin=conv.in_channels, Ho=ho, Wo=wo, Cout=conv.out_channels, ksize=3, stride=2, relu=int(relu),
                  w_bf16=self._add_bf16(wt), shift=self._add_f32(shift), modules=(conv, norm))
        if tail is not None:
            op.update(self._tail_fields(tail, conv.out_channels))
        op['out'] = self._tensor(out_name, self.N, ho, wo, op.get('tail_cout') or conv.out_channels)
        self._push(op)
        return ho, wo

    def _l2_bytes(self):
        dev = torch.device(self.device)
        if dev.type == 'cuda' and torch.cuda.is_available():
            return torch.cuda.get_device_properties(dev).L2_cache_size
        return 50 << 20          # H100 SXM, as the 132-SM fallback assumes an H100

    def _use_stem4(self, layers):
        """A 'faster' stem (3x3/s2 3->64 or 1->64, 1x1, 3x3/s2 64->64, 1x1, all 64 channels) runs as one kernel when its stem1 map -- the
        tensor the fusion keeps out of HBM -- would not stay in L2 between the two fused pairs (more than half of it).  Smaller
        plans have no HBM round trip to remove and keep the two-kernel path."""
        if not self.fuse or self.fuse_stem is False or len(layers) != 4:
            return False
        (c0, _, _), (c1, _, _), (c2, _, _), (c3, _, _) = layers

        def conv3s2(c, cin):
            return (c.in_channels == cin and c.out_channels == 64 and c.kernel_size == (3, 3) and c.stride == (2, 2)
                    and c.padding == (1, 1) and c.groups == 1 and c.dilation == (1, 1))
        if not (c0.in_channels in (1, 3) and conv3s2(c0, c0.in_channels) and conv3s2(c2, 64) and self._can_tail(c0, layers[1])
                and self._can_tail(c2, layers[3]) and c1.out_channels == 64 and c3.out_channels == 64):
            return False
        if self.fuse_stem:
            return True
        stem1_bytes = self.N * conv_out(self.H, 3, 2) * conv_out(self.W, 3, 2) * 64 * 2
        return stem1_bytes > self._l2_bytes() // 2

    def _emit_stem4(self, layers, out_name, h, w):
        (c0, n0, r0), tail1, (c2, n2, r2), (c3, n3, r3) = layers
        h1, w1 = conv_out(h, 3, 2), conv_out(w, 3, 2)
        ho, wo = conv_out(h1, 3, 2), conv_out(w1, 3, 2)
        s0, b0 = self._fold(c0, n0)
        s2, b2 = self._fold(c2, n2)
        s3, b3 = self._fold(c3, n3)
        op = dict(kind=nat.OP_STEM4, H=h, W=w, Cin=c0.in_channels, Ho=ho, Wo=wo, Cout=64, ksize=3, stride=2, relu=int(r0),
                  w_bf16=self._add_bf16(pack_stem_weight(fold_scale(c0.weight, s0), self.tdtype)), shift=self._add_f32(b0), modules=(c0, n0),
                  s2_w=self._add_bf16(pack_conv_weight(fold_scale(c2.weight, s2), 64, self.tdtype)), s2_shift=self._add_f32(b2), s2_relu=int(r2),
                  s2_modules=(c2, n2),
                  s3_w=self._add_bf16(pack_conv_weight(fold_scale(c3.weight, s3), 64, self.tdtype)), s3_shift=self._add_f32(b3), s3_relu=int(r3),
                  s3_modules=(c3, n3))
        op.update(self._tail_fields(tail1, 64))
        op['out'] = self._tensor(out_name, self.N, ho, wo, 64)
        self._push(op)
        return ho, wo

    def _emit_conv(self, conv, norm, relu, in_name, out_name, h, w, res=None, gn_groups=0, cache=None, tail=None, shortcut=None):
        k, s = conv.kernel_size[0], conv.stride[0]
        if conv.kernel_size[0] != conv.kernel_size[1] or k not in (1, 3) or s not in (1, 2) or conv.padding[0] != k // 2 \
                or conv.groups != 1 or conv.dilation != (1, 1):
            raise NotImplementedError('unsupported conv geometry for the H100 kernels: %r' % (conv,))
        cin, cout = conv.in_channels, conv.out_channels
        ho, wo = conv_out(h, k, s), conv_out(w, k, s)
        q = nat.conv_query(self.N, h, w, cin, ho, wo, cout, k, s, tail[0].out_channels if tail is not None else 0,
                           shortcut[0].out_channels if shortcut is not None else 0)
        cc = q['cc']
        key = (id(conv), id(norm), cc)
        if cache is not None and key in cache:
            w_off, sc_off, sh_off = cache[key]
        else:
            if gn_groups and tail is None:     # (with a fused tail the GroupNorm statistics belong to the TAIL's output)
                if conv.bias is not None:
                    raise NotImplementedError('conv followed by GroupNorm is expected to have no bias')
                scale, shift = torch.ones(cout), torch.zeros(cout)
            else:
                scale, shift = self._fold(conv, norm)
            w_off, sc_off, sh_off = self._add_bf16(pack_conv_weight(fold_scale(conv.weight, scale), cc, self.tdtype)), None, self._add_f32(shift)
            if cache is not None:
                cache[key] = (w_off, sc_off, sh_off)
        op = dict(kind=nat.OP_CONV, H=h, W=w, Cin=cin, Ho=ho, Wo=wo, Cout=cout, ksize=k, stride=s, relu=int(relu),
                  gn_groups=gn_groups, cc=cc, inp=in_name, res=res,
                  w_bf16=w_off, shift=sh_off, query=q, modules=(conv, None if (gn_groups and tail is None) else norm))
        if tail is not None:
            op.update(self._tail_fields(tail, cout))
        if shortcut is not None:      # (conv1x1/s2, norm, output name): same input, computed by the same kernel
            sconv, snorm, sname = shortcut
            sscale, sshift = self._fold(sconv, snorm)
            op.update(ds_cout=sconv.out_channels, ds_w=self._add_bf16(pack_conv_weight(fold_scale(sconv.weight, sscale), cin, self.tdtype)),
                      ds_shift=self._add_f32(sshift), ds_modules=(sconv, snorm),
                      out2=self._tensor(sname, self.N, ho, wo, sconv.out_channels))
        op['out'] = self._tensor(out_name, self.N, ho, wo, op.get('tail_cout') or cout)
        if gn_groups:
            op['stats'] = len([o for o in self._ops if o.get('stats') is not None and o['kind'] == nat.OP_CONV])
        self._push(op)
        return ho, wo

    # ------------------------------------------------------------------ graph walk
    def _emit_stem(self, layers, h, w):
        """The stem on the image -> (name of its output, h, w)."""
        self.in_channels = layers[0][0].in_channels
        cur = None
        i = 0
        if self._use_stem4(layers):
            h, w = self._emit_stem4(layers, 'stem3', h, w)
            cur, i = 'stem3', len(layers)
        while i < len(layers):
            conv, norm, relu = layers[i]
            tail = None
            if self.fuse and i + 1 < len(layers) and self._can_tail(conv, layers[i + 1]):
                tail = layers[i + 1]
            name = 'stem%d' % (i + (1 if tail is not None else 0))      # a fused pair is named after its last layer
            if i == 0:
                h, w = self._emit_stem0(conv, norm, relu, name, h, w, tail=tail)
            else:
                h, w = self._emit_conv(conv, norm, relu, cur, name, h, w, tail=tail)
            cur = name
            i += 2 if tail is not None else 1
        return cur, h, w

    def _emit_block(self, block, base, cur, h, w, n_taps):
        """One residual block on the tensor `cur` -> (name of its output, h, w)."""
        identity = cur
        aux = False
        pairs = block.conv_norm_pairs()
        fuse_sc = None
        if block._downsample is not None and self.fuse and self._can_fuse_shortcut(block, pairs):
            ds = list(block._downsample)
            fuse_sc = (ds[0], ds[1] if len(ds) > 1 else None, base + '_id')
            identity = base + '_id'
        elif block._downsample is not None:
            # the 1x1/s2 shortcut conv only depends on the block input: it runs on the auxiliary branch, next to the
            # block's first conv, and the block's last conv (which adds it) waits for it
            ds = list(block._downsample)
            aux = self.side_branches and n_taps + 1 <= _AUX_BRANCH
            if aux:
                self._branch = _AUX_BRANCH
            self._emit_conv(ds[0], ds[1] if len(ds) > 1 else None, False, cur, base + '_id', h, w)
            if aux:
                self._ops[-1]['wait_mask'] = 1          # the block input comes from the main stream
                self._branch = 0
            identity = base + '_id'
        x, hh, ww = cur, h, w
        for li, (conv, norm) in enumerate(pairs):
            last = li == len(pairs) - 1
            name = base + ('_out' if last else '_c%d' % li)
            hh, ww = self._emit_conv(conv, norm, True, x, name, hh, ww, res=identity if last else None,
                                     shortcut=fuse_sc if li == 0 else None)
            if last and aux:
                self._ops[-1]['wait_mask'] = 1 << _AUX_BRANCH
            x = name
        return x, hh, ww

    def _build(self, model):
        bb, neck, head = model._backbone, model._neck, model._head
        cur, h, w = self._emit_stem(bb.stem_layers(), self.H, self.W)
        self.level_sizes, self.P, offs = level_geometry(bb, head, h, w)
        self.level_offsets = offs
        taps = list(bb._out_indices)
        if make_norm_probe(head) is not None and not isinstance(make_norm_probe(head), nn.GroupNorm):
            raise NotImplementedError('the H100 head kernels implement GroupNorm towers and towers without norm layers (the shipped configs)')
        self.cls_channels = head.num_cls_channels
        cache = {}
        for si, stage in enumerate(bb.stages()):
            for bi, block in enumerate(stage):
                cur, h, w = self._emit_block(block, 's%db%d' % (si, bi), cur, h, w, len(taps))
                if (si, bi) in taps:
                    l = taps.index((si, bi))
                    assert (h, w) == self.level_sizes[l]
                    # the level's neck + head chain only depends on this tap: run it on its own stream / graph branch,
                    # concurrently with the rest of the backbone and with the other levels
                    self._branch = 1 + l if (self.side_branches and 1 + l < 8) else 0
                    self._emit_level(neck, head, l, cur, h, w, offs[l], cache)
                    self._branch = 0

    def _emit_level(self, neck, head, l, fname, fh, fw, point_off, cache):
        conv, norm = neck.level(l)
        nk = 'neck%d' % l
        cls_tower, reg_tower, fin_cls, fin_reg = head.level_paths(l)
        # merged heads: the neck's 1x1 conv (+BN+ReLU) has ONE consumer, the tower's first 1x1 conv -- run the pair as one kernel (the
        # 128-channel neck output never reaches HBM; the GroupNorm statistics are taken on the fused kernel's output as usual)
        t0 = cls_tower[0] if len(cls_tower) else None
        fuse_neck = (self.fuse and cls_tower is reg_tower and t0 is not None
                     and conv.kernel_size == (1, 1) and conv.stride == (1, 1) and conv.groups == 1 and conv.out_channels == 128
                     and t0[0].kernel_size == (1, 1) and t0[0].stride == (1, 1) and t0[0].groups == 1 and t0[0].bias is None
                     and t0[0].in_channels == 128 and t0[0].out_channels == 128
                     and isinstance(t0[1], nn.GroupNorm) and t0[1].num_channels == t0[1].num_groups * 8)
        if not fuse_neck:
            self._emit_conv(conv, norm, True, fname, nk, fh, fw)
        scale_l = float(head._scales[l]._scale.detach()) if head.uses_scale else 1.0

        def run_tower(tower, tag):
            """-> (last stored tensor, GN statistics slot or None, GN module or None).  With GroupNorm the last conv's normalisation + ReLU is
            applied inside HEAD_FINAL; without norm layers (TrafficLight configs, lfd_head.py:47-49 norm_cfg=None) every tower conv is a plain
            conv + bias + ReLU layer and HEAD_FINAL reads the activated tensor."""
            x = nk
            for ti, (tconv, tnorm) in enumerate(tower):
                if tconv.kernel_size not in ((1, 1), (3, 3)) or tconv.stride != (1, 1):
                    raise NotImplementedError('head towers use 1x1 or 3x3 stride-1 convs (lfd_head.py:47-49)')
                if tnorm is None:
                    act = 'h%d%s_act%d' % (l, tag, ti)
                    self._emit_conv(tconv, None, True, x, act, fh, fw, cache=cache)
                    x = act
                    if ti == len(tower) - 1:
                        return act, None, None
                    continue
                if not isinstance(tnorm, nn.GroupNorm) or tnorm.num_channels != tnorm.num_groups * 8:
                    raise NotImplementedError('head towers need GroupNorm with 8 channels per group (or no norm at all)')
                raw = 'h%d%s_raw%d' % (l, tag, ti)
                if ti == 0 and fuse_neck:
                    self._emit_conv(conv, norm, True, fname, raw, fh, fw, gn_groups=tnorm.num_groups, tail=(tconv, None, False))
                else:
                    self._emit_conv(tconv, None, False, x, raw, fh, fw, gn_groups=tnorm.num_groups, cache=cache)
                stats_id = self._ops[-1]['stats']
                if ti == len(tower) - 1:
                    return raw, stats_id, tnorm
                act = 'h%d%s_act%d' % (l, tag, ti)
                self._push(dict(kind=nat.OP_GN_APPLY, H=fh, W=fw, Cin=tconv.out_channels, Ho=fh, Wo=fw,
                                Cout=tconv.out_channels, gn_groups=tnorm.num_groups, inp=raw,
                                out=self._tensor(act, self.N, fh, fw, tconv.out_channels), stats=stats_id,
                                gamma=self._cached_f32(cache, ('g', id(tnorm)), tnorm.weight),
                                beta=self._cached_f32(cache, ('b', id(tnorm)), tnorm.bias), modules=(tnorm,)))
                x = act
            raise ValueError('head tower without conv layers is not supported')

        def final(raw, stats_id, tnorm, convs, n_cls, n_reg):
            ws, scs, shs = [], [], []
            for (fc, sc) in convs:
                ws.append(fc.weight.detach().float().cpu().reshape(fc.out_channels, -1).to(self.tdtype).float())
                b = fc.bias.detach().float().cpu() if fc.bias is not None else torch.zeros(fc.out_channels)
                scs.append(torch.full((fc.out_channels,), sc))
                shs.append(b * sc)
            op = dict(kind=nat.OP_HEAD_FINAL, H=fh, W=fw, Cin=ws[0].shape[1], Ho=fh, Wo=fw, Cout=n_cls + n_reg,
                      gn_groups=tnorm.num_groups if tnorm is not None else 0, inp=raw, stats=stats_id, n_cls=n_cls, n_reg=n_reg,
                      point_off=point_off, level=l, w_f32=self._add_f32(torch.cat(ws, 0)),
                      scale=self._add_f32(torch.cat(scs)), shift=self._add_f32(torch.cat(shs)),
                      modules=(tnorm, [c for c, _ in convs], [sc for _, sc in convs]))
            if tnorm is not None:
                op.update(gamma=self._cached_f32(cache, ('g', id(tnorm)), tnorm.weight), beta=self._cached_f32(cache, ('b', id(tnorm)), tnorm.bias))
            self._push(op)

        if cls_tower is reg_tower:
            raw, sid, tn = run_tower(cls_tower, 'm')
            final(raw, sid, tn, [(fin_cls, 1.0), (fin_reg, scale_l)], fin_cls.out_channels, 4)
        else:
            raw, sid, tn = run_tower(cls_tower, 'c')
            final(raw, sid, tn, [(fin_cls, 1.0)], fin_cls.out_channels, 0)
            raw, sid, tn = run_tower(reg_tower, 'r')
            final(raw, sid, tn, [(fin_reg, scale_l)], 0, 4)

    def _push(self, op):
        op['branch'] = self._branch
        self._ops.append(op)

    def _cached_f32(self, cache, key, t):
        if key not in cache:
            cache[key] = self._add_f32(t)
        return cache[key]

    # ------------------------------------------------------------------ memory plan + native plan
    def _finalize(self, reuse):
        dev = self.device
        self.params_f32 = torch.cat(self._f32).to(dev) if self._f32 else torch.zeros(4, device=dev)
        self.params_bf16 = torch.cat(self._bf16).to(dev) if self._bf16 else torch.zeros(8, dtype=torch.int16, device=dev)
        self._f32, self._bf16 = None, None
        n_stats = len([o for o in self._ops if o['kind'] == nat.OP_CONV and o.get('gn_groups')])
        stats_each = self.N * 16 * 2 * 8
        self.stats_bytes = (n_stats * stats_each + 255) & ~255
        producer = {op['out']: op['branch'] for op in self._ops if op.get('out') is not None}
        producer.update({op['out2']: op['branch'] for op in self._ops if op.get('out2') is not None})
        # a tensor read by another branch (a backbone tap) lives for the whole forward
        shared = {op[k] for op in self._ops for k in ('inp', 'res') if op.get(k) is not None and producer[op[k]] != op['branch']}
        arenas = [_Arena() for _ in range(1 + max(op['branch'] for op in self._ops))]
        local = place_tensors(self._ops, self._tensors, arenas, hold=shared if reuse else set(self._tensors))
        bases, top = [], self.stats_bytes
        for a in arenas:
            bases.append(top)
            top += (a.top + 255) & ~255
        offsets = {name: bases[producer[name]] + off for name, off in local.items()}
        self.workspace_bytes = max(top, 256)
        self.tensor_branch = {name: producer[name] for name in local}
        self.shared_tensors = shared
        self.workspace = torch.empty(self.workspace_bytes, dtype=torch.uint8, device=dev)
        self.activation_bytes = sum(self._tensors.values())
        fb, bb = self.params_f32.data_ptr(), self.params_bf16.data_ptr()
        arr = (nat.Op * len(self._ops))()
        for i, op in enumerate(self._ops):
            self._fill_op(arr[i], op, offsets, fb, bb, stats_each)
        self._op_array = arr
        self.cls_out = torch.empty((self.N, self.P, self.cls_channels), dtype=torch.float32, device=dev)
        self.reg_out = torch.empty((self.N, self.P, 4), dtype=torch.float32, device=dev)
        self._outputs = [(self.cls_out, self.reg_out)]      # slot 1 (second output pair) is allocated on first use
        self.offsets = offsets
        self.frame_level_sizes, self.frame_P = self.level_sizes, self.P   # of the last forward's frame
        self._extents = {}                  # (h, w) -> (lfd_extent table, level sizes, P) of a frame below the capacity
        self._stage = None                  # frames below the capacity are copied into its top-left corner (allocated on first use)
        self.handle = None
        if not self.create_native:
            return
        self.handle = self._create_handle()
        self.num_launches = nat.lib().lfd_plan_num_launches(self.handle)
        self.side_ctas, self.autotuned = {}, False     # branch -> bound on the persistent CTAs of its convs (autotune)

    def _fill_op(self, o, op, offsets, fb, bb, stats_each=0):
        """op dict -> nat.Op: tensor names through `offsets`, staged parameters relative to the fp32 / 16-bit buffers at fb / bb."""
        o.kind = op['kind']
        o.dtype = self.dtype_code
        o.N, o.H, o.W, o.Cin, o.Ho, o.Wo, o.Cout = self.N, op['H'], op['W'], op['Cin'], op['Ho'], op['Wo'], op['Cout']
        o.ksize, o.stride, o.relu = op.get('ksize', 1), op.get('stride', 1), op.get('relu', 0)
        o.gn_groups = op.get('gn_groups', 0)
        o.n_cls, o.n_reg, o.point_off, o.cc = op.get('n_cls', 0), op.get('n_reg', 0), op.get('point_off', 0), op.get('cc', 0)
        o.branch = op.get('branch', 0)
        o.wait_mask = op.get('wait_mask', 0)
        o.max_ctas = op.get('max_ctas', 0)
        o.tail_cout, o.tail_relu = op.get('tail_cout', 0), op.get('tail_relu', 0)
        if op.get('tail_cout'):
            o.tail_weight = bb + 2 * op['tail_w']
            o.tail_shift = fb + 4 * op['tail_shift']
        o.ds_cout, o.ds_out_off = op.get('ds_cout', 0), -1
        if op.get('ds_cout'):
            o.ds_weight = bb + 2 * op['ds_w']
            o.ds_shift = fb + 4 * op['ds_shift']
            o.ds_out_off = offsets[op['out2']]
        if op['kind'] in (nat.OP_STEM0, nat.OP_STEM4):
            nat.set_input_transform(o, self.input_transform)
        if op['kind'] == nat.OP_STEM4:
            o.s2_weight, o.s2_shift, o.s2_relu = bb + 2 * op['s2_w'], fb + 4 * op['s2_shift'], op['s2_relu']
            o.s3_weight, o.s3_shift, o.s3_relu = bb + 2 * op['s3_w'], fb + 4 * op['s3_shift'], op['s3_relu']
        o.in_off = offsets[op['inp']] if op.get('inp') is not None else -1
        o.out_off = offsets[op['out']] if op.get('out') is not None else -1
        o.res_off = offsets[op['res']] if op.get('res') is not None else -1
        o.stats_off = op['stats'] * stats_each if op.get('stats') is not None else -1
        if 'w_bf16' in op:
            o.weight = bb + 2 * op['w_bf16']
        elif 'w_f32' in op:
            o.weight = fb + 4 * op['w_f32']
        o.scale = fb + 4 * op['scale'] if 'scale' in op else None
        o.shift = fb + 4 * op['shift'] if 'shift' in op else None
        o.gamma = fb + 4 * op['gamma'] if 'gamma' in op else None
        o.beta = fb + 4 * op['beta'] if 'beta' in op else None

    def _create_handle(self):
        handle = C.c_void_p()
        with torch.cuda.device(self.device):
            nat.check(nat.lib().lfd_plan_create(self._op_array, len(self._ops), self.N, self.P, self.cls_channels, 0, self.stats_bytes,
                                                self.workspace_bytes, self.conv_impl, C.byref(handle)))
        return handle

    def _set_side_ctas(self, caps):
        for o, op in zip(self._op_array, self._ops):
            if op.get('branch', 0) > 0:      # convs: persistent CTAs; GN_APPLY / HEAD_FINAL: the SM count their grids are sized from
                o.max_ctas = int(caps.get(op['branch'], 0))

    def autotune(self, candidates=(96, 64, 48, 32), budget_s=3.0, x=None):
        """Pick, by timing the replayed CUDA graph on this device, how many persistent CTAs the convs of every side branch (the
        per-level neck + head chains) may use.  The chains of the large levels run next to the backbone's small, latency-bound deeper
        stages (the critical path of the step); when their persistent CTAs hold all SMs, every small layer queues behind a whole
        side-branch layer.  Coordinate descent over the branches (largest first), keeping a bound only when it is measurably faster.
        Results do not depend on the bound (tiles are independent).  Returns {branch: bound} (0 = unbounded)."""
        if self.handle is None:
            raise nat.LfdError('this plan was built for host-side inspection only (create_native=False)')
        if x is None:
            x = torch.zeros(self.u8_shape(self.H, self.W), dtype=torch.uint8, device=self.device)
        lib = nat.lib()

        def measure(caps):
            self._set_side_ctas(caps)
            h = self._create_handle()
            try:
                saved, self.handle = self.handle, h
                with torch.cuda.device(self.device):
                    self.forward(x, use_graph=True)          # eager pass + capture
                    self.forward(x, use_graph=True)
                    torch.cuda.synchronize(self.device)
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    self.forward(x, use_graph=True)
                    e1.record()
                    torch.cuda.synchronize(self.device)
                    reps = int(max(3, min(40, 0.01 / max(e0.elapsed_time(e1) * 1e-3, 1e-6))))
                    best = []
                    for _ in range(3):
                        e0.record()
                        for _ in range(reps):
                            self.forward(x, use_graph=True)
                        e1.record()
                        torch.cuda.synchronize(self.device)
                        best.append(e0.elapsed_time(e1) / reps)
                return sorted(best)[1]
            finally:
                self.handle = saved
                lib.lfd_plan_destroy(h)

        work = {}
        for op in self._ops:
            if op['kind'] == nat.OP_CONV and op.get('branch', 0) > 0:
                work[op['branch']] = work.get(op['branch'], 0) + self.N * op['Ho'] * op['Wo'] * (op['Cin'] + op['Cout'])
        caps, log = tune_branch_bounds(work, measure, candidates, budget_s)
        self.apply_side_ctas(caps)
        self.autotune_log = log
        return caps

    def apply_side_ctas(self, caps):
        """Re-creates the native plan with the given {branch: CTA bound} (e.g. the result of another plan's autotune for the same shape)."""
        self._set_side_ctas(caps)
        old = self.handle
        self.handle = self._create_handle()
        nat.lib().lfd_plan_destroy(old)
        self.side_ctas, self.autotuned = dict(caps), True

    def outputs(self, slot):
        while len(self._outputs) <= slot:
            self._outputs.append((torch.empty_like(self.cls_out), torch.empty_like(self.reg_out)))
        return self._outputs[slot]

    def extent_table(self, h, w):
        """The geometry of an h x w frame on this plan -> (rows, level sizes, P): per op [H, W, Ho, Wo, point_off, P], the fields a plan built
        for h x w has (point_off and P on HEAD_FINAL ops only, 0 elsewhere).  Every tensor's valid size follows from the frame through the
        op list, exactly as _build derives the sizes of a plan."""
        size, rows = {}, []
        for op in self._ops:
            H, W = (h, w) if op['kind'] in (nat.OP_STEM0, nat.OP_STEM4) else size[op['inp']]
            if op['kind'] in (nat.OP_STEM0, nat.OP_CONV):
                Ho, Wo = conv_out(H, op['ksize'], op['stride']), conv_out(W, op['ksize'], op['stride'])
            elif op['kind'] == nat.OP_STEM4:
                Ho, Wo = conv_out(conv_out(H, 3, 2), 3, 2), conv_out(conv_out(W, 3, 2), 3, 2)
            else:
                Ho, Wo = H, W
            for k in ('out', 'out2'):
                if op.get(k) is not None:
                    size[op[k]] = (Ho, Wo)
            rows.append([H, W, Ho, Wo, 0, 0])
        level_sizes = [None] * len(self.level_sizes)
        for op, r in zip(self._ops, rows):
            if op['kind'] == nat.OP_HEAD_FINAL:
                level_sizes[op['level']] = (r[0], r[1])
        offs, P = [], 0
        for fh, fw in level_sizes:
            offs.append(P)
            P += fh * fw
        for op, r in zip(self._ops, rows):
            if op['kind'] == nat.OP_HEAD_FINAL:
                r[4], r[5] = offs[op['level']], P
        return rows, level_sizes, P

    def _extent(self, h, w):
        if (h, w) not in self._extents:
            rows, level_sizes, P = self.extent_table(h, w)
            arr = (nat.Extent * len(rows))()
            for e, r in zip(arr, rows):
                e.H, e.W, e.Ho, e.Wo, e.point_off, e.P = r
            self._extents[(h, w)] = (arr, level_sizes, P)
        return self._extents[(h, w)]

    def staging(self, fmt):
        """The plan-owned input of frames below the capacity, in the capacity layout of format fmt (uint8 [N,H,W,3], float32 [N,3,H,W],
        NV12 uint8 [N,3H/2,W], 4:2:2 uint8 [N,H,W,2] or BGRA / RGBA uint8 [N,H,W,4]; a gray plan: uint8 [N,H,W], float32 [N,1,H,W] or the
        same NV12 and 4:2:2 layouts)."""
        c = self.in_channels
        if self._stage is None:
            self._stage = torch.empty(self.N * 3 * self.H * self.W * 4, dtype=torch.uint8, device=self.device)
        if fmt == nat.INPUT_U8_NHWC:
            return self._stage[:self.N * self.H * self.W * c].view(self.u8_shape(self.H, self.W))
        if fmt == nat.INPUT_U8_NV12:
            return self._stage[:self.N * self.H * self.W * 3 // 2].view(self.N, self.H * 3 // 2, self.W)
        for code, bpp in PACKED_FORMATS.values():
            if fmt == code:
                return self._stage[:self.N * self.H * self.W * bpp].view(self.N, self.H, self.W, bpp)
        return self._stage.view(torch.float32)[:self.N * c * self.H * self.W].view(self.N, c, self.H, self.W)

    def u8_shape(self, h, w):
        """The shape of N uint8 frames of h x w on this plan: [N,h,w,3] (BGR) or [N,h,w] (gray)."""
        return (self.N, h, w, 3) if self.in_channels == 3 else (self.N, h, w)

    def num_graphs(self):
        return nat.lib().lfd_plan_num_graphs(self.handle)

    def forward(self, x, use_graph=True, slot=0, frame_format=None, resize_scale=None):
        """x: cuda float32 [N,3,h,w] (contiguous) or uint8 [N,h,w,3] with h <= H and w <= W; with frame_format='nv12', NV12 video frames
        uint8 [N,3h/2,w] of even h and w (include/lfd_b200.h, LFD_INPUT_U8_NV12), which give bit for bit what the uint8 path gives on
        cv2.cvtColor(frame, cv2.COLOR_YUV2BGR_NV12).  A gray plan (in_channels 1) takes float32 [N,1,h,w] or uint8 [N,h,w] / [N,h,w,1], and
        reads only the Y plane of NV12 frames: the uint8 path on cv2.cvtColor(frame, cv2.COLOR_YUV2GRAY_NV12).  Returns the frame's (cls, reg) in the
        plan-owned buffers of output `slot` (a second slot lets the post-process of one batch overlap the forward of the next,
        lfd/pipeline.py): (N, P, C') and (N, P, 4) for the frame's P points, laid out as a plan built for h x w lays them out;
        frame_level_sizes / frame_P describe them.  A frame of the full size is read in place; a smaller one is first copied into the
        top-left corner of a plan-owned input, so that every frame size replays the same CUDA graph (one per input format).
        resize_scale=s: x holds N uint8 frames of any size h x w (above the capacity too; BGR [N,h,w,3], gray [N,h,w], or NV12 with
        frame_format='nv12'), resized on the device into the plan-owned input exactly as cv2.resize(frame, (0, 0), fx=s, fy=s) resizes them
        (lfd_resize_frames; NV12 as cv2.resize of the converted frame), and the forward runs at the resized size (nat.resize_query), which
        must fit the capacity.
        frame_format='yuy2' / 'uyvy' (YUV 4:2:2 uint8 [N,h,w,2], w even) or 'bgra' / 'rgba' (uint8 [N,h,w,4], the alpha byte never read):
        packed camera frames, read by the stem kernels (and by the resize, with resize_scale) as the uint8 BGR path reads
        cv2.cvtColor(frame, cv2.COLOR_{YUY2,UYVY,BGRA,RGBA}2BGR), bit for bit.  A gray plan takes 4:2:2 frames, of which it reads the Y
        bytes (cv2.COLOR_YUV2GRAY_YUY2 / _UYVY), and raises ValueError for 'bgra' / 'rgba'."""
        if self.handle is None:
            raise nat.LfdError('this plan was built for host-side inspection only (create_native=False)')
        if frame_format not in (None, 'nv12') and frame_format not in PACKED_FORMATS:
            raise ValueError("frame_format must be None (float32 NCHW or uint8 BGR, by dtype) or 'nv12', got %r (packed camera frames: 'yuy2', "
                             "'uyvy', 'bgra', 'rgba')" % (frame_format,))
        if resize_scale is not None:
            return self._forward_resized(x, use_graph, slot, frame_format, float(resize_scale))
        if frame_format is None:
            fmt, h, w = check_frame(x, self.N, self.H, self.W, self.in_channels)
            if fmt == nat.INPUT_U8_NHWC and self.in_channels == 1:
                x = x.view(self.N, h, w)
        elif frame_format == 'nv12':
            fmt, (h, w) = nat.INPUT_U8_NV12, check_nv12_frame(x, self.N, self.H, self.W)
        else:
            fmt, h, w = check_packed(x, frame_format, self.N, self.in_channels, self.H, self.W)
        cls_out, reg_out = self.outputs(slot)
        lib = nat.lib()
        if (h, w) == (self.H, self.W):
            with torch.cuda.device(self.device):
                nat.check(lib.lfd_plan_forward(self.handle, nat.ptr(x), fmt, nat.ptr(self.workspace), nat.ptr(cls_out),
                                               nat.ptr(reg_out), int(bool(use_graph)), nat.stream_ptr()))
            self.frame_level_sizes, self.frame_P = self.level_sizes, self.P
            return cls_out, reg_out
        if self.conv_impl != nat.CONV_UMMA:
            raise nat.LfdError('the SIMT cross-check plan runs frames of its full size %dx%d only (got %dx%d)' % (self.H, self.W, h, w))
        table, level_sizes, P = self._extent(h, w)
        with torch.cuda.device(self.device):
            stage = self.staging(fmt)
            if fmt == nat.INPUT_U8_NV12:
                stage_nv12(stage, x, h, w)
            elif fmt == nat.INPUT_F32_NCHW:
                stage[:, :, :h, :w].copy_(x)
            else:
                stage[:, :h, :w].copy_(x)
            nat.check(lib.lfd_plan_forward_extent(self.handle, nat.ptr(stage), fmt, h, w, table, nat.ptr(self.workspace), nat.ptr(cls_out),
                                                  nat.ptr(reg_out), int(bool(use_graph)), nat.stream_ptr()))
        return self._frame_outputs(cls_out, reg_out, level_sizes, P)

    def _frame_outputs(self, cls_out, reg_out, level_sizes, P):
        self.frame_level_sizes, self.frame_P = level_sizes, P
        n, c = self.N, self.cls_channels
        return cls_out.view(-1)[:n * P * c].view(n, P, c), reg_out.view(-1)[:n * P * 4].view(n, P, 4)

    def _forward_resized(self, x, use_graph, slot, frame_format, s):
        """forward(x, resize_scale=s): the resize into the uint8 staging input, then the forward at the resized extent on that input (one
        CUDA graph for the capacity, one for every size below it, as for frames staged by copy)."""
        if self.conv_impl != nat.CONV_UMMA:
            raise nat.LfdError('the SIMT cross-check plan does not take resized frames')
        if frame_format in PACKED_FORMATS:
            fmt, h, w = check_packed(x, frame_format, self.N, self.in_channels)
        else:
            fmt, h, w = check_source(x, self.N, self.in_channels, frame_format == 'nv12')
        _, dh, dw = nat.resize_query(h, w, s)
        if dh > self.H or dw > self.W:
            raise ValueError('%dx%d frames at resize scale %r are %dx%d, beyond the plan\'s capacity %dx%d' % (h, w, s, dh, dw, self.H, self.W))
        cls_out, reg_out = self.outputs(slot)
        lib = nat.lib()
        with torch.cuda.device(self.device):
            stage = self.staging(nat.INPUT_U8_NHWC)
            st = nat.stream_ptr()
            nat.check(lib.lfd_resize_frames(nat.ptr(x), fmt, self.in_channels, self.N, h, w, s, nat.ptr(stage), self.H, self.W, st))
            if (dh, dw) == (self.H, self.W):
                nat.check(lib.lfd_plan_forward(self.handle, nat.ptr(stage), nat.INPUT_U8_NHWC, nat.ptr(self.workspace), nat.ptr(cls_out),
                                               nat.ptr(reg_out), int(bool(use_graph)), st))
                return self._frame_outputs(cls_out, reg_out, self.level_sizes, self.P)
            table, level_sizes, P = self._extent(dh, dw)
            nat.check(lib.lfd_plan_forward_extent(self.handle, nat.ptr(stage), nat.INPUT_U8_NHWC, dh, dw, table, nat.ptr(self.workspace),
                                                  nat.ptr(cls_out), nat.ptr(reg_out), int(bool(use_graph)), st))
        return self._frame_outputs(cls_out, reg_out, level_sizes, P)

    def tensor(self, name):
        """Debug view of an intermediate activation as NHWC bf16 / fp16 (valid right after an eager forward only if
        its buffer has not been reused by a later layer)."""
        op = [o for o in self._ops if name in (o.get('out'), o.get('out2'))][0]
        c = op['ds_cout'] if op.get('out2') == name else (op.get('tail_cout') or op['Cout'])
        n = self.N * op['Ho'] * op['Wo'] * c
        raw = self.workspace[self.offsets[name]: self.offsets[name] + 2 * n]
        return raw.view(self.tdtype).view(self.N, op['Ho'], op['Wo'], c)

    def describe(self):
        """One row per launch.  The fused four-conv stem is reported as a 'stem0' row from the image to the stem3 map with
        fused_stem=4: its bytes are then exactly the kernel's (image in, stem3 out, weights), its flops count stem0 at the
        stem3 resolution + one 1x1 conv only (tests/debug_stem_fusion.py has the true count)."""
        names = {nat.OP_STEM0: 'stem0', nat.OP_CONV: 'conv', nat.OP_GN_APPLY: 'gn_apply', nat.OP_HEAD_FINAL: 'head_final', nat.OP_STEM4: 'stem0'}
        rows = []
        for op in self._ops:
            rows.append(dict(kind=names[op['kind']], H=op['H'], W=op['W'], Cin=op['Cin'], Ho=op['Ho'], Wo=op['Wo'], Cout=op['Cout'],
                             ksize=op.get('ksize', 1), stride=op.get('stride', 1), res=op.get('res') is not None, tail_cout=op.get('tail_cout', 0), ds_cout=op.get('ds_cout', 0),
                             out=op.get('out'), query=op.get('query'), fused_stem=4 if op['kind'] == nat.OP_STEM4 else 0))
        return rows

    def export(self, path, post):
        """Writes this plan and the post-process `post` (a PostPlan for N images of this plan's level geometry) to the model file `path`
        (include/lfd_b200.h "model files", DESIGN.md "Model files"), which lfd_engine_open reads without Python or torch.  The ops are
        the records this plan hands to lfd_plan_create, with the current CTA bounds (autotune), their pointers as (blob, offset) into the
        two staging buffers.  The same plan gives the same bytes.  -> the file's size."""
        data = self.model_file_bytes(post)
        with open(path, 'wb') as f:
            f.write(data)
        return len(data)

    def model_file_bytes(self, post):
        """The bytes export writes."""
        if self.conv_impl != nat.CONV_UMMA:
            raise ValueError('model files hold wgmma plans (conv_impl=CONV_UMMA), not the SIMT cross-check')
        c = post.cfg
        if (c.N, c.P, c.cls_channels, c.num_levels) != (self.N, self.P, self.cls_channels, len(self.level_sizes)) or \
                [(c.level_off[l], c.level_w[l]) for l in range(c.num_levels)] != [(self.level_offsets[l], s[1]) for l, s in enumerate(self.level_sizes)]:
            raise ValueError('the post-process was not made for this plan (N, P, cls_channels or level geometry differ)')
        producer = {}
        records, aux = [], []
        for i, op in enumerate(self._ops):
            o = nat.Op()
            self._fill_op(o, op, self.offsets, MODEL_BLOB_F32, MODEL_BLOB_16, self.N * 16 * 2 * 8)
            o.max_ctas = self._op_array[i].max_ctas         # the autotuned CTA bounds live in the op array
            records.append(C.string_at(C.addressof(o), C.sizeof(o)))
            aux.append(struct.pack('<ii', producer[op['inp']] if op.get('inp') is not None else -1,
                                   op['level'] if op['kind'] == nat.OP_HEAD_FINAL else -1))
            for k in ('out', 'out2'):
                if op.get(k) is not None:
                    producer[op[k]] = i
        blob_f32 = self.params_f32.detach().cpu().contiguous().numpy().tobytes()
        blob_16 = self.params_bf16.detach().cpu().contiguous().numpy().tobytes()
        xf = self.input_transform
        swap, mean, scale = (0, (0.0,) * 3, (0.0,) * 3) if xf is None else (int(xf.swap_rb), tuple(xf.mean), tuple(xf.scale))
        soft = (1,) + tuple(post.soft) if post.soft is not None else (0, 0, 0.0, 0.0)
        plan = struct.pack('<8i3qi3f3f2i2fi2q', self.N, self.H, self.W, self.P, self.cls_channels, self.dtype_code, self.conv_impl, len(records),
                           0, self.stats_bytes, self.workspace_bytes, swap, *mean, *scale, *soft, 0, len(blob_f32), len(blob_16))
        payload = b''.join([plan, C.string_at(C.addressof(c), C.sizeof(c))] + records + aux + [blob_f32, blob_16])
        header = MODEL_MAGIC + struct.pack('<II8sIIQII', MODEL_FORMAT_VERSION, nat.ABI_VERSION, b'sm_90a', C.sizeof(nat.Op), C.sizeof(nat.PostCfg),
                                           len(payload), zlib.crc32(payload), 0)
        return header + payload

    def __del__(self):
        try:
            if getattr(self, 'handle', None):
                nat.lib().lfd_plan_destroy(self.handle)
                self.handle = None
        except Exception:
            pass


class PrefixEmitter(InferencePlan):
    """The inference plan's stem and residual-block emitters, for a training plan's frozen backbone prefix (lfd/_train.py): the same
    BatchNorm folding, weight packing and fusion decisions (STEM4 gate, fused tails and shortcuts), bf16, every op on the main stream.
    The training plan places the ops in its own workspace and runs them as LFD_TOP_INFER ops."""

    side_branches = False

    def __init__(self, N, H, W, device, input_transform=None):
        self._configure(N, H, W, device, nat.CONV_UMMA, False, 'bf16', None)
        self.input_transform = input_transform

    def staged(self):
        """-> (fp32, int16) host tensors of the folded / packed parameters the ops' offsets point into."""
        f32 = torch.cat(self._f32) if self._f32 else torch.zeros(4)
        b16 = torch.cat(self._bf16) if self._bf16 else torch.zeros(8, dtype=torch.int16)
        return f32, b16


def make_norm_probe(head):
    """First norm module of the head tower (None when the head has no norm)."""
    tower = head.level_paths(0)[0]
    return tower[0][1] if tower else None


class PostPlan(object):
    """Pre-allocated device post-process (lfd_postprocess, or lfd_postprocess_soft_nms when soft = (method code, sigma, min_score)) for a
    fixed batch size / level geometry."""

    def __init__(self, cfg, device, soft=None):
        self.cfg, self.device, self.soft = cfg, device, soft
        N, cap = cfg.N, cfg.cap
        self.ws = torch.empty(max(nat.lib().lfd_postprocess_workspace_bytes(C.byref(cfg)), 256), dtype=torch.uint8, device=device)
        self.dets = torch.empty((N, cap, 5), dtype=torch.float32, device=device)
        self.labels = torch.empty((N, cap), dtype=torch.int32, device=device)
        self.src = torch.empty((N, cap), dtype=torch.int32, device=device)
        self.count = torch.empty((N + 1,), dtype=torch.int32, device=device)   # [N] = overflow flag
        self.meta = torch.zeros((3, N), dtype=torch.float32, device=device)   # widths, heights, resize scales
        self._meta_host = None

    def set_meta(self, widths, heights, scales):
        host = (tuple(map(float, widths)), tuple(map(float, heights)), tuple(map(float, scales)))
        if host != self._meta_host:
            self.meta.copy_(torch.tensor(host, dtype=torch.float32))
            self._meta_host = host

    def run(self, cls, reg, score_thr=None, iou_thr=None):
        """cls/reg: contiguous float32 CUDA tensors.  Results stay on the device (dets, labels, src, count[+overflow])."""
        if score_thr is not None:
            self.cfg.score_thr = float(score_thr)
        if iou_thr is not None:
            self.cfg.iou_thr = float(iou_thr)
        with torch.cuda.device(self.device):
            args = (C.byref(self.cfg), nat.ptr(cls), nat.ptr(reg), nat.ptr(self.meta[0]), nat.ptr(self.meta[1]), nat.ptr(self.meta[2]),
                    nat.ptr(self.ws), nat.ptr(self.dets), nat.ptr(self.labels), nat.ptr(self.src), nat.ptr(self.count),
                    nat.ptr(self.count[self.cfg.N:]))
            if self.soft is None:
                nat.check(nat.lib().lfd_postprocess(*args, nat.stream_ptr()))
            else:
                method, sigma, min_score = self.soft
                nat.check(nat.lib().lfd_postprocess_soft_nms(*args, int(method), float(sigma), float(min_score), nat.stream_ptr()))
        return self.dets, self.labels, self.src, self.count
