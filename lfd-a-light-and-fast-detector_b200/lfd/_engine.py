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
import os

import torch
import torch.nn as nn

from . import _native as nat

BN_TYPES = (nn.BatchNorm2d,)


def _conv_out(size, k, s):
    return (size + 2 * (k // 2) - k) // s + 1


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
    """[Cout, 3, 3, 3] float -> bf16 [kh][2][Cout][8]: element (kh, kc, n, j) is the weight of output n for input channel
    j % 4 and filter column kw = 2*kc + j // 4 (zero for kw = 3 and for the padded 4th channel) -- the B operand of the stem
    conv, whose K runs over the 4 pixels x 4 channels that follow a filter row's first input pixel (conv_umma.cu, kStem*)."""
    cout = weight.shape[0]
    w = weight.detach().float().cpu()                      # [n, ci, kh, kw]
    full = torch.zeros(3, 4, 4, cout)                      # [kh, pixel, channel, n]
    full[:, :3, :3, :] = w.permute(2, 3, 1, 0)
    return full.reshape(3, 2, 8, cout).permute(0, 1, 3, 2).contiguous().to(dtype)


_AUX_BRANCH = 7      # graph branch of the residual blocks' shortcut convs (LFD_MAX_BRANCHES - 1)


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


class InferencePlan(object):
    """One native forward plan for a fixed input shape."""

    def __init__(self, model, N, H, W, device, conv_impl=nat.CONV_UMMA, create_native=True, act_dtype='bf16', fuse_stem=None):
        """fuse_stem: run a four-conv 'faster' stem as one kernel (LFD_OP_STEM4) -- None: when its stem1 map would not stay in
        L2 (see _use_stem4), True / False: always / never (tests).  LFD_B200_NO_STEM_FUSION=1 turns it off."""
        self._configure(N, H, W, device, conv_impl, create_native, act_dtype, fuse_stem)
        self._build(model)
        self._finalize()

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
        self.concurrent_levels = not os.environ.get('LFD_B200_NO_BRANCHES')
        self.aux_shortcut = not os.environ.get('LFD_B200_NO_AUX')
        self.fuse_shortcuts = conv_impl == nat.CONV_UMMA and not os.environ.get('LFD_B200_NO_FUSED_SHORTCUT')
        # conv -> 1x1 conv pairs run as ONE kernel (tensor-core kernels only; the SIMT cross-check runs them unfused)
        self.fuse_tails = conv_impl == nat.CONV_UMMA and not os.environ.get('LFD_B200_NO_TAIL')
        self.fuse_stem = fuse_stem

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
                and sc.in_channels == c0.in_channels and sc.out_channels == c0.out_channels and c0.out_channels in (32, 64, 128)
                and sc.groups == 1 and c0.groups == 1)

    @staticmethod
    def _can_tail(conv, nxt):
        """nxt = (conv, norm, relu): a bias-free-or-not 1x1/s1 conv directly consuming `conv`'s output."""
        c2 = nxt[0]
        return (c2.kernel_size == (1, 1) and c2.stride == (1, 1) and c2.groups == 1 and c2.in_channels == conv.out_channels
                and conv.out_channels in (32, 64) and c2.out_channels in (32, 64, 128))

    def _emit_stem0(self, conv, norm, relu, out_name, h, w, tail=None):
        if conv.in_channels != 3 or conv.kernel_size != (3, 3) or conv.stride != (2, 2):
            raise NotImplementedError('the H100 stem kernel handles the 3x3/s2 conv on a 3-channel image only')
        ho, wo = _conv_out(h, 3, 2), _conv_out(w, 3, 2)
        scale, shift = self._fold(conv, norm)
        wt = pack_stem_weight(fold_scale(conv.weight, scale), self.tdtype)
        op = dict(kind=nat.OP_STEM0, H=h, W=w, Cin=3, Ho=ho, Wo=wo, Cout=conv.out_channels, ksize=3, stride=2, relu=int(relu),
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
        """A 'faster' stem (3x3/s2 3->64, 1x1, 3x3/s2 64->64, 1x1, all 64 channels) runs as one kernel when its stem1 map -- the
        tensor the fusion keeps out of HBM -- would not stay in L2 between the two fused pairs (more than half of it).  Smaller
        plans have no HBM round trip to remove and keep the two-kernel path."""
        if not self.fuse_tails or self.fuse_stem is False or os.environ.get('LFD_B200_NO_STEM_FUSION') or len(layers) != 4:
            return False
        (c0, _, _), (c1, _, _), (c2, _, _), (c3, _, _) = layers

        def conv3s2(c, cin):
            return (c.in_channels == cin and c.out_channels == 64 and c.kernel_size == (3, 3) and c.stride == (2, 2)
                    and c.padding == (1, 1) and c.groups == 1 and c.dilation == (1, 1))
        if not (conv3s2(c0, 3) and conv3s2(c2, 64) and self._can_tail(c0, layers[1]) and self._can_tail(c2, layers[3])
                and c1.out_channels == 64 and c3.out_channels == 64):
            return False
        if self.fuse_stem:
            return True
        stem1_bytes = self.N * _conv_out(self.H, 3, 2) * _conv_out(self.W, 3, 2) * 64 * 2
        return stem1_bytes > self._l2_bytes() // 2

    def _emit_stem4(self, layers, out_name, h, w):
        (c0, n0, r0), tail1, (c2, n2, r2), (c3, n3, r3) = layers
        h1, w1 = _conv_out(h, 3, 2), _conv_out(w, 3, 2)
        ho, wo = _conv_out(h1, 3, 2), _conv_out(w1, 3, 2)
        s0, b0 = self._fold(c0, n0)
        s2, b2 = self._fold(c2, n2)
        s3, b3 = self._fold(c3, n3)
        op = dict(kind=nat.OP_STEM4, H=h, W=w, Cin=3, Ho=ho, Wo=wo, Cout=64, ksize=3, stride=2, relu=int(r0),
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
        ho, wo = _conv_out(h, k, s), _conv_out(w, k, s)
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
        cur = None
        i = 0
        if self._use_stem4(layers):
            h, w = self._emit_stem4(layers, 'stem3', h, w)
            cur, i = 'stem3', len(layers)
        while i < len(layers):
            conv, norm, relu = layers[i]
            tail = None
            if self.fuse_tails and i + 1 < len(layers) and self._can_tail(conv, layers[i + 1]):
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
        if block._downsample is not None and self.fuse_shortcuts and self._can_fuse_shortcut(block, pairs):
            ds = list(block._downsample)
            fuse_sc = (ds[0], ds[1] if len(ds) > 1 else None, base + '_id')
            identity = base + '_id'
        elif block._downsample is not None:
            # the 1x1/s2 shortcut conv only depends on the block input: it runs on the auxiliary branch, next to the
            # block's first conv, and the block's last conv (which adds it) waits for it
            ds = list(block._downsample)
            aux = self.concurrent_levels and self.aux_shortcut and n_taps + 1 <= _AUX_BRANCH
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
        taps = list(bb._out_indices)
        if len(taps) != head._num_heads:
            raise ValueError('backbone taps (%d) and head levels (%d) differ' % (len(taps), head._num_heads))
        if make_norm_probe(head) is not None and not isinstance(make_norm_probe(head), nn.GroupNorm):
            raise NotImplementedError('the H100 head kernels implement GroupNorm towers and towers without norm layers (the shipped configs)')
        # point offsets need every level size up front: strides are fixed by the stage index
        sizes, hh, ww = {}, h, w
        for si, stage in enumerate(bb.stages()):
            hh, ww = _conv_out(hh, 3, 2), _conv_out(ww, 3, 2)
            for bi in range(len(stage)):
                if (si, bi) in taps:
                    sizes[(si, bi)] = (hh, ww)
        self.level_sizes = [sizes[t] for t in taps]
        self.P = sum(fh * fw for (fh, fw) in self.level_sizes)
        self.cls_channels = head.num_cls_channels
        offs, acc = [], 0
        for (fh, fw) in self.level_sizes:
            offs.append(acc)
            acc += fh * fw
        cache = {}
        for si, stage in enumerate(bb.stages()):
            for bi, block in enumerate(stage):
                cur, h, w = self._emit_block(block, 's%db%d' % (si, bi), cur, h, w, len(taps))
                if (si, bi) in taps:
                    l = taps.index((si, bi))
                    assert (h, w) == self.level_sizes[l]
                    # the level's neck + head chain only depends on this tap: run it on its own stream / graph branch,
                    # concurrently with the rest of the backbone and with the other levels
                    self._branch = 1 + l if (self.concurrent_levels and 1 + l < 8) else 0
                    self._emit_level(neck, head, l, cur, h, w, offs[l], cache)
                    self._branch = 0

    def _emit_level(self, neck, head, l, fname, fh, fw, point_off, cache):
        conv, norm = neck.level(l)
        nk = 'neck%d' % l
        cls_tower, reg_tower, fin_cls, fin_reg = head.level_paths(l)
        # merged heads: the neck's 1x1 conv (+BN+ReLU) has ONE consumer, the tower's first 1x1 conv -- run the pair as one kernel (the
        # 128-channel neck output never reaches HBM; the GroupNorm statistics are taken on the fused kernel's output as usual)
        t0 = cls_tower[0] if len(cls_tower) else None
        fuse_neck = (self.fuse_tails and not os.environ.get('LFD_B200_NO_NECK_TAIL') and cls_tower is reg_tower and t0 is not None
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
                      point_off=point_off, w_f32=self._add_f32(torch.cat(ws, 0)),
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
    def _finalize(self):
        dev = self.device
        self.params_f32 = torch.cat(self._f32).to(dev) if self._f32 else torch.zeros(4, device=dev)
        self.params_bf16 = torch.cat(self._bf16).to(dev) if self._bf16 else torch.zeros(8, dtype=torch.int16, device=dev)
        self._f32, self._bf16 = None, None
        n_stats = len([o for o in self._ops if o['kind'] == nat.OP_CONV and o.get('gn_groups')])
        stats_each = self.N * 16 * 2 * 8
        self.stats_bytes = (n_stats * stats_each + 255) & ~255
        producer = {op['out']: op['branch'] for op in self._ops if op.get('out') is not None}
        producer.update({op['out2']: op['branch'] for op in self._ops if op.get('out2') is not None})
        last_use, shared = {}, set()
        for i, op in enumerate(self._ops):
            for k in ('inp', 'res'):
                if op.get(k) is not None:
                    last_use[op[k]] = i
                    if producer[op[k]] != op['branch']:
                        shared.add(op[k])      # read by another branch (a backbone tap): lives for the whole forward
        n_br = 1 + max(op['branch'] for op in self._ops)
        arenas = [_Arena(base=0) for _ in range(n_br)]
        local = {}                              # name -> (branch, offset inside the branch's arena)
        no_reuse = bool(os.environ.get('LFD_B200_NO_REUSE'))
        for i, op in enumerate(self._ops):
            for key in ('out', 'out2'):
                if op.get(key) is not None:
                    local[op[key]] = (op['branch'], arenas[op['branch']].alloc(self._tensors[op[key]]))
            for name, lu in list(last_use.items()):
                if lu == i:
                    del last_use[name]
                    if not no_reuse and name not in shared:
                        arenas[local[name][0]].release(local[name][1], self._tensors[name])
        bases, top = [], self.stats_bytes
        for a in arenas:
            bases.append(top)
            top += (a.top + 255) & ~255
        offsets = {name: bases[b] + off for name, (b, off) in local.items()}
        self.workspace_bytes = max(top, 256)
        self.tensor_branch = {name: b for name, (b, _) in local.items()}
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
        import time
        if self.handle is None:
            raise nat.LfdError('this plan was built for host-side inspection only (create_native=False)')
        if x is None:
            x = torch.zeros((self.N, self.H, self.W, 3), dtype=torch.uint8, device=self.device)
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

        t_end = time.time() + budget_s
        work = {}
        for op in self._ops:
            if op['kind'] == nat.OP_CONV and op.get('branch', 0) > 0:
                work[op['branch']] = work.get(op['branch'], 0) + self.N * op['Ho'] * op['Wo'] * (op['Cin'] + op['Cout'])
        caps = {b: 0 for b in work}
        base = measure(caps)
        log = [('all SMs', base)]
        for b in sorted(work, key=lambda k: -work[k]):
            for c in candidates:
                if time.time() > t_end:
                    break
                trial = dict(caps)
                trial[b] = c
                t = measure(trial)
                log.append(('branch %d <= %d CTAs' % (b, c), t))
                if t < base * 0.995:
                    base, caps = t, trial
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

    def forward(self, x, use_graph=True, slot=0):
        """x: cuda float32 [N,3,H,W] (contiguous) or uint8 [N,H,W,3].  Returns the plan-owned (cls, reg) buffers of output
        `slot` (a second slot lets the post-process of one batch overlap the forward of the next, lfd/pipeline.py)."""
        if x.dtype == torch.float32:
            fmt, ok = nat.INPUT_F32_NCHW, tuple(x.shape) == (self.N, 3, self.H, self.W)
        elif x.dtype == torch.uint8:
            fmt, ok = nat.INPUT_U8_NHWC, tuple(x.shape) == (self.N, self.H, self.W, 3)
        else:
            raise TypeError('input must be float32 NCHW or uint8 NHWC, got %s' % (x.dtype,))
        if self.handle is None:
            raise nat.LfdError('this plan was built for host-side inspection only (create_native=False)')
        if not ok or not x.is_cuda or not x.is_contiguous():
            raise ValueError('input must be a contiguous CUDA tensor matching the plan shape N=%d H=%d W=%d (got %s)'
                             % (self.N, self.H, self.W, tuple(x.shape)))
        cls_out, reg_out = self.outputs(slot)
        with torch.cuda.device(self.device):
            nat.check(nat.lib().lfd_plan_forward(self.handle, nat.ptr(x), fmt, nat.ptr(self.workspace), nat.ptr(cls_out),
                                                 nat.ptr(reg_out), int(bool(use_graph)), nat.stream_ptr()))
        return cls_out, reg_out

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

    def __init__(self, N, H, W, device):
        self._configure(N, H, W, device, nat.CONV_UMMA, False, 'bf16', None)
        self.aux_shortcut = False

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
    """Pre-allocated device post-process (lfd_postprocess) for a fixed batch size / level geometry."""

    def __init__(self, cfg, device):
        self.cfg, self.device = cfg, device
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
            nat.check(nat.lib().lfd_postprocess(C.byref(self.cfg), nat.ptr(cls), nat.ptr(reg), nat.ptr(self.meta[0]), nat.ptr(self.meta[1]),
                                                nat.ptr(self.meta[2]), nat.ptr(self.ws), nat.ptr(self.dets), nat.ptr(self.labels),
                                                nat.ptr(self.src), nat.ptr(self.count), nat.ptr(self.count[self.cfg.N:]), nat.stream_ptr()))
        return self.dets, self.labels, self.src, self.count
