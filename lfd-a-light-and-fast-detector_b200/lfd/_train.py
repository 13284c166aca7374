# -*- coding: utf-8 -*-
"""Native training step of the LFD conv stack: forward in train mode (BatchNorm batch statistics), backward (data and weight
gradients of every conv, BatchNorm / GroupNorm / ReLU / residual backward, final head convs + Scale) -- all hand-written
sm_90a kernels behind liblfd_b200.so (lfd_train_plan_*), driven by two op lists built here from the module tree.

Replaces what the reference gets from autograd over its nn.Module graph in `Executor.train` (lfd/execution/executor.py:185-214:
`model(x)` ... `loss.backward()`), i.e. LFD.forward in train mode (lfd/model/lfd.py:511-542) and its backward.

Data layout: activations and their gradients bf16 NHWC in ONE workspace (every forward tensor is kept for the backward);
parameters, gradients and BatchNorm running statistics are fp32 torch tensors -- all parameters are views into ONE flat
buffer (`FlatParameters`), all gradients views into one flat gradient buffer, so that the gradient all-reduce and the fused
clip + SGD step (lfd/execution/optim.py) are single calls.  Per step the fp32 master weights are re-staged as bf16 tensor-core
operands (PACK), weight gradients are accumulated in fp32 staging tensors by the wgmma wgrad kernel and scattered into the
OIHW gradient tensors at the end (UNPACK).

Fine-tuning (frozen parameters, LFDResNet(frozen_stages=k)): backward ops are emitted only for what reaches a trainable parameter, and the
frozen backbone prefix runs on the inference plan's ops and packing (LFD_TOP_INFER), keeping only the tensors the trainable part reads.

Rounding points (bf16 training): conv output z (fp32 accumulate) -> bf16; BatchNorm statistics over the stored z (fp64 sums);
normalised + residual + ReLU output -> bf16; every activation gradient -> bf16; weight / norm-parameter gradients fp32.
"""
import os
import ctypes as C

import torch
import torch.nn as nn

from . import _native as nat
from ._engine import PrefixEmitter, _Arena

__all__ = ['FlatParameters', 'TrainPlan', 'train_forward']


def _conv_out(size, k, s):
    return (size + 2 * (k // 2) - k) // s + 1


class FlatParameters(object):
    """All parameters of a module as views into one flat fp32 buffer (+ one flat gradient buffer).  Shared parameters
    (share_head_flag aliases) appear once."""

    def __init__(self, module, allow_cpu=False):
        params, seen = [], set()
        for p in module.parameters():
            if id(p) not in seen:
                seen.add(id(p))
                params.append(p)
        if not params:
            raise ValueError('module without parameters')
        dev = params[0].device
        if dev.type != 'cuda' and not allow_cpu:      # allow_cpu: host-side planning only (CPU tests of the planner)
            raise RuntimeError('lfd_b200 has no CPU path: move the model to a CUDA (H100) device before training')
        for p in params:
            if p.dtype != torch.float32 or p.device != dev:
                raise TypeError('native training keeps fp32 master parameters on one device')
        self.params = params
        self.offsets, n = [], 0
        for p in params:
            self.offsets.append(n)
            n += (p.numel() + 3) // 4 * 4              # 16-byte aligned slots (vector loads in the optimizer kernels)
        self.numel = n
        self.data = torch.zeros(n, dtype=torch.float32, device=dev)
        self.grad = torch.zeros(n, dtype=torch.float32, device=dev)
        for p, off in zip(params, self.offsets):
            self.data[off:off + p.numel()].copy_(p.data.reshape(-1))
            p.data = self.data[off:off + p.numel()].view(p.shape)
        self.attach_grads()

    def attach_grads(self):
        """(Re-)installs the .grad views (optimizer.zero_grad(set_to_none=True) drops them).  A frozen parameter (requires_grad False)
        has no gradient, as after torch's backward: its slot of the flat gradient stays zero and its .grad None."""
        for p, off in zip(self.params, self.offsets):
            g = self.grad[off:off + p.numel()].view(p.shape)
            if not p.requires_grad:
                if p.grad is not None and p.grad.data_ptr() == g.data_ptr():
                    p.grad = None
            elif p.grad is None or p.grad.data_ptr() != g.data_ptr():
                p.grad = g

    def intact(self):
        return all(p.data_ptr() == self.data.data_ptr() + 4 * off for p, off in zip(self.params, self.offsets))

    def grad_ptr(self, p):
        return self.grad.data_ptr() + 4 * self.offsets[self._index(p)]

    def _index(self, p):
        if not hasattr(self, '_idx'):
            self._idx = {id(q): i for i, q in enumerate(self.params)}
        return self._idx[id(p)]


def flat_parameters(model, allow_cpu=False):
    fp = getattr(model, '_flat_parameters', None)
    if fp is None or not fp.intact() or len(fp.params) != len({id(p) for p in model.parameters()}):
        fp = FlatParameters(model, allow_cpu=allow_cpu)
        model._flat_parameters = fp
        model._train_plans = {}
    return fp


class _Table(object):
    """Device table of PACK / UNPACK descriptors."""

    def __init__(self, cls):
        self.cls, self.items = cls, []

    def add(self, **kw):
        self.items.append(self.cls(**kw))

    def upload(self, device):
        arr = (self.cls * len(self.items))(*self.items)
        raw = bytearray(bytes(memoryview(arr).cast('B')))
        self.tensor = torch.frombuffer(raw, dtype=torch.uint8).to(device)
        self.max_n = max([d.n for d in self.items] + [1])
        return self.tensor


class TrainPlan(object):
    """Forward (train mode) + backward op lists for a fixed input shape."""

    def __init__(self, model, N, H, W, device, create_native=True):
        self.N, self.H, self.W, self.device = N, H, W, device
        self.model = model
        self.create_native = create_native               # False: host-side planning only (CPU tests of the planner)
        self.branches = os.environ.get('LFD_B200_TRAIN_BRANCHES', '1') != '0'      # per-level chains on side streams (0: one stream, A/B runs)
        self.flat = flat_parameters(model, allow_cpu=not create_native)
        self._off, self._top = {}, 256                  # workspace regions: name -> byte offset
        self._sizes = {}
        self._fwd, self._bwd = [], []                    # op dicts (kind + fields), converted to nat.Top at the end
        self._layers = []                                # forward records, walked in reverse for the backward
        self._pack, self._unpack = _Table(nat.PackDesc), _Table(nat.UnpackDesc)
        self._wstage, self._gstage, self._hstage = {}, {}, {}
        self._const = None                               # constant tensors of the no-norm head path
        self._grad_written = set()
        self._zero_fwd, self._zero_bwd = [], []          # (name) regions cleared at the start of the forward / backward
        self._check_supported(model)
        self._trainable = {id(p) for p in model.parameters() if p.requires_grad}
        self._needs_grad = set()                         # forward tensors with a trainable parameter upstream: the only ones given a gradient
        self._prefix = None                              # the frozen backbone prefix, run on the inference kernels (_emit_prefix)
        self._build(model)
        self._finalize()

    # ------------------------------------------------------------------ checks
    @staticmethod
    def _check_supported(model):
        for m in model.modules():
            if isinstance(m, nn.BatchNorm2d):
                if not (m.affine and m.track_running_stats and m.momentum is not None):
                    raise NotImplementedError('native training needs affine BatchNorm2d with running statistics and a fixed momentum')
            if isinstance(m, nn.Conv2d) and (m.groups != 1 or m.dilation != (1, 1)):
                raise NotImplementedError('grouped / dilated convolutions are outside the LFD hot path')
        if not any(p.requires_grad for p in model.parameters()):
            raise ValueError('no parameter of the model is trainable (every requires_grad is False): nothing to train')

    # ------------------------------------------------------------------ workspace
    def _alloc(self, name, nbytes):
        if name in self._sizes:
            raise KeyError('workspace region %r allocated twice' % name)
        self._sizes[name] = nbytes       # offsets are assigned in _layout(): cleared regions first (two memsets per step)
        return name

    def _act(self, name, h, w, c):
        return self._alloc(name, self.N * h * w * c * 2)

    def _wpack(self, conv, kind, cc):
        """bf16 tensor-core operand of a conv's weight (re-staged from the fp32 master every step)."""
        key = (id(conv.weight), kind, cc)
        if key not in self._wstage:
            name = self._alloc('w%d' % len(self._wstage), conv.weight.numel() * 2 if kind != nat.PACK_STEM else 3 * 2 * conv.out_channels * 8 * 2)
            self._wstage[key] = name
            k = conv.kernel_size[0]
            n = conv.weight.numel() if kind != nat.PACK_STEM else 3 * 2 * conv.out_channels * 8
            self._pack.items.append(dict(kind=kind, Cout=conv.out_channels, Cin=conv.in_channels, k=k, cc=cc, n=n, src=conv.weight, dst=name))
        return self._wstage[key]

    def _gstage_of(self, conv):
        """fp32 staging [k*k][Cin][Cout] of a conv's weight gradient (shared by every use of the parameter)."""
        key = id(conv.weight)
        if key not in self._gstage:
            # (the stem conv's staging has 32 rows: its tensor-core path pads the 27 (tap, ci) rows to a 32-channel 1x1 problem)
            name = self._alloc('g%d' % len(self._gstage), (conv.weight.numel() if conv.in_channels != 3 else 32 * conv.out_channels) * 4)
            self._gstage[key] = name
            self._zero_bwd.append(name)
            kk = conv.kernel_size[0] ** 2
            self._unpack.items.append(dict(kind=nat.UNPACK_CONV, Cout=conv.out_channels, Cin=conv.in_channels, kk=kk, n=conv.weight.numel(),
                                           src=name, dst=conv.weight))
        return self._gstage[key]

    def _tr(self, *params):
        return any(p is not None and id(p) in self._trainable for p in params)

    def _mark(self, outs, inputs, params):
        """The tensors `outs` need a gradient when one of `inputs` does or one of `params` is trainable."""
        if any(t is not None and t in self._needs_grad for t in inputs) or self._tr(*params):
            self._needs_grad.update(outs)

    # ------------------------------------------------------------------ forward emitters
    def _conv_bn(self, name, conv, norm, relu, x, h, w, res=None):
        """conv (no bias) -> BatchNorm (batch statistics) -> (+res) -> ReLU.  x = None: the stem conv on the image."""
        k, s = conv.kernel_size[0], conv.stride[0]
        if conv.kernel_size[0] != conv.kernel_size[1] or k not in (1, 3) or s not in (1, 2) or conv.padding[0] != k // 2:
            raise NotImplementedError('unsupported conv geometry for the H100 kernels: %r' % (conv,))
        if conv.bias is not None or not isinstance(norm, nn.BatchNorm2d):
            raise NotImplementedError('native training implements conv(bias=False) + BatchNorm2d for backbone / neck layers')
        cin, cout = conv.in_channels, conv.out_channels
        ho, wo = _conv_out(h, k, s), _conv_out(w, k, s)
        z, y = self._act(name + '_z', ho, wo, cout), self._act(name, ho, wo, cout)
        sums = self._alloc(name + '_sums', cout * 16)
        self._zero_fwd.append(sums)
        geo = dict(N=self.N, H=h, W=w, Cin=cin, Ho=ho, Wo=wo, Cout=cout, ksize=k, stride=s)
        if x is None:
            wp = self._wpack(conv, nat.PACK_STEM, 0)
            self._fwd.append(dict(kind=nat.TOP_STEM0, off={1: z, 4: wp}, **geo))
            cc = 0
        else:
            cc = self._query(self.N, h, w, cin, ho, wo, cout, k, s)['cc']
            wp = self._wpack(conv, nat.PACK_CONV_FWD, cc)
            self._fwd.append(dict(kind=nat.TOP_CONV, cc=cc, off={0: x, 1: z, 4: wp}, **geo))
        frozen = int(not norm.training)       # a BatchNorm2d in eval mode inside a training step (norm_eval / frozen stages): running statistics
        bn_geo = dict(N=self.N, H=ho, W=wo, Cout=cout, eps=float(norm.eps), frozen=frozen)
        if not frozen:
            self._fwd.append(dict(kind=nat.TOP_BN_STATS, off={0: z, 3: sums}, **bn_geo))
        self._fwd.append(dict(kind=nat.TOP_BN_APPLY, relu=int(relu), momentum=float(norm.momentum), off={0: z, 1: y, 2: res, 3: sums},
                              ptr={0: norm.weight, 1: norm.bias, 2: norm.running_mean, 3: norm.running_var}, **bn_geo))
        self._layers.append(dict(type='bn', name=name, conv=conv, norm=norm, relu=relu, x=x, z=z, y=y, res=res, sums=sums, geo=geo, frozen=frozen))
        self._mark([y], [x, res], [conv.weight, norm.weight, norm.bias])
        if not frozen:
            self._bn_modules.append(norm)
        return y, ho, wo

    def _conv_gn(self, name, conv, norm, x, h, w, last):
        """1x1 / 3x3 conv -> GroupNorm (statistics from the conv epilogue) -> ReLU; `last`: the apply is fused into HEAD_FINAL."""
        k = conv.kernel_size[0]
        if conv.kernel_size not in ((1, 1), (3, 3)) or conv.stride != (1, 1) or conv.padding != (k // 2, k // 2) or conv.bias is not None:
            raise NotImplementedError('head towers: 1x1 / 3x3 stride-1 conv without bias followed by GroupNorm')
        if not isinstance(norm, nn.GroupNorm) or norm.num_groups != 16 or norm.num_channels != 128 or not norm.affine:
            raise NotImplementedError('head towers need GroupNorm(16, 128) with affine parameters')
        cin, cout = conv.in_channels, conv.out_channels
        raw = self._act(name + '_raw', h, w, cout)
        stats = self._alloc(name + '_gnstats', self.N * 16 * 2 * 8)
        self._zero_fwd.append(stats)
        cc = self._query(self.N, h, w, cin, h, w, cout, k, 1)['cc']
        wp = self._wpack(conv, nat.PACK_CONV_FWD, cc)
        geo = dict(N=self.N, H=h, W=w, Cin=cin, Ho=h, Wo=w, Cout=cout, ksize=k, stride=1)
        self._fwd.append(dict(kind=nat.TOP_CONV, cc=cc, groups=16, off={0: x, 1: raw, 3: stats, 4: wp}, **geo))
        act = None
        if not last:
            act = self._act(name, h, w, cout)
            self._fwd.append(dict(kind=nat.TOP_GN_APPLY, N=self.N, H=h, W=w, Cout=cout, groups=16, eps=float(norm.eps), off={0: raw, 1: act, 3: stats},
                                  ptr={0: norm.weight, 1: norm.bias}))
        self._layers.append(dict(type='gn', name=name, conv=conv, norm=norm, x=x, raw=raw, act=act, stats=stats, geo=geo))
        self._mark([raw, act], [x], [conv.weight, norm.weight, norm.bias])
        return raw, act, stats

    @staticmethod
    def _query(*a):
        try:
            return nat.conv_query(*a)
        except nat.LfdError as e:          # e.g. a 16-channel data gradient (FastestBlock bodies below 32 channels)
            raise NotImplementedError('native training: %s' % e)

    def _conv_bias(self, name, conv, x, h, w):
        """conv + bias + ReLU of a head tower without norm layers (TrafficLight configs, lfd_head.py norm_cfg=None): evaluated as conv ->
        'frozen BatchNorm' with constant statistics (mean 0, variance 1 - eps, gamma 1, beta = the conv's bias): y = relu(z + bias), and in the
        backward dz = g, d bias = sum g -- no extra kernels."""
        k = conv.kernel_size[0]
        if conv.kernel_size not in ((1, 1), (3, 3)) or conv.stride != (1, 1) or conv.padding != (k // 2, k // 2) or conv.bias is None:
            raise NotImplementedError('head towers without norm: 1x1 / 3x3 stride-1 conv with bias')
        cin, cout = conv.in_channels, conv.out_channels
        z, y = self._act(name + '_z', h, w, cout), self._act(name, h, w, cout)
        cc = self._query(self.N, h, w, cin, h, w, cout, k, 1)['cc']
        wp = self._wpack(conv, nat.PACK_CONV_FWD, cc)
        geo = dict(N=self.N, H=h, W=w, Cin=cin, Ho=h, Wo=w, Cout=cout, ksize=k, stride=1)
        self._fwd.append(dict(kind=nat.TOP_CONV, cc=cc, off={0: x, 1: z, 4: wp}, **geo))
        if self._const is None:
            dev = self.flat.data.device
            self._const = dict(ones=torch.ones(256, device=dev), zeros=torch.zeros(256, device=dev), var=torch.full((256,), 1.0 - 1e-5, device=dev),
                               sink=torch.zeros(256, device=dev))
        c = self._const
        bn_geo = dict(N=self.N, H=h, W=w, Cout=cout, eps=1e-5, frozen=1)
        self._fwd.append(dict(kind=nat.TOP_BN_APPLY, relu=1, momentum=0.0, off={0: z, 1: y}, ptr={0: c['ones'], 1: conv.bias, 2: c['zeros'], 3: c['var']}, **bn_geo))
        import types
        fake = types.SimpleNamespace(weight=c['ones'], bias=conv.bias, running_mean=c['zeros'], running_var=c['var'], eps=1e-5)
        self._layers.append(dict(type='bn', name=name, conv=conv, norm=fake, relu=True, x=x, z=z, y=y, res=None, sums=None, geo=geo, frozen=1,
                                 dgamma=c['sink'], dbeta=('grad', conv.bias) if self._tr(conv.bias) else None))
        self._mark([y], [x], [conv.weight, conv.bias])
        return y

    def _head_final(self, name, l, raw, stats, norm, convs, n_cls, n_reg, h, w, point_off, scale_param):
        """convs = [final conv, ...] whose outputs are concatenated (classification rows first)."""
        no, Cc = n_cls + n_reg, 128
        key = tuple(id(c.weight) for c in convs)
        if key not in self._hstage:
            ds = self._alloc('hg%d' % len(self._hstage), (no * Cc + no) * 4)          # dW | dbias, shared by the levels of a shared head
            self._hstage[key] = ds
            self._zero_bwd.append(ds)
            row = 0
            for c in convs:
                r = c.out_channels
                if self._tr(c.weight):
                    self._unpack.items.append(dict(kind=nat.UNPACK_ADD, n=r * Cc, src=(ds, row * Cc * 4), dst=c.weight))
                if self._tr(c.bias):
                    self._unpack.items.append(dict(kind=nat.UNPACK_ADD, n=r, src=(ds, (no * Cc + row) * 4), dst=c.bias))
                row += r
        ds = self._hstage[key]
        # the weight rows are shared by the levels; scale / shift / bias depend on the level's Scale parameter, so every level
        # gets its own staging copy of them (and of the rounded weights, which keeps the kernel's layout contiguous)
        lst = self._alloc('%s_stage' % name, (no * Cc + 3 * no) * 4)
        row = 0
        for c in convs:
            r = c.out_channels
            if c.bias is None:
                raise NotImplementedError('final head convs carry a bias in every shipped config')
            is_reg = row >= n_cls
            self._pack.items.append(dict(kind=nat.PACK_ROUND_F32, n=r * Cc, src=c.weight, dst=(lst, row * Cc * 4)))
            self._pack.items.append(dict(kind=nat.PACK_SCALE_SHIFT, n=r, src=c.bias, src2=scale_param if is_reg else None,
                                         dst=(lst, (no * Cc + row) * 4), dst2=(lst, (no * Cc + no + row) * 4), dst3=(lst, (no * Cc + 2 * no + row) * 4)))
            row += r
        dscale = None
        if scale_param is not None and n_reg and self._tr(scale_param):
            dscale = self._alloc('%s_dscale' % name, 4)
            self._zero_bwd.append(dscale)
            self._unpack.items.append(dict(kind=nat.UNPACK_ADD, n=1, src=dscale, dst=scale_param))
        gn = norm is not None          # None: the tower has no norm layers, `raw` is already the activated tensor
        geo = dict(N=self.N, H=h, W=w, Cout=Cc, groups=16 if gn else 0, n_cls=n_cls, n_reg=n_reg, P=None, point_off=point_off, cls_stride=None,
                   eps=float(norm.eps) if gn else 1e-5)
        nptr = {0: norm.weight, 1: norm.bias} if gn else {}
        self._fwd.append(dict(kind=nat.TOP_HEAD_FINAL, off={0: raw, 3: stats, 4: lst}, ptr={**nptr, 2: 'cls', 3: 'reg'}, **geo))
        self._layers.append(dict(type='final', name=name, raw=raw, stats=stats, norm=norm, stage=lst, dstage=ds, dscale=dscale, geo=geo,
                                 dact='d_' + (raw + '_act' if gn else raw)))

    # ------------------------------------------------------------------ graph walk (same order as the inference plan)
    @staticmethod
    def _prefix_units(model):
        """Modules of the frozen backbone prefix: the longest run of backbone units from the input (the stem, then whole residual
        blocks) whose parameters are all frozen and whose BatchNorms are all in eval mode -- with BatchNorm folded, exactly the
        inference network.  LFDResNet(frozen_stages=k >= 1) freezes the stem and stages 0..k-1 so."""
        bb = model._backbone
        units = [bb._stem] + [block for stage in bb.stages() for block in stage]
        n = 0
        for u in units:
            if any(p.requires_grad for p in u.parameters()) or any(isinstance(m, nn.BatchNorm2d) and m.training for m in u.modules()):
                break
            n += 1
        return units[:n]

    def _emit_prefix(self, model, n_units):
        """The first n_units backbone units on the inference plan's emitters -> (emitter, [(first op, end op, output, h, w) per unit])."""
        bb = model._backbone
        pre = PrefixEmitter(self.N, self.H, self.W, self.device)
        cur, h, w = pre._emit_stem(bb.stem_layers(), self.H, self.W)
        units = [(0, len(pre._ops), cur, h, w)]
        blocks = [('s%db%d' % (si, bi), block) for si, stage in enumerate(bb.stages()) for bi, block in enumerate(stage)]
        for base, block in blocks[:n_units - 1]:
            b0 = len(pre._ops)
            cur, h, w = pre._emit_block(block, base, cur, h, w, len(bb._out_indices))
            units.append((b0, len(pre._ops), cur, h, w))
        return pre, units

    def _infer_unit(self, unit):
        """LFD_TOP_INFER ops of one prefix unit (their Op descriptors are filled in by _stage_prefix once the workspace is laid out)."""
        for op in self._prefix['emitter']._ops[unit[0]:unit[1]]:
            self._fwd.append(dict(kind=nat.TOP_INFER, N=self.N, H=op['H'], W=op['W'], Cin=op['Cin'], Ho=op['Ho'], Wo=op['Wo'], Cout=op['Cout'],
                                  ksize=op.get('ksize', 1), stride=op.get('stride', 1), relu=op.get('relu', 0),
                                  off={0: op.get('inp'), 1: op['out'], 2: op.get('res'), 3: op.get('out2')}, ptr={0: None}))
            self._prefix['ops'].append((self._fwd[-1], op))

    def _build(self, model):
        bb, neck, head = model._backbone, model._neck, model._head
        self._bn_modules = []
        h, w = self.H, self.W
        cur = None
        modules = self._prefix_units(model)
        units = []
        if modules:
            pre, units = self._emit_prefix(model, len(modules))
            self._prefix = dict(emitter=pre, modules=modules, ops=[])
            self._infer_unit(units[0])
            cur, h, w = units[0][2:]
        else:
            for i, (conv, norm, relu) in enumerate(bb.stem_layers()):
                cur, h, w = self._conv_bn('stem%d' % i, conv, norm, relu, cur, h, w)
        taps = list(bb._out_indices)
        if len(taps) != head._num_heads:
            raise ValueError('backbone taps (%d) and head levels (%d) differ' % (len(taps), head._num_heads))
        sizes, hh, ww = {}, h, w
        for si, stage in enumerate(bb.stages()):
            hh, ww = _conv_out(hh, 3, 2), _conv_out(ww, 3, 2)
            for bi in range(len(stage)):
                if (si, bi) in taps:
                    sizes[(si, bi)] = (hh, ww)
        self.level_sizes = [sizes[t] for t in taps]
        self.P = sum(fh * fw for fh, fw in self.level_sizes)
        self.cls_channels = head.num_cls_channels
        offs, acc = [], 0
        for fh, fw in self.level_sizes:
            offs.append(acc)
            acc += fh * fw
        ui = 0
        for si, stage in enumerate(bb.stages()):
            for bi, block in enumerate(stage):
                base = 's%db%d' % (si, bi)
                ui += 1
                if ui < len(units):                      # a block of the frozen prefix
                    self._infer_unit(units[ui])
                    cur, h, w = units[ui][2:]
                else:
                    identity = cur
                    if block._downsample is not None:
                        ds = list(block._downsample)
                        identity, _, _ = self._conv_bn(base + '_id', ds[0], ds[1] if len(ds) > 1 else None, False, cur, h, w)
                    x, hh, ww = cur, h, w
                    pairs = block.conv_norm_pairs()
                    for li, (conv, norm) in enumerate(pairs):
                        last = li == len(pairs) - 1
                        x, hh, ww = self._conv_bn(base + ('_out' if last else '_c%d' % li), conv, norm, True, x, hh, ww, res=identity if last else None)
                    cur, h, w = x, hh, ww
                if (si, bi) in taps:
                    l = taps.index((si, bi))
                    f0, l0 = len(self._fwd), len(self._layers)
                    self._level(neck, head, l, cur, h, w, offs[l])
                    # the level's neck + head chain depends on the tap only: its own branch (side stream), in the forward and in the backward
                    br = (1 + l % (nat.MAX_BRANCHES - 1)) if self.branches else 0
                    for op in self._fwd[f0:]:
                        op['branch'] = br
                    for L in self._layers[l0:]:
                        L['branch'] = br

    def _level(self, neck, head, l, fname, fh, fw, point_off):
        conv, norm = neck.level(l)
        nk, _, _ = self._conv_bn('neck%d' % l, conv, norm, True, fname, fh, fw)
        cls_tower, reg_tower, fin_cls, fin_reg = head.level_paths(l)
        scale_param = head._scales[l]._scale if head.uses_scale else None

        def tower(t, tag):
            x = nk
            for ti, (tconv, tnorm) in enumerate(t):
                if tnorm is None:
                    x = self._conv_bias('h%d%s%d' % (l, tag, ti), tconv, x, fh, fw)
                    raw, stats = x, None
                else:
                    raw, act, stats = self._conv_gn('h%d%s%d' % (l, tag, ti), tconv, tnorm, x, fh, fw, last=ti == len(t) - 1)
                    x = act
            return raw, stats, t[-1][1]

        if cls_tower is reg_tower:
            raw, stats, tn = tower(cls_tower, 'm')
            self._head_final('h%dfin' % l, l, raw, stats, tn, [fin_cls, fin_reg], fin_cls.out_channels, 4, fh, fw, point_off, scale_param)
        else:
            raw, stats, tn = tower(cls_tower, 'c')
            self._head_final('h%dfinc' % l, l, raw, stats, tn, [fin_cls], fin_cls.out_channels, 0, fh, fw, point_off, None)
            raw, stats, tn = tower(reg_tower, 'r')
            self._head_final('h%dfinr' % l, l, raw, stats, tn, [fin_reg], 0, 4, fh, fw, point_off, scale_param)

    # ------------------------------------------------------------------ backward emitters
    def _grad_of(self, name, h, w, c):
        g = 'd_' + name
        if g not in self._sizes:
            self._act(g, h, w, c)
        return g

    def _emit_conv_backward(self, L, dz, dz_up):
        """Weight gradient (trainable weight) and data gradient (input with a trainable parameter upstream) of L['conv'] given the
        gradient of its output."""
        conv, geo, x = L['conv'], L['geo'], L['x']
        if self._tr(conv.weight):
            gs = self._gstage_of(conv)
            if x is None:
                x27 = self._act('stem_im2col', geo['Ho'], geo['Wo'], 32)      # scratch of the im2col + wgmma path
                self._bwd.append(dict(kind=nat.TOP_WGRAD_STEM, impl=nat.WGRAD_UMMA, off={0: x27, 1: dz, 5: gs}, **geo))
                return
            self._bwd.append(dict(kind=nat.TOP_WGRAD, impl=nat.WGRAD_UMMA, off={0: x, 1: dz, 5: gs}, **geo))
        if x is None or x not in self._needs_grad:
            return
        # data gradient = the forward kernel on the transposed / tap-flipped weights (stride 2: on the zero-inserted dz)
        k, s, cin, cout, h, w = geo['ksize'], geo['stride'], geo['Cin'], geo['Cout'], geo['H'], geo['W']
        cc = self._query(self.N, h, w, cout, h, w, cin, k, 1)['cc']
        wp = self._wpack(conv, nat.PACK_CONV_DGRAD, cc)
        dx = self._grad_of(x, h, w, cin)
        acc = dx in self._grad_written
        self._bwd.append(dict(kind=nat.TOP_CONV, cc=cc, N=self.N, H=h, W=w, Cin=cout, Ho=h, Wo=w, Cout=cin, ksize=k, stride=1,
                              off={0: dz_up if s == 2 else dz, 1: dx, 2: dx if acc else None, 4: wp}))
        self._grad_written.add(dx)

    def _build_backward(self):
        # level chains first: they only need the loss gradients, so they start at once on their side streams and are the first writers of
        # the taps' gradients; the backbone (main stream) accumulates into those and waits for the level's branch there (_assign_waits)
        order = [L for L in reversed(self._layers) if L.get('branch', 0)] + [L for L in reversed(self._layers) if not L.get('branch', 0)]
        for L in order:
            b0 = len(self._bwd)
            self._backward_of(L)
            for op in self._bwd[b0:]:
                op['branch'] = L.get('branch', 0)

    def _grad_ptr(self, p):
        """Where a norm backward deposits d loss / d p: p's gradient slot, or nothing for a frozen parameter."""
        return ('grad', p) if self._tr(p) else None

    def _backward_of(self, L):
        geo = L['geo']
        if L['type'] != 'final' and L['raw' if L['type'] == 'gn' else 'y'] not in self._needs_grad:
            return                                    # no trainable parameter at or upstream of this layer: no backward
        if L['type'] == 'final':
            dact = L['dact']
            acc = dact in self._grad_written          # (never: every tower has its own last tensor)
            if acc:
                raise RuntimeError('two head-final ops share one tower output')
            if dact not in self._sizes:
                self._act(dact, geo['H'], geo['W'], 128)
            nptr = {0: L['norm'].weight, 1: L['norm'].bias} if L['norm'] is not None else {}
            self._bwd.append(dict(kind=nat.TOP_HEAD_FINAL_BWD, off={0: L['raw'], 1: dact, 3: L['stats'], 4: L['stage'], 5: L['dstage'], 6: L['dscale']},
                                  ptr={**nptr, 2: 'gcls', 3: 'greg'}, **geo))
            self._grad_written.add(dact)
        elif L['type'] == 'gn':
            h, w, cout = geo['H'], geo['W'], geo['Cout']
            dact = 'd_' + (L['act'] if L['act'] is not None else L['raw'] + '_act')
            if dact not in self._grad_written:
                raise RuntimeError('gradient of %s is never produced' % L['name'])
            bs = self._alloc(L['name'] + '_bsums', (cout * 2 + self.N * 16 * 2) * 8)
            self._zero_bwd.append(bs)
            draw = self._grad_of(L['raw'], h, w, cout)
            n_geo = dict(N=self.N, H=h, W=w, Cout=cout, groups=16, relu=1, eps=float(L['norm'].eps))
            offs = {0: dact, 2: L['raw'], 3: L['stats'], 4: bs}
            self._bwd.append(dict(kind=nat.TOP_NORM_BWD_REDUCE, off=dict(offs), ptr={0: L['norm'].weight, 1: L['norm'].bias}, **n_geo))
            offs[5] = draw
            self._bwd.append(dict(kind=nat.TOP_NORM_BWD_APPLY, off=offs, ptr={0: L['norm'].weight, 1: L['norm'].bias, 2: self._grad_ptr(L['norm'].weight),
                                                                           3: self._grad_ptr(L['norm'].bias)}, **n_geo))
            self._emit_conv_backward(L, draw, None)
        else:
            ho, wo, cout, s = geo['Ho'], geo['Wo'], geo['Cout'], geo['stride']
            dy = 'd_' + L['y']
            if dy not in self._grad_written:
                raise RuntimeError('gradient of %s is never produced' % L['name'])
            bs = self._alloc(L['name'] + '_bsums', cout * 16)
            self._zero_bwd.append(bs)
            dz = self._grad_of(L['z'], ho, wo, cout)
            need_up = s == 2 and L['x'] is not None and L['x'] in self._needs_grad
            dz_up = self._act('d_' + L['z'] + '_up', geo['H'], geo['W'], cout) if need_up else None
            dres, acc = None, 0
            if L['res'] is not None and L['res'] in self._needs_grad:
                dres = self._grad_of(L['res'], ho, wo, cout)
                acc = int(dres in self._grad_written)
                self._grad_written.add(dres)
            n_geo = dict(N=self.N, H=ho, W=wo, Cout=cout, groups=0, relu=int(L['relu']), eps=float(L['norm'].eps), frozen=L['frozen'])
            offs = {0: dy, 1: L['y'] if L['relu'] else None, 2: L['z'], 3: L['sums'], 4: bs}
            rstats = {4: L['norm'].running_mean, 5: L['norm'].running_var}
            self._bwd.append(dict(kind=nat.TOP_NORM_BWD_REDUCE, off=dict(offs), ptr={0: L['norm'].weight, 1: L['norm'].bias, 4: rstats[4], 5: rstats[5]}, **n_geo))
            offs.update({5: dz, 6: dz_up, 7: dres})
            self._bwd.append(dict(kind=nat.TOP_NORM_BWD_APPLY, accumulate=acc, upH=geo['H'] if need_up else 0, upW=geo['W'] if need_up else 0, off=offs,
                                  ptr={0: L['norm'].weight, 1: L['norm'].bias,
                                       2: L['dgamma'] if 'dgamma' in L else self._grad_ptr(L['norm'].weight),
                                       3: L['dbeta'] if 'dbeta' in L else self._grad_ptr(L['norm'].bias),
                                       4: rstats[4], 5: rstats[5]},
                                  **n_geo))
            self._emit_conv_backward(L, dz, dz_up)

    # role of every off[] entry (include/lfd_b200.h, lfd_top table): R read, W write / read-modify-write, A atomic accumulation (commutes)
    _ROLES = {nat.TOP_STEM0: {1: 'W', 3: 'A', 4: 'R'}, nat.TOP_CONV: {0: 'R', 1: 'W', 2: 'R', 3: 'A', 4: 'R'},
              nat.TOP_BN_STATS: {0: 'R', 3: 'A'}, nat.TOP_BN_APPLY: {0: 'R', 1: 'W', 2: 'R', 3: 'R'}, nat.TOP_GN_APPLY: {0: 'R', 1: 'W', 3: 'R'},
              nat.TOP_HEAD_FINAL: {0: 'R', 3: 'R', 4: 'R'}, nat.TOP_HEAD_FINAL_BWD: {0: 'R', 1: 'W', 3: 'R', 4: 'R', 5: 'A', 6: 'A'},
              nat.TOP_NORM_BWD_REDUCE: {0: 'R', 1: 'R', 2: 'R', 3: 'R', 4: 'A'},
              nat.TOP_NORM_BWD_APPLY: {0: 'R', 1: 'R', 2: 'R', 3: 'R', 4: 'R', 5: 'W', 6: 'W', 7: 'W'},
              nat.TOP_WGRAD: {0: 'R', 1: 'R', 5: 'A'}, nat.TOP_WGRAD_STEM: {0: 'W', 1: 'R', 5: 'A'},
              nat.TOP_INFER: {0: 'R', 1: 'W', 2: 'R', 3: 'W'}}

    @classmethod
    def _assign_waits(cls, ops):
        """wait_mask of every op from the hazards between branches: an op waits for branch w when it touches a tensor that an op of w
        wrote (or, for a write, read / accumulated into) earlier in the list.  PACK / ZERO / UNPACK (no named tensors) are barriers: they sit
        on the main stream before the first fork resp. wait for every branch.  (Parameters and their gradients are absolute pointers: read-only
        resp. atomic accumulations, no ordering needed.)"""
        seq, synced, state, started = {0: -1}, {}, {}, set()
        for op in ops:
            b = op.get('branch', 0)
            if b and b not in started:
                started.add(b)
                seq[b] = -1
                synced[(b, 0)] = seq[0]
            need = {}

            def after(entry):
                if entry is not None and entry[0] != b and synced.get((b, entry[0]), -1) < entry[1]:
                    need[entry[0]] = max(need.get(entry[0], -1), entry[1])
            roles = cls._ROLES.get(op['kind'])
            if roles is None:                                   # PACK / ZERO / UNPACK
                if b:
                    raise RuntimeError('PACK / ZERO / UNPACK belong on the main stream')
                for w in started:
                    need[w] = seq[w]
            else:
                touched = {}
                for j, name in op.get('off', {}).items():
                    if name is None:
                        continue
                    r = roles[j]
                    touched[name] = 'W' if 'W' in (r, touched.get(name)) else ('A' if 'A' in (r, touched.get(name)) else 'R')
                for name, r in touched.items():
                    st = state.setdefault(name, dict(w=None, r={}, a={}))
                    after(st['w'])
                    if r in ('W', 'A'):
                        for e in st['r'].items():
                            after(e)
                    if r in ('W', 'R'):
                        for e in st['a'].items():
                            after(e)
            mask = 0
            for w in need:
                mask |= 1 << w
                synced[(b, w)] = seq[w]
            seq[b] += 1
            me = seq[b]
            if roles is not None:
                for name, r in touched.items():
                    st = state[name]
                    if r == 'W':
                        st['w'], st['r'], st['a'] = (b, me), {}, {}
                    elif r == 'A':
                        st['a'][b] = me
                    else:
                        st['r'][b] = me
            op['wait_mask'] = mask

    # ------------------------------------------------------------------ frozen prefix
    def _place_prefix(self):
        """Workspace of the prefix: the tensors the trainable part reads (taps inside the prefix, the boundary tensor) get their own
        regions; every other prefix tensor lives in one scratch region, reused by liveness as in the inference plan."""
        pre, ops = self._prefix['emitter'], [op for _, op in self._prefix['ops']]
        outs = {op[k] for op in ops for k in ('out', 'out2') if op.get(k) is not None}
        read = {v for op in self._fwd if op['kind'] != nat.TOP_INFER for v in op.get('off', {}).values()}
        keep = outs & read
        shapes = {}
        for op in ops:
            shapes[op['out']] = (op['Ho'], op['Wo'], op.get('tail_cout') or op['Cout'])
            if op.get('out2') is not None:
                shapes[op['out2']] = (op['Ho'], op['Wo'], op['ds_cout'])
        self.prefix_outputs = {n: shapes[n] for n in keep}          # name -> (h, w, channels), bf16 NHWC
        for n in sorted(keep):
            self._alloc(n, pre._tensors[n])
        last = {op[k]: i for i, op in enumerate(ops) for k in ('inp', 'res') if op.get(k) is not None and op[k] not in keep}
        arena, local = _Arena(), {}
        for i, op in enumerate(ops):
            for k in ('out', 'out2'):
                if op.get(k) is not None and op[k] not in keep:
                    local[op[k]] = arena.alloc(pre._tensors[op[k]])
            for n, lu in last.items():
                if lu == i:
                    arena.release(local[n], pre._tensors[n])
        if local:
            self._alloc('prefix_scratch', arena.top)
        self._prefix['scratch'] = local

    def _prefix_fingerprint(self):
        return tuple((t.data_ptr(), t._version) for m in self._prefix['modules'] for t in list(m.parameters()) + list(m.buffers()))

    def _stage_prefix(self):
        """Folded BatchNorm + packed weights of the prefix (host-built, as the inference plan builds them) and one Op descriptor per
        LFD_TOP_INFER op pointing at them."""
        pre = self._prefix['emitter']
        for n, o in self._prefix['scratch'].items():
            self._off[n] = self._off['prefix_scratch'] + o
        f32, b16 = pre.staged()
        self._prefix['f32'], self._prefix['b16'] = f32.to(self.device), b16.to(self.device)
        self._prefix['fp'] = self._prefix_fingerprint()
        fb, bb = self._prefix['f32'].data_ptr(), self._prefix['b16'].data_ptr()
        arr = (nat.Op * len(self._prefix['ops']))()
        for i, (top, op) in enumerate(self._prefix['ops']):
            pre._fill_op(arr[i], op, self._off, fb, bb)
            top['ptr'][0] = C.addressof(arr[i])
        self._prefix['arr'] = arr

    def _restage_prefix(self):
        """A prefix parameter or buffer changed (load_state_dict, a checkpoint resume, a pretrained-weight load): fold and pack again
        into the same device buffers, which the native plans and their CUDA graphs point at."""
        pre, _ = self._emit_prefix(self.model, len(self._prefix['modules']))
        f32, b16 = pre.staged()
        if f32.shape != self._prefix['f32'].shape or b16.shape != self._prefix['b16'].shape:
            raise RuntimeError('the frozen prefix changed its structure; build a new training plan')
        self._prefix['f32'].copy_(f32)
        self._prefix['b16'].copy_(b16)
        self._prefix['fp'] = self._prefix_fingerprint()

    def _layout(self):
        """Byte offsets: [regions cleared before the forward][regions cleared before the backward][everything else]."""
        zf, zb = set(self._zero_fwd), set(self._zero_bwd)
        order = list(self._zero_fwd) + list(self._zero_bwd) + [n for n in self._sizes if n not in zf and n not in zb]
        for name in order:
            self._off[name] = self._top
            self._top = (self._top + self._sizes[name] + 255) & ~255

    # ------------------------------------------------------------------ native plans
    def _finalize(self):
        dev = self.device
        self._build_backward()
        if self._prefix is not None:
            self._place_prefix()
        self._layout()
        if self._prefix is not None:
            self._stage_prefix()
        self.workspace_bytes = self._top + 256
        self.workspace = torch.zeros(self.workspace_bytes, dtype=torch.uint8, device=dev)
        base = self.workspace.data_ptr()
        self.cls_out = torch.zeros((self.N, self.P, self.cls_channels), dtype=torch.float32, device=dev)
        self.reg_out = torch.zeros((self.N, self.P, 4), dtype=torch.float32, device=dev)
        self.gcls = torch.zeros_like(self.cls_out)
        self.greg = torch.zeros_like(self.reg_out)
        self.anchor = torch.zeros(1, dtype=torch.float32, device=dev, requires_grad=True)
        named = {'cls': self.cls_out, 'reg': self.reg_out, 'gcls': self.gcls, 'greg': self.greg}

        def addr(v):      # workspace name | (name, byte offset) | tensor | ('grad', param) | None | address -> absolute pointer
            if v is None:
                return 0
            if isinstance(v, int):
                return v
            if isinstance(v, str):
                return named[v].data_ptr() if v in named else base + self._off[v]
            if isinstance(v, tuple) and v[0] == 'grad':
                return self.flat.grad_ptr(v[1])
            if isinstance(v, tuple):
                return base + self._off[v[0]] + v[1]
            return v.data_ptr()

        for d in self._pack.items:
            for k in ('src', 'src2', 'dst', 'dst2', 'dst3'):
                d[k] = addr(d.get(k))
        self._pack.items = [nat.PackDesc(**d) for d in self._pack.items]
        for d in self._unpack.items:
            d['src'] = addr(d['src'])
            d['dst'] = self.flat.grad_ptr(d['dst'])
        self._unpack.items = [nat.UnpackDesc(**d) for d in self._unpack.items]
        pack_t, unpack_t = self._pack.upload(dev), self._unpack.upload(dev)

        def zero_ops(names):
            # merge adjacent regions into few memsets
            spans = sorted((self._off[n], self._off[n] + ((self._sizes[n] + 255) & ~255)) for n in names)
            merged = []
            for b, e in spans:
                if merged and merged[-1][1] == b:
                    merged[-1][1] = e
                else:
                    merged.append([b, e])
            return [dict(kind=nat.TOP_ZERO, off={0: b, 1: e - b}) for b, e in merged]

        fwd = [dict(kind=nat.TOP_PACK, n_desc=len(self._pack.items), max_n=self._pack.max_n, ptr={0: pack_t})] + zero_ops(self._zero_fwd) + self._fwd
        bwd = zero_ops(self._zero_bwd) + self._bwd + [dict(kind=nat.TOP_UNPACK, n_desc=len(self._unpack.items), max_n=self._unpack.max_n, ptr={0: unpack_t})]

        self._assign_waits(fwd)
        self._assign_waits(bwd)

        def to_array(ops):
            arr = (nat.Top * len(ops))()
            for i, op in enumerate(ops):
                t = arr[i]
                for j in range(8):
                    t.off[j] = -1
                for key, v in op.items():
                    if key == 'off':
                        for j, o in v.items():
                            t.off[j] = -1 if o is None else (o if isinstance(o, int) else self._off[o])
                    elif key == 'ptr':
                        for j, pv in v.items():
                            t.ptr[j] = addr(pv)
                    elif key == 'P':
                        t.P = self.P
                    elif key == 'cls_stride':
                        t.cls_stride = self.cls_channels
                    else:
                        setattr(t, key, v)
            return arr

        self._fwd_arr, self._bwd_arr = to_array(fwd), to_array(bwd)
        self.fwd_ops, self.bwd_ops = fwd, bwd
        self._keep = (pack_t, unpack_t)
        self.fwd_handle, self.bwd_handle = C.c_void_p(), C.c_void_p()
        self._input = None
        self._bn_tracked = [m.num_batches_tracked for m in self._bn_modules if m.num_batches_tracked is not None]
        if not self.create_native:
            return
        with torch.cuda.device(dev):
            nat.check(nat.lib().lfd_train_plan_create(self._fwd_arr, len(fwd), self.workspace_bytes, C.byref(self.fwd_handle)))
            nat.check(nat.lib().lfd_train_plan_create(self._bwd_arr, len(bwd), self.workspace_bytes, C.byref(self.bwd_handle)))

    # ------------------------------------------------------------------ execution
    def forward(self, x, use_graph=False):
        if x.dtype == torch.float32:
            fmt, ok = nat.INPUT_F32_NCHW, tuple(x.shape) == (self.N, 3, self.H, self.W)
        elif x.dtype == torch.uint8:
            fmt, ok = nat.INPUT_U8_NHWC, tuple(x.shape) == (self.N, self.H, self.W, 3)
        else:
            raise TypeError('input must be float32 NCHW or uint8 NHWC, got %s' % (x.dtype,))
        if not ok or not x.is_cuda:
            raise ValueError('input must be a CUDA tensor matching the plan shape N=%d H=%d W=%d (got %s)' % (self.N, self.H, self.W, tuple(x.shape)))
        # the backward reads the image again (stem weight gradient): keep it in a plan-owned buffer with a fixed address
        if self._input is None or self._input.dtype != x.dtype:
            self._input = torch.empty_like(x, memory_format=torch.contiguous_format)
        self._input.copy_(x)
        if self._prefix is not None and self._prefix_fingerprint() != self._prefix['fp']:
            self._restage_prefix()
        self._fmt = fmt
        with torch.cuda.device(self.device):
            nat.check(nat.lib().lfd_train_plan_run(self.fwd_handle, nat.ptr(self._input), fmt, nat.ptr(self.workspace), int(bool(use_graph)), nat.stream_ptr()))
        if self._bn_tracked:
            torch._foreach_add_(self._bn_tracked, 1)
        return self.cls_out, self.reg_out

    def backward(self, grad_cls, grad_reg, use_graph=False):
        """Accumulates d loss / d parameter into the flat gradient buffer (the .grad views of the parameters)."""
        self.flat.attach_grads()
        self.gcls.copy_(grad_cls)
        self.greg.copy_(grad_reg)
        with torch.cuda.device(self.device):
            nat.check(nat.lib().lfd_train_plan_run(self.bwd_handle, nat.ptr(self._input), self._fmt, nat.ptr(self.workspace), int(bool(use_graph)), nat.stream_ptr()))

    def autotune(self, candidates=(96, 64, 48), budget_s=4.0):
        """As InferencePlan.autotune: bounds on the persistent CTAs of the side-branch (per-level chain) convs / data-gradient convs /
        weight-gradient kernels, picked per branch by timing the replayed forward and backward graphs.  Model state touched by the timing
        runs (BatchNorm running statistics, the flat gradient buffer, the plan's outputs) is saved and restored."""
        import time
        if not self.create_native or not self.branches:
            return {}
        dev, lib = self.device, nat.lib()
        saved = [t.clone() for m in self._bn_modules for t in (m.running_mean, m.running_var)]
        tracked = [t.clone() for t in self._bn_tracked]
        grad = self.flat.grad.clone() if self.flat.grad is not None else None
        outs = [t.clone() for t in (self.cls_out, self.reg_out, self.gcls, self.greg)]
        if self._input is None:
            self._input = torch.zeros((self.N, self.H, self.W, 3), dtype=torch.uint8, device=dev)
            self._fmt = nat.INPUT_U8_NHWC
        tuned = (nat.TOP_CONV, nat.TOP_WGRAD)
        result = {}
        t_end = time.time() + budget_s
        try:
            for which, arr, ops in (('fwd', self._fwd_arr, self.fwd_ops), ('bwd', self._bwd_arr, self.bwd_ops)):
                def set_caps(caps):
                    for o, op in zip(arr, ops):
                        if op['kind'] in tuned and op.get('branch', 0) > 0:
                            o.max_ctas = int(caps.get(op['branch'], 0))

                def measure(caps):
                    set_caps(caps)
                    h = C.c_void_p()
                    with torch.cuda.device(dev):
                        nat.check(lib.lfd_train_plan_create(arr, len(ops), self.workspace_bytes, C.byref(h)))
                        try:
                            def run():
                                nat.check(lib.lfd_train_plan_run(h, nat.ptr(self._input), self._fmt, nat.ptr(self.workspace), 1, nat.stream_ptr()))
                            run()
                            run()
                            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                            best = []
                            for _ in range(3):
                                e0.record()
                                for _ in range(3):
                                    run()
                                e1.record()
                                torch.cuda.synchronize(dev)
                                best.append(e0.elapsed_time(e1) / 3)
                            return sorted(best)[1]
                        finally:
                            lib.lfd_train_plan_destroy(h)

                work = {}
                for op in ops:
                    if op['kind'] in tuned and op.get('branch', 0) > 0:
                        work[op['branch']] = work.get(op['branch'], 0) + op['N'] * op['Ho'] * op['Wo'] * (op['Cin'] + op['Cout'])
                caps = {b: 0 for b in work}
                base = measure(caps)
                log = [('all SMs', base)]
                for b in sorted(work, key=lambda k: -work[k])[:3]:
                    for c in candidates:
                        if time.time() > t_end:
                            break
                        trial = dict(caps)
                        trial[b] = c
                        t = measure(trial)
                        log.append(('branch %d <= %d CTAs' % (b, c), t))
                        if t < base * 0.995:
                            base, caps = t, trial
                set_caps(caps)
                name = which + '_handle'
                old = getattr(self, name)
                h = C.c_void_p()
                with torch.cuda.device(dev):
                    nat.check(lib.lfd_train_plan_create(arr, len(ops), self.workspace_bytes, C.byref(h)))
                setattr(self, name, h)
                lib.lfd_train_plan_destroy(old)
                result[which] = dict(ctas=caps, log=log)
        finally:
            torch.cuda.synchronize(dev)
            it = iter(saved)
            for m in self._bn_modules:
                m.running_mean.copy_(next(it))
                m.running_var.copy_(next(it))
            for t, v in zip(self._bn_tracked, tracked):
                t.copy_(v)
            if grad is not None:
                self.flat.grad.copy_(grad)
            for t, v in zip((self.cls_out, self.reg_out, self.gcls, self.greg), outs):
                t.copy_(v)
        self.autotune_result = result
        return result

    def tensor(self, name, h, w, c):
        """Debug view of a workspace activation / gradient as bf16 NHWC."""
        off = self._off[name]
        return self.workspace[off:off + self.N * h * w * c * 2].view(torch.bfloat16).view(self.N, h, w, c)

    def profile(self, which='fwd'):
        handle, ops = (self.fwd_handle, self.fwd_ops) if which == 'fwd' else (self.bwd_handle, self.bwd_ops)
        ms = (C.c_float * len(ops))()
        with torch.cuda.device(self.device):
            nat.check(nat.lib().lfd_train_plan_profile(handle, nat.ptr(self._input), self._fmt, nat.ptr(self.workspace), ms, nat.stream_ptr()))
        return list(ms)

    def __del__(self):
        try:
            for h in ('fwd_handle', 'bwd_handle'):
                if getattr(self, h, None):
                    nat.lib().lfd_train_plan_destroy(getattr(self, h))
                    setattr(self, h, None)
        except Exception:
            pass


class _TrainFn(torch.autograd.Function):
    """Autograd node of the whole native forward: backward() runs the native backward plan, which deposits the parameter
    gradients directly into the flat gradient buffer (so `loss.backward()` of the reference's train loop keeps working)."""

    @staticmethod
    def forward(ctx, anchor, x, plan):
        ctx.plan = plan
        cls, reg = plan.forward(x, use_graph=plan.use_graph)
        return cls.detach(), reg.detach()      # fresh tensor objects over the plan-owned buffers (autograd attaches its node to them)

    @staticmethod
    def backward(ctx, grad_cls, grad_reg):
        plan = ctx.plan
        if grad_cls is None:
            grad_cls = torch.zeros_like(plan.cls_out)
        if grad_reg is None:
            grad_reg = torch.zeros_like(plan.reg_out)
        plan.backward(grad_cls, grad_reg, use_graph=plan.use_graph)
        return None, None, None


def train_forward(model, x):
    """Training-mode LFD.forward: (classification [N,P,C'], regression [N,P,4]) float32, differentiable (the outputs are
    plan-owned buffers, overwritten by the next forward of the same shape)."""
    if x.dtype == torch.uint8:
        n, h, w = x.shape[0], x.shape[1], x.shape[2]
    else:
        n, h, w = x.shape[0], x.shape[2], x.shape[3]
    plan = model.train_plan_for(n, h, w, x.device)
    for i, hw in enumerate(plan.level_sizes):
        model._head_indexes_to_feature_map_sizes[i] = hw
    return _TrainFn.apply(plan.anchor, x, plan)
