# -*- coding: utf-8 -*-
"""Every op of a native training step, replayed one at a time on the plan's own workspace and checked per element against float64.

The op-level tests (test_gpu_train_kernel_configs.py, test_gpu_conv_configs.py, test_gpu_wgrad_configs.py) hold each kernel to its
per-element bound on operands they build.  Here the operands are what TrainPlan launches: real activations, the plan's geometry and flags,
its in-place accumulations and its pointer wiring.  One ordinary step fills plan.gcls / plan.greg with the loss gradients; the starting
state is restored (running statistics, a zero flat gradient, a zero workspace) and plan._fwd_arr, then plan._bwd_arr, are replayed through
lfd_run_top in list order (a valid linear order of the plan's hazards: _assign_waits derives the waits from it).  Before each op its
read regions are snapshotted and every region it only writes is NaN-filled, so an element it never writes fails; after it, every output
element is compared with a float64 reference computed on the GPU from the snapshots (train_op_ref.py), with the same K * 2^-24 * S and
faithful-rounding bounds as the op-level tests.  The values a reference depends on -- eps, momentum, eval-mode BatchNorm, strides, up-sampled
sizes, which producer of a gradient writes and which accumulates, each level's first point -- come from the modules and the layer records,
not from the op, so a wrong field in the op list fails.

Then the same step runs through lfd_train_plan_run (branches on, CUDA graph: the eager first call captures, the second replays) from the
same starting state, and every region, the flat gradient, the running statistics and cls / reg must agree with the replay up to the
order of the fp32 / fp64 atomics (test_gpu_schedule_invariance.py's rule for the 16-bit tensors)."""
import ctypes as C
import re
import time

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import synth
from gpu_train_ops import gn_bwd_blocks, grid_sms, head_bwd_grid, reduce_blocks
from helpers import synth_model
from lfd import _native as nat
from gpu_ops import ref_conv64, stem_operand, ulp16
from lfd._engine import pack_stem_weight
from train_op_ref import (U, bf, bn_apply_ref, bn_bwd_ref, bn_running_ref, bn_stats_ref, check_amb, check_conv_op, check_faithful, check_within, conv_pack_ref,
                          gn_bwd_ref, head_activation, head_backward_ref, head_forward_ref, layer_relu)

DEV = 'cuda'
WGRAD_K = 1e-5 / U          # the wgrad config test's bound 1e-5 * S: a tile lost or counted twice moves an element by about S / tiles
ALL_KINDS = {nat.TOP_PACK, nat.TOP_ZERO, nat.TOP_STEM0, nat.TOP_CONV, nat.TOP_BN_STATS, nat.TOP_BN_APPLY, nat.TOP_GN_APPLY, nat.TOP_HEAD_FINAL,
             nat.TOP_HEAD_FINAL_BWD, nat.TOP_NORM_BWD_REDUCE, nat.TOP_NORM_BWD_APPLY, nat.TOP_WGRAD, nat.TOP_WGRAD_STEM, nat.TOP_UNPACK,
             nat.TOP_INFER}
KIND_NAMES = {v: k[4:] for k, v in vars(nat).items() if k.startswith('TOP_') and isinstance(v, int)}
WORST = {}          # largest err / tol per (kind, output) over the replays of a session


def _conv64(x, w, shift, stride, relu=False, res=None):
    """gpu_ops.ref_conv64 on the GPU for a conv whose 16-bit weights w are given as they are (no BatchNorm fold); shift None: none."""
    cout = w.shape[0]
    sh = torch.zeros(cout) if shift is None else shift.float().cpu()
    return ref_conv64(x, w.float().cpu(), torch.ones(cout), sh, stride, relu, res=res, device=DEV)


def _image(x):
    """The stem's 16-bit operand (rounding point R0), on the GPU."""
    return stem_operand(x, 'u8' if x.dtype == torch.uint8 else 'f32', None, 'bf16')


class Replay(object):
    """One training step of `model` on x (cuda, f32 NCHW or u8 NHWC), replayed op by op."""

    def __init__(self, model, x, ann):
        self.model, self.x = model, x
        n = x.shape[0]
        h, w = (x.shape[1], x.shape[2]) if x.dtype == torch.uint8 else (x.shape[2], x.shape[3])
        self.bn = [m for m in model.modules() if isinstance(m, nn.BatchNorm2d)]
        self.relu = layer_relu(model)          # the frozen prefix's ReLUs, from the layer records
        self.bn0 = [(m.running_mean.clone(), m.running_var.clone()) for m in self.bn]
        out = model(x)
        model.get_loss(out, ann)['loss'].backward()
        torch.cuda.synchronize()
        self.plan = plan = model.train_plan_for(n, h, w, x.device)
        self.N = n
        self.base = plan.workspace.data_ptr()
        self.sms = nat.lib().lfd_device_sm_count()
        self.regions = {name: plan._off[name] for name in plan._sizes}
        self.by_off = {o: name for name, o in self.regions.items()}
        assert len(self.by_off) == len(self.regions), 'two workspace regions at one offset'
        self.shapes = {}          # region -> (dtype, shape)
        self.layer_of = {}        # region -> the layer record that owns it
        N = n
        for L in plan._layers:
            g = L['geo']
            if L['type'] == 'bn':
                for t in (L['z'], L['y']):
                    self._shape(t, torch.bfloat16, (N, g['Ho'], g['Wo'], g['Cout']), L)
                    self._shape('d_' + t, torch.bfloat16, (N, g['Ho'], g['Wo'], g['Cout']), L)
                self._shape('d_' + L['z'] + '_up', torch.bfloat16, (N, g['H'], g['W'], g['Cout']), L)
                if L['sums'] is not None:
                    self._shape(L['sums'], torch.float64, (g['Cout'], 2), L)
                self._shape(L['name'] + '_bsums', torch.float64, (g['Cout'], 2), L)
            elif L['type'] == 'gn':
                for t in (L['raw'], L['act'], L['raw'] + '_act'):
                    if t is not None:
                        self._shape(t, torch.bfloat16, (N, g['H'], g['W'], g['Cout']), L)
                        self._shape('d_' + t, torch.bfloat16, (N, g['H'], g['W'], g['Cout']), L)
                self._shape(L['stats'], torch.float64, (N, 16, 2), L)
                self._shape(L['name'] + '_bsums', torch.float64, (g['Cout'] * 2 + N * 32,), L)
            else:
                no = g['n_cls'] + g['n_reg']
                self._shape(L['stage'], torch.float32, (no * 128 + 3 * no,), L)
                self._shape(L['dstage'], torch.float32, (no * 128 + no,), None)
                if L['dscale'] is not None:
                    self._shape(L['dscale'], torch.float32, (1,), L)
                self._shape(L['dact'], torch.bfloat16, (N, g['H'], g['W'], 128), L)
            if L.get('x') is not None:
                self._shape(L['x'], torch.bfloat16, (N, g['H'], g['W'], g['Cin']), None)
                self._shape('d_' + L['x'], torch.bfloat16, (N, g['H'], g['W'], g['Cin']), None)
            if L['type'] != 'final' and L.get('x', 0) is None:
                self._shape('stem_im2col', torch.bfloat16, (N, g['Ho'], g['Wo'], 32), L)
        for name, (hh, ww, c) in getattr(plan, 'prefix_outputs', {}).items():
            self._shape(name, torch.bfloat16, (N, hh, ww, c), None)
        # each level's first point, from the level sizes (and those from the layers that run at them)
        self.point_off, acc = [], 0
        for hh, ww in plan.level_sizes:
            self.point_off.append(acc)
            acc += hh * ww
        assert acc == plan.P
        self.param_of = {p.data_ptr(): p for p in plan.flat.params}
        self.tol_grad = torch.zeros(plan.flat.numel, dtype=torch.float64, device=DEV)     # per-element bound of the flat gradient
        self.tol = {}                                                                      # fp32 / fp64 region -> its per-element bound
        self.checked = {'fwd': 0, 'bwd': 0}
        self.out_tol = {'cls': torch.zeros_like(plan.cls_out, dtype=torch.float64), 'reg': torch.zeros_like(plan.reg_out, dtype=torch.float64)}

    def _shape(self, name, dtype, shape, L):
        if name in self.regions:
            self.shapes[name] = (dtype, shape)
            if L is not None:
                self.layer_of.setdefault(name, L)

    # ------------------------------------------------------------------ workspace access
    def view(self, name, ws=None):
        ws = self.plan.workspace if ws is None else ws
        dtype, shape = self.shapes[name]
        o = self.regions[name]
        n = 1
        for s in shape:
            n *= s
        return ws[o:o + n * torch.empty(0, dtype=dtype).element_size()].view(dtype).view(shape)

    def name_at(self, off):
        if off < 0:
            return None
        assert off in self.by_off, 'offset %d is not the start of a workspace region' % off
        return self.by_off[off]

    def nan_fill(self, name):
        self.view(name).fill_(float('nan'))

    def grad_of(self, p):
        o = self.plan.flat.offsets[self.plan.flat._index(p)]
        return slice(o, o + p.numel())

    def restore(self):
        plan = self.plan
        for m, (rm, rv) in zip(self.bn, self.bn0):
            m.running_mean.copy_(rm)
            m.running_var.copy_(rv)
        plan.flat.grad.zero_()
        plan.workspace.zero_()
        if plan._const is not None:
            plan._const['sink'].zero_()
        plan.cls_out.fill_(float('nan'))
        plan.reg_out.fill_(float('nan'))
        torch.cuda.synchronize()

    def run(self, t):
        plan = self.plan
        with torch.cuda.device(plan.device):
            nat.check(nat.lib().lfd_run_top(C.byref(t), nat.ptr(plan._input), plan._fmt, nat.ptr(plan.workspace), nat.stream_ptr()))
            torch.cuda.synchronize()

    def note(self, kind, out, ratio):
        key = '%s %s' % (KIND_NAMES[kind], out)
        WORST[key] = max(WORST.get(key, 0.0), ratio)

    # ------------------------------------------------------------------ the replay
    def replay(self):
        plan = self.plan
        self.restore()
        self.written = set()          # gradient tensors some earlier backward op wrote: later producers accumulate
        self.K_s = {}                 # BatchNorm sums -> the fp32 roundings of the BN_STATS that produced them
        self.grad_written = set()     # parameters whose gradient slot some op wrote
        self.prefix_ops = [op for _, op in plan._prefix['ops']] if plan._prefix is not None else []
        self.n_infer = 0
        self.zero_spans = {'fwd': [], 'bwd': []}
        for which, arr in (('fwd', plan._fwd_arr), ('bwd', plan._bwd_arr)):
            self.which = which
            for i in range(len(arr)):
                t = arr[i]
                self.what = '%s op %d (%s)' % (which, i, KIND_NAMES[t.kind])
                getattr(self, 'op_' + KIND_NAMES[t.kind].lower())(t)
                self.checked[which] += 1
            if which == 'fwd':
                assert not bool(torch.isnan(plan.cls_out).any()) and not bool(torch.isnan(plan.reg_out).any()), 'cls / reg points no level wrote'
        self._check_zero_cover()
        for name in getattr(plan, 'prefix_outputs', {}):       # the frozen prefix is not differentiated
            assert not [r for r in self.regions if r.startswith('d_' + name)], 'gradient region of the frozen prefix tensor %s' % name
        assert self.checked == {'fwd': len(plan._fwd_arr), 'bwd': len(plan._bwd_arr)}
        assert self.n_infer == len(self.prefix_ops)
        torch.cuda.synchronize()

    # --------------------------------------------------------------- tables and memsets
    def op_zero(self, t):
        b, e = t.off[0], t.off[0] + t.off[1]
        self.plan.workspace[b:e].fill_(0xFF)
        self.run(t)
        assert bool((self.plan.workspace[b:e] == 0).all()), self.what
        self.zero_spans[self.which].append((b, e))

    def _check_zero_cover(self):
        """The regions every step must start from zero (fp64 statistics, atomically accumulated gradient staging) lie in the memsets of
        their pass."""
        pats = {'fwd': r'(_sums|_gnstats)$', 'bwd': r'(_bsums|_dscale)$|^h?g\d+$'}
        for which, pat in pats.items():
            for name in self.regions:
                if re.search(pat, name):
                    b, e = self.regions[name], self.regions[name] + self.plan._sizes[name]
                    assert any(lo <= b and e <= hi for lo, hi in self.zero_spans[which]), '%s is not cleared before the %s pass' % (name, which)

    def _ptr_region(self, ptr, nbytes):
        ws = self.plan.workspace
        o = ptr - self.base
        assert 0 <= o and o + nbytes <= ws.numel(), 'pointer outside the workspace'
        return ws[o:o + nbytes]

    def op_pack(self, t):
        items = self.plan._pack.items
        assert t.n_desc == len(items) and t.max_n == max(d.n for d in items)
        checks = []
        for d in items:
            p = self.param_of[d.src]
            if d.kind in (nat.PACK_CONV_FWD, nat.PACK_CONV_DGRAD):
                want = conv_pack_ref(p.detach(), d.cc, d.kind == nat.PACK_CONV_DGRAD)
                dst = self._ptr_region(d.dst, d.n * 2).view(torch.bfloat16)
                assert d.n == p.numel()
                checks.append((dst, want))
            elif d.kind == nat.PACK_STEM:
                want = pack_stem_weight(p.detach()).reshape(-1).to(DEV)
                checks.append((self._ptr_region(d.dst, d.n * 2).view(torch.bfloat16), want))
            elif d.kind == nat.PACK_ROUND_F32:
                checks.append((self._ptr_region(d.dst, d.n * 4).view(torch.float32), p.detach().reshape(-1)[:d.n].to(torch.bfloat16).float()))
            else:
                s = self.param_of[d.src2].detach().float().expand(d.n) if d.src2 else torch.ones(d.n, device=DEV)
                b = p.detach().float().reshape(-1)
                for ptr, want in ((d.dst, s), (d.dst2, b * s), (d.dst3, b)):
                    checks.append((self._ptr_region(ptr, d.n * 4).view(torch.float32), want))
        for dst, _ in checks:
            dst.fill_(float('nan'))
        self.run(t)
        for i, (dst, want) in enumerate(checks):
            assert torch.equal(dst.float(), want.float()), '%s: descriptor %d' % (self.what, i)

    def op_unpack(self, t):
        plan = self.plan
        items = plan._unpack.items
        assert t.n_desc == len(items)
        g0 = plan.flat.grad.clone()
        want = g0.clone()
        tol = self.tol_grad.clone()
        seen = set()
        for d in items:
            o = (d.dst - plan.flat.grad.data_ptr()) // 4
            assert d.dst not in seen and 0 <= o and o + d.n <= plan.flat.numel
            seen.add(d.dst)
            p = plan.flat.params[plan.flat.offsets.index(o)]
            assert p.numel() == d.n and p.requires_grad
            if d.kind == nat.UNPACK_CONV:
                name = self.by_off[d.src - self.base]
                co, ci, k = p.shape[0], p.shape[1], p.shape[2]
                stage = self._ptr_region(d.src, ci * co * k * k * 4).view(torch.float32).view(k * k, ci, co)
                src = stage.permute(2, 1, 0).reshape(-1)
                stol = self.tol[name][:k * k * ci * co].view(k * k, ci, co).permute(2, 1, 0).reshape(-1)
            else:
                src = self._ptr_region(d.src, d.n * 4).view(torch.float32)
                name = [nm for nm, off in self.regions.items() if off <= d.src - self.base < off + plan._sizes[nm]][0]
                stol = self.tol[name].reshape(-1)[(d.src - self.base - self.regions[name]) // 4:][:d.n]
            want[o:o + d.n] += src
            self.grad_written.add(id(p))
            tol[o:o + d.n] += stol + U * (want[o:o + d.n].double().abs())
        self.run(t)
        assert torch.equal(plan.flat.grad, want), self.what
        self.tol_grad = tol
        # a frozen parameter has no gradient (its slot stays zero); every trainable one was written by UNPACK or a norm backward
        for p in plan.flat.params:
            if not p.requires_grad:
                assert bool((plan.flat.grad[self.grad_of(p)] == 0).all()), '%s: gradient of a frozen parameter' % self.what
        missing = [i for i, p in enumerate(plan.flat.params) if p.requires_grad and id(p) not in self.grad_written]
        assert not missing, '%s: trainable parameters %s get no gradient' % (self.what, missing)

    # --------------------------------------------------------------- forward convs
    def _conv_layer(self, t):
        L = self.layer_of[self.name_at(t.off[1])]
        assert L['type'] in ('bn', 'gn') and self.name_at(t.off[1]) == (L['z'] if L['type'] == 'bn' else L['raw'])
        return L

    def op_stem0(self, t):
        L = self._conv_layer(t)
        conv = L['conv']
        z = self.name_at(t.off[1])
        self.nan_fill(z)
        self.run(t)
        ref, S, K = _conv64(_image(self.x), bf(conv.weight.detach()), None, 2)
        self.note(t.kind, 'z', check_faithful(self.view(z), ref, S, K, self.what + ' z'))

    def op_conv(self, t):
        if self.which == 'bwd':
            return self._dgrad(t)
        L = self._conv_layer(t)
        conv, g = L['conv'], L['geo']
        assert (t.ksize, t.stride, t.H, t.W, t.Cin, t.Cout) == (conv.kernel_size[0], conv.stride[0], g['H'], g['W'], conv.in_channels, conv.out_channels)
        x, z = self.name_at(t.off[0]), self.name_at(t.off[1])
        assert x == L['x'] and t.off[2] < 0
        st = self.name_at(t.off[3])
        assert st == (L['stats'] if L['type'] == 'gn' else None)
        if st is not None:
            st0 = self.view(st).clone()
        self.nan_fill(z)
        self.run(t)
        ref, S, K = _conv64(self.view(x), bf(conv.weight.detach()), None, conv.stride[0])
        out = self.view(z)
        self.note(t.kind, 'z', check_faithful(out, ref, S, K, self.what + ' z'))
        if st is not None:       # fused GroupNorm statistics of the stored output: fp32 partials of a few dozen values, fp64 atomics
            o = out.double().reshape(self.N, -1, 16, 8)
            s1, s2, a1 = o.sum((1, 3)), (o * o).sum((1, 3)), o.abs().sum((1, 3))
            got = self.view(st)
            self.note(t.kind, 'GroupNorm sums', check_within(got[..., 0], st0[..., 0] + s1, a1 + st0[..., 0].abs(), 1e-5 / U, self.what + ' sum x'))
            self.note(t.kind, 'GroupNorm sums', check_within(got[..., 1], st0[..., 1] + s2, s2 + st0[..., 1].abs(), 1e-5 / U, self.what + ' sum x^2'))
            self.tol[st] = 1e-5 * torch.stack([a1, s2], -1)

    def _dgrad(self, t):
        """Data gradient: the forward kernel on the transposed, tap-flipped weights over dz (stride 1) or its zero-inserted copy (stride 2)."""
        src, dx = self.name_at(t.off[0]), self.name_at(t.off[1])
        L = self.layer_of[src]
        conv, g = L['conv'], L['geo']
        dz = 'd_' + (L['z'] if L['type'] == 'bn' else L['raw'])
        assert src == (dz + '_up' if conv.stride[0] == 2 else dz), self.what
        assert dx == 'd_' + L['x'] and (t.H, t.W, t.Cin, t.Cout, t.ksize, t.stride) == (g['H'], g['W'], conv.out_channels, conv.in_channels, conv.kernel_size[0], 1)
        acc = dx in self.written
        assert (t.off[2] >= 0) == acc and (not acc or t.off[2] == t.off[1]), '%s: accumulate into %s is %d, expected %d' % (self.what, dx, t.off[2] >= 0, acc)
        prev = self.view(dx).clone() if acc else None
        if not acc:
            self.nan_fill(dx)
        self.run(t)
        wt = bf(conv.weight.detach()).permute(1, 0, 2, 3).flip(2, 3)
        ref, S, K = _conv64(self.view(src), wt, None, 1, res=prev)
        self.note(t.kind, 'dx', check_faithful(self.view(dx), ref, S, K, self.what + ' dx'))
        self.written.add(dx)

    # --------------------------------------------------------------- BatchNorm forward
    def _bn_layer(self, t):
        L = self.layer_of[self.name_at(t.off[0])]
        assert L['type'] == 'bn' and self.name_at(t.off[0]) == L['z'], self.what
        g = L['geo']
        assert (t.N, t.H, t.W, t.Cout) == (self.N, g['Ho'], g['Wo'], g['Cout']), self.what
        norm = L['norm']
        frozen = not getattr(norm, 'training', False)       # (the constant statistics of a conv + bias tower: a frozen BatchNorm)
        return L, norm, frozen

    def op_bn_stats(self, t):
        L, norm, frozen = self._bn_layer(t)
        assert not frozen and self.name_at(t.off[3]) == L['sums'], self.what
        s0 = self.view(L['sums']).clone()
        self.run(t)
        g = L['geo']
        z = self.view(L['z']).double().reshape(-1, g['Cout'])
        ref, S, K = bn_stats_ref(z, reduce_blocks(z.numel() // 8, grid_sms(t.max_ctas, self.sms)))
        self.note(t.kind, 'sums', check_within(self.view(L['sums']), s0 + ref, S + s0.abs(), K, self.what + ' sums'))
        self.tol[L['sums']] = K * U * (S + s0.abs())
        self.K_s[L['sums']] = K

    def op_bn_apply(self, t):
        L, norm, frozen = self._bn_layer(t)
        g = L['geo']
        assert t.frozen == int(frozen), '%s: frozen = %d for a BatchNorm in %s mode' % (self.what, t.frozen, 'eval' if frozen else 'train')
        assert t.relu == int(L['relu']) and abs(t.eps - norm.eps) <= 1e-6 * norm.eps, self.what
        y, res = self.name_at(t.off[1]), self.name_at(t.off[2])
        assert y == L['y'] and res == L['res'] and self.name_at(t.off[3]) in ((None, L['sums']) if frozen else (L['sums'],))   # (eval mode: unread)
        rm0, rv0 = norm.running_mean.clone(), norm.running_var.clone()
        self.nan_fill(y)
        self.run(t)
        C_ = g['Cout']
        z = self.view(L['z']).double().reshape(-1, C_)
        r = self.view(res).double().reshape(-1, C_) if res is not None else None
        K_s = 0 if frozen else self.K_s[L['sums']]          # the fp32 roundings BN_STATS put into these sums
        ref, S, K = bn_apply_ref(z, r, norm.weight.detach()[:C_], norm.bias.detach()[:C_], norm.eps, L['relu'], frozen, rm0[:C_], rv0[:C_], K_s)
        self.note(t.kind, 'y', check_faithful(self.view(y).reshape(-1, C_), ref, S, K, self.what + ' y'))
        if frozen:
            assert torch.equal(norm.running_mean, rm0) and torch.equal(norm.running_var, rv0), '%s: running statistics of an eval-mode BatchNorm written' % self.what
            return
        assert abs(t.momentum - norm.momentum) <= 1e-6
        (wm, Sm, Km), (wv, Sv, Kv) = bn_running_ref(z, rm0, rv0, norm.momentum, K_s)
        self.note(t.kind, 'running stats', check_within(norm.running_mean, wm, Sm, Km, self.what + ' running_mean'))
        self.note(t.kind, 'running stats', check_within(norm.running_var, wv, Sv, Kv, self.what + ' running_var'))
        self.tol.setdefault('running', []).append((norm, Km * U * Sm, Kv * U * Sv))

    # --------------------------------------------------------------- GroupNorm apply and the head
    def op_gn_apply(self, t):
        raw, act = self.name_at(t.off[0]), self.name_at(t.off[1])
        L = self.layer_of[raw]
        assert L['type'] == 'gn' and raw == L['raw'] and act == L['act'] and self.name_at(t.off[3]) == L['stats']
        norm = L['norm']
        assert t.groups == norm.num_groups and abs(t.eps - norm.eps) <= 1e-6 * norm.eps, self.what
        self.nan_fill(act)
        self.run(t)
        x = self.view(raw).reshape(self.N, -1, 128)
        a, a_b, amb = head_activation(x, norm.weight.detach(), norm.bias.detach(), self.view(L['stats']), 16, norm.eps)
        check_amb(amb, self.what)
        got = self.view(act).double().reshape(a.shape)
        bad = (got != a) & (got != a_b)
        assert not bool(bad.any()), '%s: %d elements differ from the exact emulation' % (self.what, int(bad.sum()))
        self.note(t.kind, 'act', 0.0)

    def _final(self, t):
        stage = self.name_at(t.off[4])
        L = self.layer_of[stage]
        g = L['geo']
        lvl = int(re.match(r'h(\d+)fin', L['name']).group(1))
        assert self.plan.level_sizes[lvl] == (g['H'], g['W'])
        assert self.name_at(t.off[0]) == L['raw'] and self.name_at(t.off[3]) == L['stats'], self.what
        assert (t.n_cls, t.n_reg, t.P, t.cls_stride) == (g['n_cls'], g['n_reg'], self.plan.P, self.plan.cls_channels), self.what
        assert t.point_off == self.point_off[lvl], '%s: point_off %d, level %d starts at %d' % (self.what, t.point_off, lvl, self.point_off[lvl])
        norm = L['norm']
        x = self.view(L['raw']).reshape(self.N, -1, 128)
        if norm is not None:
            assert t.groups == 16 and abs(t.eps - norm.eps) <= 1e-6 * norm.eps
            a, a_b, amb = head_activation(x, norm.weight.detach(), norm.bias.detach(), self.view(L['stats']), 16, norm.eps)
            check_amb(amb, self.what)
        else:
            assert t.groups == 0
            a, a_b, _ = head_activation(x, None, None, None, 0, 1e-5)
        no = g['n_cls'] + g['n_reg']
        stg = self.view(stage).double()
        w, scale, shift, bias = stg[:no * 128].view(no, 128), stg[no * 128:no * 128 + no], stg[no * 128 + no:no * 128 + 2 * no], stg[no * 128 + 2 * no:]
        return L, g, self.point_off[lvl], a, a_b, w, scale, shift, bias

    def op_head_final(self, t):
        plan = self.plan
        L, g, po, a, a_b, w, scale, shift, bias = self._final(t)
        cls0, reg0 = plan.cls_out.clone(), plan.reg_out.clone()
        self.run(t)
        HW, nc = g['H'] * g['W'], g['n_cls']
        ref, S, K = head_forward_ref(a, a_b, w, scale, shift)
        sl = slice(po, po + HW)
        for out, before, cols, name in ((plan.cls_out, cls0, slice(0, nc), 'cls'), (plan.reg_out, reg0, slice(nc, nc + g['n_reg']), 'reg')):
            n_out = cols.stop - cols.start
            if n_out:
                self.note(t.kind, name, check_within(out[:, sl, :n_out], ref[..., cols], S[..., cols], K, '%s %s' % (self.what, name)))
                self.out_tol[name][:, sl, :n_out] = K * U * S[..., cols]
            keep = out.clone()
            keep[:, sl, :n_out] = before[:, sl, :n_out]
            assert torch.equal(keep.view(torch.int32), before.view(torch.int32)), '%s: %s written outside its level' % (self.what, name)

    def op_head_final_bwd(self, t):
        plan = self.plan
        L, g, po, a, a_b, w, scale, shift, bias = self._final(t)
        dact, dstage, dscale = self.name_at(t.off[1]), self.name_at(t.off[5]), self.name_at(t.off[6])
        assert dact == L['dact'] and dstage == L['dstage'] and dscale == L['dscale'], self.what
        assert dact not in self.written
        ds0 = self.view(dstage).clone()
        dsc0 = self.view(dscale).clone() if dscale is not None else None
        self.nan_fill(dact)
        self.run(t)
        HW, nc, nr = g['H'] * g['W'], g['n_cls'], g['n_reg']
        no = nc + nr
        up = torch.cat([plan.gcls[:, po:po + HW, :nc], plan.greg[:, po:po + HW, :nr]], -1).double()
        bx, tiles = head_bwd_grid(HW, no, self.N, grid_sms(t.max_ctas, self.sms))
        r = head_backward_ref(a, a_b, up, w, scale, bias, nc, bx, tiles, self.N)
        self.note(t.kind, 'dact', check_faithful(self.view(dact).reshape(a.shape), *r['dact'], what=self.what + ' dact'))
        got = self.view(dstage)
        (rw, Sw, Kw), (rb, Sb, Kb) = r['dW'], r['dbias']
        ref = ds0.double() + torch.cat([rw.reshape(-1), rb])
        # a shared head's staging already holds the other levels' sums: each of the bx * N block atomics rounds a total that includes them
        n_atom = bx * self.N
        tol = torch.cat([Kw * U * Sw.reshape(-1), Kb * U * Sb]) + n_atom * U * ds0.double().abs()
        self.note(t.kind, 'dW dbias', check_within(got, ref, tol / U, 1, self.what + ' dW | dbias'))
        self.tol[dstage] = self.tol.get(dstage, 0) + tol
        if dscale is not None:
            rs, Ss, Ks = r['dscale']
            tol = Ks * U * Ss + n_atom * U * dsc0.double().abs()
            self.note(t.kind, 'dScale', check_within(self.view(dscale), dsc0.double() + rs, tol / U, 1, self.what + ' dScale'))
            self.tol[dscale] = self.tol.get(dscale, 0) + tol
        self.written.add(dact)

    # --------------------------------------------------------------- norm backward
    def _nb(self, t):
        z = self.name_at(t.off[2])
        L = self.layer_of[z]
        norm = L['norm']
        if L['type'] == 'gn':
            assert z == L['raw'] and self.name_at(t.off[0]) == 'd_' + (L['act'] if L['act'] is not None else L['raw'] + '_act')
            assert self.name_at(t.off[3]) == L['stats'] and self.name_at(t.off[1]) is None and t.groups == 16 and t.relu == 1
        else:
            frozen = not getattr(norm, 'training', False)
            assert z == L['z'] and self.name_at(t.off[0]) == 'd_' + L['y'] and self.name_at(t.off[1]) == (L['y'] if L['relu'] else None)
            assert self.name_at(t.off[3]) in ((None, L['sums']) if frozen else (L['sums'],)), self.what      # (eval mode: unread)
            assert t.frozen == int(frozen), '%s: frozen = %d for a BatchNorm in %s mode' % (self.what, t.frozen, 'eval' if frozen else 'train')
            assert t.groups == 0 and t.relu == int(L['relu'])
        assert self.name_at(t.off[4]) == L['name'] + '_bsums' and abs(t.eps - norm.eps) <= 1e-6 * norm.eps, self.what
        return L, norm

    def _nb_ref(self, L, norm, t):
        g = L['geo']
        sms = grid_sms(t.max_ctas, self.sms)
        if L['type'] == 'gn':
            HW = g['H'] * g['W']
            z = self.view(L['raw']).double().reshape(self.N, HW, 16, 8)
            dy = self.view(self.name_at(t.off[0])).double().reshape(self.N, HW, 16, 8)
            r = gn_bwd_ref(z, dy, self.view(L['stats']), norm.weight.detach(), norm.bias.detach(), norm.eps, gn_bwd_blocks(HW * 16, self.N, sms))
            check_amb(r['amb'], self.what)
            return r
        C_ = g['Cout']
        frozen = not getattr(norm, 'training', False)
        z = self.view(L['z']).double().reshape(-1, C_)
        blocks = reduce_blocks(z.numel() // 8, sms)
        return bn_bwd_ref(z, self.view('d_' + L['y']).double().reshape(-1, C_), self.view(L['y']).double().reshape(-1, C_),
                          None if frozen else self.view(L['sums']), norm.weight.detach()[:C_], norm.eps, L['relu'], frozen,
                          norm.running_mean[:C_], norm.running_var[:C_], blocks)

    def op_norm_bwd_reduce(self, t):
        L, norm = self._nb(t)
        bs = L['name'] + '_bsums'
        b0 = self.view(bs).clone()
        self.run(t)
        r = self._nb_ref(L, norm, t)
        got = self.view(bs)
        if L['type'] == 'gn':
            C_ = L['geo']['Cout']
            (rc, Sc, Kc), (rg, Sg, Kg) = r['bsums']
            self.note(t.kind, 'sums', check_within(got[:C_ * 2].view(C_, 2), b0[:C_ * 2].view(C_, 2) + rc, Sc + b0[:C_ * 2].view(C_, 2).abs(), Kc, self.what + ' channel sums'))
            self.note(t.kind, 'sums', check_within(got[C_ * 2:].view(self.N, 16, 2), b0[C_ * 2:].view(self.N, 16, 2) + rg, Sg + b0[C_ * 2:].view(self.N, 16, 2).abs(), Kg,
                                                   self.what + ' group sums'))
            self.tol[bs] = torch.cat([(Kc * U * (Sc + b0[:C_ * 2].view(C_, 2).abs())).reshape(-1),
                                      (Kg * U * (Sg + b0[C_ * 2:].view(self.N, 16, 2).abs())).reshape(-1)])
        else:
            ref, S, K = r['bsums']
            self.note(t.kind, 'sums', check_within(got, b0 + ref, S + b0.abs(), K, self.what + ' sums'))
            self.tol[bs] = K * U * (S + b0.abs())

    def _param_grad(self, ptr, p, out):
        """Where dgamma / dbeta go: the parameter's slice of the flat gradient (one fp32 atomic of the finished sum), nothing for a frozen
        parameter.  -> the slice, or None."""
        plan = self.plan
        if p is None or not p.requires_grad:
            assert not ptr, '%s: %s gradient of a frozen parameter is written' % (self.what, out)
            return None
        sl = self.grad_of(p)
        assert ptr == plan.flat.grad.data_ptr() + 4 * sl.start, '%s: %s pointer' % (self.what, out)
        return sl

    def op_norm_bwd_apply(self, t):
        plan = self.plan
        L, norm = self._nb(t)
        g = L['geo']
        dz, dzu, dres = self.name_at(t.off[5]), self.name_at(t.off[6]), self.name_at(t.off[7])
        if L['type'] == 'gn':
            assert dz == 'd_' + L['raw'] and dzu is None and dres is None
        else:
            assert dz == 'd_' + L['z'], self.what
            need_up = L['conv'].stride[0] == 2 and L['x'] is not None and ('d_' + L['x']) in self.regions
            assert dzu == ('d_' + L['z'] + '_up' if need_up else None), self.what
            if need_up:
                assert (t.upH, t.upW) == (g['H'], g['W']), '%s: upH x upW = %d x %d, the conv input is %d x %d' % (self.what, t.upH, t.upW, g['H'], g['W'])
            want_res = 'd_' + L['res'] if L['res'] is not None and ('d_' + L['res']) in self.regions else None
            assert dres == want_res, self.what
        acc = dres is not None and dres in self.written
        assert t.accumulate == int(acc), '%s: accumulate = %d into %s, expected %d' % (self.what, t.accumulate, dres, acc)
        prev = self.view(dres).clone() if acc else None
        if 'dgamma' in L:           # conv + bias tower: gamma is the constant 1 (its gradient goes to a sink), beta the conv's bias
            assert t.ptr[2] == L['dgamma'].data_ptr(), self.what
            slw, slb = None, self._param_grad(t.ptr[3], L['conv'].bias, 'dbeta')
        else:
            slw, slb = self._param_grad(t.ptr[2], L['norm'].weight, 'dgamma'), self._param_grad(t.ptr[3], L['norm'].bias, 'dbeta')
        g0 = plan.flat.grad.clone()
        for name in (dz, dzu, dres if not acc else None):
            if name is not None:
                self.nan_fill(name)
        self.run(t)
        r = self._nb_ref(L, norm, t)
        C_ = g['Cout']
        if L['type'] == 'gn':
            self.note(t.kind, 'dz', check_faithful(self.view(dz).double().reshape(self.N, -1, 16, 8), *r['dz'], what=self.what + ' dz'))
        else:
            self.note(t.kind, 'dz', check_faithful(self.view(dz).reshape(-1, C_), *r['dz'], what=self.what + ' dz'))
        if dzu is not None:
            up = self.view(dzu)
            assert torch.equal(up[:, ::2, ::2].contiguous().view(torch.int16), self.view(dz).view(torch.int16)), '%s: dz_up placement' % self.what
            mask = torch.ones(up.shape[:3], dtype=torch.bool, device=DEV)
            mask[:, ::2, ::2] = False
            assert bool((up[mask].view(torch.int16) == 0).all()), '%s: dz_up zeros' % self.what
        if dres is not None:
            gm = r['g'].reshape(self.view(dres).shape)
            if acc:
                self.note(t.kind, 'dres', check_faithful(self.view(dres), prev.double() + gm, prev.double().abs() + gm.abs(), 1, self.what + ' dres'))
            else:
                assert torch.equal(self.view(dres).double(), gm), '%s: dres' % self.what
            self.written.add(dres)
        for sl, key in ((slw, 'dgamma'), (slb, 'dbeta')):
            if sl is None:
                continue
            ref, S, K = r[key]
            before = g0[sl].double()
            tol = K * U * S + U * before.abs()
            self.note(t.kind, key, check_within(plan.flat.grad[sl], before + ref, tol / U, 1, '%s %s' % (self.what, key)))
            self.tol_grad[sl] += tol
            self.grad_written.add(id(plan.flat.params[plan.flat.offsets.index(sl.start)]))
        others = torch.ones(plan.flat.numel, dtype=torch.bool, device=DEV)
        for sl in (slw, slb):
            if sl is not None:
                others[sl] = False
        assert torch.equal(plan.flat.grad[others], g0[others]), '%s: gradient written outside dgamma / dbeta' % self.what

    # --------------------------------------------------------------- weight gradients
    def op_wgrad(self, t):
        x, dz, gs = self.name_at(t.off[0]), self.name_at(t.off[1]), self.name_at(t.off[5])
        L = self.layer_of[dz[2:]]
        conv = L['conv']
        assert dz == 'd_' + (L['z'] if L['type'] == 'bn' else L['raw']) and x == L['x'] and gs == self.plan._gstage[id(conv.weight)], self.what
        assert (t.ksize, t.stride, t.Cin, t.Cout) == (conv.kernel_size[0], conv.stride[0], conv.in_channels, conv.out_channels)
        k, ci, co = conv.kernel_size[0], conv.in_channels, conv.out_channels
        n = k * k * ci * co
        st = self._ptr_region(self.base + self.regions[gs], n * 4).view(torch.float32)
        s0 = st.clone()
        self.run(t)
        xd, dzd = self.view(x).double().permute(0, 3, 1, 2), self.view(dz).double().permute(0, 3, 1, 2)
        ref = torch.nn.grad.conv2d_weight(xd, (co, ci, k, k), dzd, stride=conv.stride[0], padding=k // 2)
        S = torch.nn.grad.conv2d_weight(xd.abs(), (co, ci, k, k), dzd.abs(), stride=conv.stride[0], padding=k // 2)
        ref, S = ref.permute(2, 3, 1, 0).reshape(-1), S.permute(2, 3, 1, 0).reshape(-1)      # -> the staging's [tap][ci][co]
        self.note(t.kind, 'dW', check_within(st, s0.double() + ref, S + s0.double().abs(), WGRAD_K, self.what + ' dW'))
        self.tol[gs] = self.tol.get(gs, 0) + WGRAD_K * U * (S + s0.double().abs())

    def op_wgrad_stem(self, t):
        x27, dz, gs = self.name_at(t.off[0]), self.name_at(t.off[1]), self.name_at(t.off[5])
        L = self.layer_of[dz[2:]]
        conv = L['conv']
        assert L['x'] is None and x27 == 'stem_im2col' and gs == self.plan._gstage[id(conv.weight)] and t.impl == nat.WGRAD_UMMA
        co = conv.out_channels
        st = self._ptr_region(self.base + self.regions[gs], 32 * co * 4).view(torch.float32).view(32, co)
        s0 = st.clone()
        self.nan_fill(x27)
        self.run(t)
        xs = _image(self.x)
        cols = F.unfold(xs.double().permute(0, 3, 1, 2), 3, padding=1, stride=2)           # [N][ci * 9 + tap][pixels]
        N, Ho, Wo = self.N, L['geo']['Ho'], L['geo']['Wo']
        cols = cols.view(N, 3, 9, Ho, Wo).permute(0, 3, 4, 2, 1).reshape(N, Ho, Wo, 27)   # -> channel tap * 3 + ci
        got = self.view(x27).double()
        assert torch.equal(got[..., :27], cols) and bool((got[..., 27:] == 0).all()), '%s: im2col' % self.what
        dzd = self.view(dz).double().reshape(-1, co)
        c = cols.reshape(-1, 27)
        ref = torch.cat([c.t() @ dzd, torch.zeros(5, co, dtype=torch.float64, device=DEV)])
        S = torch.cat([c.abs().t() @ dzd.abs(), torch.zeros(5, co, dtype=torch.float64, device=DEV)])
        self.note(t.kind, 'dW', check_within(st, s0.double() + ref, S + s0.double().abs(), WGRAD_K, self.what + ' dW'))
        self.tol[gs] = self.tol.get(gs, 0) + WGRAD_K * U * (S + s0.double().abs()).reshape(-1)

    # --------------------------------------------------------------- the frozen prefix on the inference kernels
    def op_infer(self, t):
        op = self.prefix_ops[self.n_infer]
        self.n_infer += 1
        pre = self.plan._prefix

        def tensor(name, off):
            if name is None:
                assert off < 0
                return None
            sh = pre['emitter']._tensors[name]
            assert off == (self.regions[name] if name in self.regions else self.regions['prefix_scratch'] + pre['scratch'][name]), self.what
            return self.plan.workspace[off:off + sh].view(torch.bfloat16)
        N = self.N
        out = tensor(op['out'], t.off[1])
        cf = op.get('tail_cout') or op['Cout']
        out = out.view(N, op['Ho'], op['Wo'], cf)
        out2 = tensor(op.get('out2'), t.off[3])
        res = tensor(op.get('res'), t.off[2])
        res = res.view(N, op['Ho'], op['Wo'], cf).clone() if res is not None else None
        out.fill_(float('nan'))
        if out2 is not None:
            out2.fill_(float('nan'))
        self.run(t)

        if op['kind'] in (nat.OP_STEM0, nat.OP_STEM4):
            x = _image(self.x)
        else:
            x = tensor(op['inp'], t.off[0]).view(N, op['H'], op['W'], op['Cin'])
        for name, ratio in check_conv_op(op, x, out, out2, res, 'bf16', self.what, self.relu):
            self.note(t.kind, name, ratio)

    # ------------------------------------------------------------------ the executor on the same step
    def executor_matches(self):
        """The same step through lfd_train_plan_run (branches, CUDA graph): the first call runs eagerly and captures, the second replays.
        16-bit regions: at most 1 ulp apart on at most 1e-3 of their elements; fp32 / fp64 accumulations, the flat gradient and the running
        statistics: within twice their bound; cls / reg within twice theirs."""
        plan = self.plan
        ws_ref, grad_ref = plan.workspace.clone(), plan.flat.grad.clone()
        cls_ref, reg_ref = plan.cls_out.clone(), plan.reg_out.clone()
        run_ref = [(m.running_mean.clone(), m.running_var.clone()) for m in self.bn]
        lib = nat.lib()
        for _ in range(2):
            self.restore()
            with torch.cuda.device(plan.device):
                nat.check(lib.lfd_train_plan_run(plan.fwd_handle, nat.ptr(plan._input), plan._fmt, nat.ptr(plan.workspace), 1, nat.stream_ptr()))
                nat.check(lib.lfd_train_plan_run(plan.bwd_handle, nat.ptr(plan._input), plan._fmt, nat.ptr(plan.workspace), 1, nat.stream_ptr()))
            torch.cuda.synchronize()
        flips = {}               # BatchNorm dz -> where the stored output's ReLU mask differs between the two runs
        for L in plan._layers:
            if L['type'] == 'bn' and L['relu'] and ('d_' + L['z']) in self.shapes:
                flips['d_' + L['z']] = (self.view(L['y']) > 0) != (self.view(L['y'], ws_ref) > 0)
        rules = {}
        for name in self.regions:
            o, nb = self.regions[name], plan._sizes[name]
            if name in self.tol and torch.is_tensor(self.tol[name]):        # fp32 / fp64 accumulations: within twice their bound
                tol = self.tol[name].reshape(-1)
                dt = torch.float64 if name.endswith(('_sums', '_bsums', '_gnstats')) else torch.float32
                a_, b_ = (w[o:o + tol.numel() * (8 if dt == torch.float64 else 4)].view(dt).double() for w in (plan.workspace, ws_ref))
                assert bool(((a_ - b_).abs() <= 2 * tol).all()), '%s: the executor differs from the replay' % name
                rules[name] = 'bound'
            elif name in self.shapes and self.shapes[name][0] == torch.bfloat16:   # 16-bit tensors: <= 1 ulp on <= 1e-3 of them
                a_, b_ = self.view(name).double(), self.view(name, ws_ref).double()
                d = (a_ - b_).abs()
                flip = flips.get(name, torch.zeros_like(d, dtype=torch.bool)).reshape(d.shape)
                n_flip = int(flip.sum())
                assert n_flip <= max(1, 1e-4 * d.numel()), '%s: %d ReLU decisions differ between the runs' % (name, n_flip)
                over = (d > ulp16(torch.maximum(a_.abs(), b_.abs()))) & ~flip
                assert not bool(over.any()), '%s: the executor differs from the replay by more than one ulp at %d elements' % (name, int(over.sum()))
                assert int((d > 0).sum()) <= max(1, 1e-3 * d.numel()) + n_flip, '%s: %d elements differ by one ulp' % (name, int((d > 0).sum()))
                rules[name] = 'ulp'
            else:       # packed weights, head staging, the prefix's scratch: deterministic writes, bit for bit
                assert torch.equal(plan.workspace[o:o + nb], ws_ref[o:o + nb]), '%s: the executor differs from the replay' % name
                rules[name] = 'exact'
        assert set(rules) == set(self.regions)
        assert bool(((plan.flat.grad.double() - grad_ref.double()).abs() <= 2 * self.tol_grad).all()), 'flat gradient: the executor differs from the replay'
        for m, (rm, rv) in zip(self.bn, run_ref):
            hit = [x for x in self.tol.get('running', []) if x[0] is m]
            if not hit:
                assert torch.equal(m.running_mean, rm) and torch.equal(m.running_var, rv)
                continue
            _, tm, tv = hit[0]
            assert bool(((m.running_mean.double() - rm.double()).abs() <= 2 * tm).all()) and bool(((m.running_var.double() - rv.double()).abs() <= 2 * tv).all())
        for got, ref, name in ((plan.cls_out, cls_ref, 'cls'), (plan.reg_out, reg_ref, 'reg')):
            d = (got.double() - ref.double()).abs()
            assert bool((d <= 2 * self.out_tol[name]).all()), '%s: the executor differs from the replay' % name


# ---------------------------------------------------------------------------------------------------------------- the cases
def _model(cfg, variant, device=DEV):
    model, _ = synth_model(cfg, cls_bias=-2.0)
    model.to(device).train()
    if variant == 'bn_eval':
        for m in model.modules():
            if isinstance(m, nn.BatchNorm2d):
                m.eval()
    elif variant and variant.startswith('frozen'):
        k = variant[len('frozen'):]
        bb = model._backbone
        bb._frozen_stages = len(bb.stages()) if k == 'all' else int(k)
        model.train()
    elif variant == 'head_branch':
        cls_tower, _, fin_cls, _ = model._head.level_paths(0)
        for conv, norm in cls_tower:
            for p in list(conv.parameters()) + list(norm.parameters()):
                p.requires_grad = False
        for p in fin_cls.parameters():
            p.requires_grad = False
    return model


def _input(fmt, n, h, w, seed=0):
    if fmt == 'f32':
        return synth.synth_input(n, h, w, seed=seed).cuda()
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (n, h, w, 3), generator=g, dtype=torch.uint8).cuda()


# (config, shape, input format, variant): stride-2 layers see odd and even inputs at 186 x 250; WIDERFACE_L at the benchmark's per-image
# 640 x 640; WIDERFACE_S at 656 x 640 runs its frozen stem as STEM4
CASES = [('WIDERFACE_XS', (2, 186, 250), 'f32', None), ('WIDERFACE_S', (2, 186, 250), 'u8', None), ('WIDERFACE_M', (2, 186, 250), 'f32', None),
         ('WIDERFACE_L', (2, 186, 250), 'f32', None), ('TT100K_S', (2, 186, 250), 'f32', None), ('TT100K_L', (1, 186, 250), 'f32', None),
         ('TL_L', (2, 186, 250), 'f32', None), ('TEST_FAST', (2, 186, 250), 'f32', None),
         ('WIDERFACE_L', (2, 640, 640), 'u8', None),
         ('WIDERFACE_XS', (2, 186, 250), 'f32', 'bn_eval'), ('WIDERFACE_L', (2, 186, 250), 'f32', 'frozen1'),
         ('TT100K_L', (1, 186, 250), 'f32', 'frozen2'), ('WIDERFACE_L', (2, 186, 250), 'u8', 'frozenall'),
         ('WIDERFACE_S', (2, 656, 640), 'u8', 'frozen1'), ('WIDERFACE_S', (2, 186, 250), 'f32', 'frozen2'), ('TL_L', (2, 186, 250), 'f32', 'frozen2'),
         ('TT100K_L', (1, 186, 250), 'f32', 'frozenall'), ('TT100K_L', (1, 186, 250), 'f32', 'head_branch')]


@pytest.mark.gpu
@pytest.mark.parametrize('cfg,shape,fmt,variant', CASES, ids=['%s-%dx%dx%d-%s-%s' % (c[0], *c[1], c[2], c[3]) for c in CASES])
def test_every_op_of_the_training_step_matches_fp64(cfg, shape, fmt, variant, timing):
    model = _model(cfg, variant)
    x = _input(fmt, *shape)
    ann = synth.synth_annotations(shape[0], shape[1], shape[2], model._num_classes, seed=3)
    r = Replay(model, x, ann)
    if variant == 'frozen1' and shape == (2, 656, 640):
        assert any(op['kind'] == nat.OP_STEM4 for _, op in r.plan._prefix['ops'])
    r.replay()
    r.executor_matches()
    timing['kinds'] |= {t.kind for arr in (r.plan._fwd_arr, r.plan._bwd_arr) for t in arr}


@pytest.fixture(scope='module')
def timing():
    state = dict(t0=time.time(), kinds=set())
    yield state
    print('\nreplay: %.0f s; largest err / tol per op kind and output:' % (time.time() - state['t0']))
    for k in sorted(WORST):
        print('  %-40s %.3g' % (k, WORST[k]))


def test_the_cases_cover_every_op_kind():
    """Every lfd_top kind occurs in the plans of CASES (host-side planning, no GPU): the replays, which check every op of their plans,
    therefore check every kind."""
    from lfd._train import TrainPlan
    kinds = set()
    for cfg, shape, fmt, variant in CASES:
        model = _model(cfg, variant, device='cpu')
        plan = TrainPlan(model, shape[0], shape[1], shape[2], 'cpu', create_native=False)
        kinds |= {op['kind'] for op in plan.fwd_ops + plan.bwd_ops}
    assert kinds == ALL_KINDS, sorted(KIND_NAMES[k] for k in ALL_KINDS - kinds)


@pytest.mark.gpu
def test_a_config_the_planner_rejects_raises():
    from oracle import lfd_oracle as orc
    model, _ = synth_model('TEST_FASTEST', cls_bias=-2.0)
    model.cuda().train()
    assert {c[0] for c in CASES} | {'TEST_FASTEST'} == set(orc.CONFIGS)
    with pytest.raises(NotImplementedError):
        model.train_plan_for(2, 186, 250, torch.device(DEV))
