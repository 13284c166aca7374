# -*- coding: utf-8 -*-
"""Every op of an inference plan, replayed one at a time on the plan's own reused workspace and checked per element against float64.

The plan is the one model(x) builds (reuse=True): a liveness allocator packs the tensors into a workspace several times smaller than their
sum, and the ops run on up to 8 graph branches.  plan._op_array is replayed in list order through lfd_run_op on plan.workspace, cls_out and
reg_out, after the statistics region is zeroed as the executor zeroes it.  Before each op every tensor it reads (input, residual, GroupNorm
statistics) must still hold, bit for bit, the bytes its producer left -- liveness on the real offsets, and a kernel that writes past its
tensor into a live neighbour fails here -- and everything it writes (outputs, its level's cls / reg points) is NaN-filled, so an element
it never writes fails.  After it, every output element is compared with a float64 reference computed on the GPU from those snapshots:
faithful rounding for STEM0 / CONV and their fused shortcuts (train_op_ref.check_conv_op), the interval train_op_ref.chain_interval
propagates behind the in-kernel 16-bit intermediates (fused tails, STEM4), float64 sums for the fused GroupNorm statistics, the exact
emulation for GN_APPLY and the head activation, and check_within for the head outputs.  The references take their operands from the
modules (op['modules'], tail_modules, ds_modules, s2 / s3_modules, InferencePlan._fold) and the ReLUs from the model's layer records
(train_op_ref.layer_relu), so a wrong field of a record fails.

Then the product run: the workspace and the outputs are poisoned and plan.forward runs the plan (branches, CUDA graph: the first call
captures, the second replays); cls / reg equal the replay bit for bit where they do not depend on a GroupNorm, and within
helpers.close_downstream_of_gn where they do (its fp64 atomics add in another order)."""
import ctypes as C
import time

import numpy as np
import pytest
import torch

import synth
from gpu_ops import DTYPES, assert_gn_stats, stem_operand
from gray_models import gray_pair
from helpers import close_downstream_of_gn, downstream_of_gn, model_of, poison, same_bits
from lfd import _native as nat
from lfd._engine import InferencePlan
from nv12_oracle import nv12_frames
from oracle import lfd_oracle as orc
from train_op_ref import check_amb, check_conv_op, check_within, head_activation, head_forward_ref, layer_relu

DEV = 'cuda'
KIND_NAMES = {nat.OP_STEM0: 'STEM0', nat.OP_CONV: 'CONV', nat.OP_STEM4: 'STEM4', nat.OP_GN_APPLY: 'GN_APPLY', nat.OP_HEAD_FINAL: 'HEAD_FINAL'}
WORST = {}          # largest err / tol per (kind, output) over the replays of a session


class Replay(object):
    """The plan's ops, one at a time, on frames x (cuda; fmt 'f32', 'u8' or 'nv12') -> replay() returns (cls, reg)."""

    def __init__(self, plan, model, x, fmt):
        self.plan, self.model, self.x, self.fmt = plan, model, x, fmt
        self.code = {'f32': nat.INPUT_F32_NCHW, 'u8': nat.INPUT_U8_NHWC, 'nv12': nat.INPUT_U8_NV12}[fmt]
        self.dtype = plan.act_dtype
        self.tdt = DTYPES[self.dtype][0]
        self.ws = plan.workspace
        self.snap = {}            # tensor name -> the bytes its producer left
        self.stats = {}           # byte offset of a GroupNorm statistics slot -> the bytes its conv left
        self.relu = layer_relu(model)

    def note(self, kind, out, ratio):
        key = '%s %s' % (KIND_NAMES[kind], out)
        WORST[key] = max(WORST.get(key, 0.0), ratio)

    def bytes_of(self, off, n):
        assert off >= 0 and off + n <= self.ws.numel(), '%s: bytes [%d, %d) outside the workspace' % (self.what, off, off + n)
        return self.ws[off:off + n]

    def tensor(self, off, n, h, w, c):
        return self.bytes_of(off, 2 * n * h * w * c).view(self.tdt).view(n, h, w, c)

    def read(self, name, off, n, h, w, c):
        """A tensor the op reads: the bytes its producer left, bit for bit (none of it recycled or overwritten since)."""
        t = self.tensor(off, n, h, w, c)
        raw = t.view(torch.uint8).reshape(-1)
        assert raw.numel() == self.snap[name].numel(), '%s: reads %s as %d bytes, its producer wrote %d' % (self.what, name, raw.numel(), self.snap[name].numel())
        bad = raw != self.snap[name]
        assert not bool(bad.any()), '%s: %d bytes of %s changed between its producer and this reader, the first at byte %d of it' % (
            self.what, int(bad.sum()), name, int(bad.nonzero()[0]))
        return t.clone()

    def run(self, o):
        plan = self.plan
        with torch.cuda.device(plan.device):
            nat.check(nat.lib().lfd_run_op(C.byref(o), nat.ptr(self.x), self.code, nat.ptr(self.ws), nat.ptr(plan.cls_out), nat.ptr(plan.reg_out),
                                           plan.P, plan.cls_channels, plan.conv_impl, nat.stream_ptr()))
            torch.cuda.synchronize()

    def replay(self):
        plan = self.plan
        self.ws.fill_(0xff)                       # NaN in both 16-bit types: a read of bytes nobody wrote carries a NaN
        self.ws[:plan.stats_bytes].zero_()        # the executor's memset of the GroupNorm statistics
        plan.cls_out.fill_(float('nan'))
        plan.reg_out.fill_(float('nan'))
        torch.cuda.synchronize()
        for i, (o, op) in enumerate(zip(plan._op_array, plan._ops)):
            self.what = 'op %d (%s -> %s)' % (i, KIND_NAMES[o.kind], op.get('out'))
            {nat.OP_STEM0: self.conv, nat.OP_CONV: self.conv, nat.OP_STEM4: self.conv, nat.OP_GN_APPLY: self.gn_apply,
             nat.OP_HEAD_FINAL: self.head_final}[o.kind](o, op)
        for t, name in ((plan.cls_out, 'cls'), (plan.reg_out, 'reg')):
            assert not bool(torch.isnan(t).any()), '%s points no level wrote' % name
        return plan.cls_out.clone(), plan.reg_out.clone()

    # ------------------------------------------------------------------ ops
    def conv(self, o, op):
        N = o.N
        cf = o.tail_cout or o.Cout
        if o.kind == nat.OP_CONV:
            x = self.read(op['inp'], o.in_off, N, o.H, o.W, o.Cin)
        else:
            assert o.in_off < 0
            x = stem_operand(self.x, self.fmt, self.plan.input_transform, self.dtype)
            assert tuple(x.shape) == (N, o.H, o.W, o.Cin), (self.what, tuple(x.shape))
        res = self.read(op['res'], o.res_off, N, o.Ho, o.Wo, cf) if o.res_off >= 0 else None
        assert (res is None) == (op.get('res') is None), self.what
        gn = o.kind == nat.OP_CONV and o.gn_groups > 0
        if gn:
            st = self.bytes_of(o.stats_off, N * o.gn_groups * 16)
            assert bool((st == 0).all()), '%s: statistics slot not zero before its conv' % self.what
        out = self.tensor(o.out_off, N, o.Ho, o.Wo, cf)
        out.fill_(float('nan'))
        out2 = None
        if o.ds_cout:
            out2 = self.tensor(o.ds_out_off, N, o.Ho, o.Wo, o.ds_cout)
            out2.fill_(float('nan'))
        assert bool(o.ds_cout) == (op.get('out2') is not None), self.what
        self.run(o)
        self.snap[op['out']] = out.view(torch.uint8).reshape(-1).clone()
        if out2 is not None:
            self.snap[op['out2']] = out2.view(torch.uint8).reshape(-1).clone()
        for name, ratio in check_conv_op(op, x, out, out2, res, self.dtype, self.what, self.relu):
            self.note(o.kind, name, ratio)
        if gn:
            self.stats[o.stats_off] = st.clone()
            self.note(o.kind, 'GroupNorm sums', assert_gn_stats(st.view(torch.float64).view(N, o.gn_groups, 2), out, o.gn_groups,
                                                                 self.what + ' GroupNorm sums'))

    def _stats(self, o):
        st = self.bytes_of(o.stats_off, o.N * o.gn_groups * 16)
        assert o.stats_off in self.stats, '%s: reads statistics no conv accumulated' % self.what
        assert torch.equal(st, self.stats[o.stats_off]), '%s: statistics changed between their conv and this reader' % self.what
        return st.view(torch.float64).view(o.N, o.gn_groups, 2).clone()

    def gn_apply(self, o, op):
        tnorm = op['modules'][0]
        x = self.read(op['inp'], o.in_off, o.N, o.H, o.W, o.Cin)
        stats = self._stats(o)
        assert o.gn_groups == tnorm.num_groups and o.Cout == o.Cin == tnorm.num_channels, self.what
        out = self.tensor(o.out_off, o.N, o.Ho, o.Wo, o.Cout)
        out.fill_(float('nan'))
        self.run(o)
        self.snap[op['out']] = out.view(torch.uint8).reshape(-1).clone()
        a, a_b, amb = head_activation(x.reshape(o.N, -1, o.Cin), tnorm.weight.detach(), tnorm.bias.detach(), stats, tnorm.num_groups, tnorm.eps, self.dtype)
        check_amb(amb, self.what)
        got = out.double().reshape(a.shape)
        bad = (got != a) & (got != a_b)
        assert not bool(bad.any()), '%s: %d elements differ from the exact emulation' % (self.what, int(bad.sum()))
        self.note(o.kind, 'act', 0.0)

    def head_final(self, o, op):
        plan = self.plan
        tnorm, convs, scales = op['modules']
        x = self.read(op['inp'], o.in_off, o.N, o.H, o.W, o.Cin).reshape(o.N, -1, o.Cin)
        if tnorm is not None:
            assert o.gn_groups == tnorm.num_groups, self.what
            a, a_b, amb = head_activation(x, tnorm.weight.detach(), tnorm.bias.detach(), self._stats(o), tnorm.num_groups, tnorm.eps, self.dtype)
            check_amb(amb, self.what)
        else:
            assert o.gn_groups == 0 and o.stats_off < 0, self.what
            a, a_b, _ = head_activation(x, None, None, None, 0, 1e-5, self.dtype)
        w = torch.cat([fc.weight.detach().reshape(fc.out_channels, -1).to(self.tdt) for fc in convs]).double().to(DEV)
        scale = torch.cat([torch.full((fc.out_channels,), float(sc), dtype=torch.float32) for fc, sc in zip(convs, scales)])
        shift = torch.cat([(fc.bias.detach().float().cpu() if fc.bias is not None else torch.zeros(fc.out_channels)) * sc for fc, sc in zip(convs, scales)])
        ref, S, K = head_forward_ref(a, a_b, w, scale.to(DEV), shift.to(DEV))
        # the level's points, from the level sizes the model gives (plan.level_offsets: level_geometry)
        l = op['level']
        assert (o.H, o.W) == plan.level_sizes[l], self.what
        po, HW, nc = plan.level_offsets[l], plan.level_sizes[l][0] * plan.level_sizes[l][1], o.n_cls
        assert o.point_off == po, '%s: point_off %d, level %d starts at %d' % (self.what, o.point_off, l, po)
        sl = slice(po, po + HW)
        outs = [(plan.cls_out, slice(0, nc), 'cls'), (plan.reg_out, slice(nc, nc + o.n_reg), 'reg')]
        for out, cols, _ in outs:
            out[:, sl, :cols.stop - cols.start] = float('nan')
        before = [out.clone() for out, _, _ in outs]
        self.run(o)
        for (out, cols, name), b in zip(outs, before):
            n_out = cols.stop - cols.start
            if n_out:
                self.note(o.kind, name, check_within(out[:, sl, :n_out], ref[..., cols], S[..., cols], K, '%s %s' % (self.what, name)))
            keep = out.clone()
            keep[:, sl, :n_out] = b[:, sl, :n_out]
            assert torch.equal(keep.view(torch.int32), b.view(torch.int32)), '%s: %s written outside its level' % (self.what, name)


# ------------------------------------------------------------------------------------------------------------------ the product run
def gn_points(plan):
    """-> bool [P] per output: the points whose values depend on a GroupNorm."""
    tainted = downstream_of_gn(plan)
    masks = {'cls': torch.zeros(plan.P, dtype=torch.bool), 'reg': torch.zeros(plan.P, dtype=torch.bool)}
    for op in plan._ops:
        if op['kind'] == nat.OP_HEAD_FINAL and (op.get('gn_groups') or op['inp'] in tainted):
            sl = slice(op['point_off'], op['point_off'] + op['H'] * op['W'])
            for name, n in (('cls', op['n_cls']), ('reg', op['n_reg'])):
                if n:
                    masks[name][sl] = True
    return masks


def assert_outputs_match(what, plan, got, want):
    """cls / reg of the product run against the replay: bit for bit at the points that do not depend on a GroupNorm, within
    close_downstream_of_gn at those that do."""
    masks = gn_points(plan)
    for g, w, name in zip(got, want, ('cls', 'reg')):
        m = masks[name].to(g.device)
        same_bits(g[:, ~m], w[:, ~m], '%s %s (no GroupNorm upstream)' % (what, name))
        if bool(m.any()):
            close_downstream_of_gn('%s %s' % (what, name), g[:, m], w[:, m])


def product_run(plan, x, fmt):
    """plan.forward twice on poisoned buffers (the first call runs eagerly and captures the CUDA graph, the second replays it)."""
    outs = []
    for _ in range(2):
        poison(plan)
        c, r = plan.forward(x, use_graph=True, frame_format='nv12' if fmt == 'nv12' else None)
        torch.cuda.synchronize()
        outs.append((c.clone(), r.clone()))
    return outs


# ------------------------------------------------------------------------------------------------------------------ the cases
def _model(name, device=DEV):
    if name == 'gray TL_S':
        return gray_pair('TL_S')[0].to(device).eval()
    return model_of(name, device)


def _frames(fmt, n, h, w, channels=3, seed=0):
    g = torch.Generator().manual_seed(seed)
    if fmt == 'f32':
        x = synth.synth_input(n, h, w, seed=seed)[:, :channels].contiguous()
    elif fmt == 'u8':
        x = torch.randint(0, 256, (n, h, w) + ((3,) if channels == 3 else ()), generator=g, dtype=torch.uint8)
    else:
        x = torch.from_numpy(nv12_frames(n, h, w, seed=seed))
    return x.to(DEV)


def _transform(name):
    if name is None:
        return None
    from lfd.data_pipeline.augmentation import BGR2RGB, Compose, input_transform_of, standard_normalize
    return input_transform_of(Compose([BGR2RGB(), standard_normalize]))


NAMES = sorted(orc.CONFIGS) + ['TL_S']
# (model, shape, dtype, frame format, extra): extra = fuse_stem / conv_impl / input transform / side-branch CTA bounds.  Stride-2 layers
# see odd and even inputs at 186 x 250; WIDERFACE_S at 656 x 640 runs STEM4
CASES = ([(n, (2, 186, 250), d, 'f32', None) for n in NAMES for d in ('bf16', 'fp16')]
         + [('WIDERFACE_S', (2, 656, 640), d, 'u8', 'stem4') for d in ('bf16', 'fp16')]
         + [('gray TL_S', (2, 186, 250), 'bf16', 'f32', None), ('gray TL_S', (2, 186, 250), 'fp16', 'u8', None),
            ('TL_L', (2, 186, 250), 'bf16', 'u8', 'rgb-standard'), ('WIDERFACE_S', (2, 186, 250), 'bf16', 'nv12', None),
            ('WIDERFACE_L', (2, 186, 250), 'bf16', 'u8', 'side16'),
            ('TL_S', (2, 186, 250), 'bf16', 'f32', 'simt'), ('gray TL_S', (2, 186, 250), 'bf16', 'f32', 'simt')])


def _plan(name, shape, dtype, extra, device=DEV, create_native=True):
    model = _model(name, device)
    kw = dict(act_dtype=dtype, create_native=create_native)
    if extra == 'stem4':
        kw['fuse_stem'] = True
    elif extra == 'simt':
        kw['conv_impl'] = nat.CONV_SIMT
    elif extra == 'rgb-standard':
        kw['input_transform'] = _transform(extra)
    plan = InferencePlan(model, *shape, torch.device(device), **kw)     # reuse=True, as model(x) builds it
    if extra == 'side16' and create_native:
        plan.apply_side_ctas({b: 16 for b in range(1, len(plan.level_sizes) + 1)})
    return model, plan


@pytest.mark.gpu
@pytest.mark.parametrize('name,shape,dtype,fmt,extra', CASES, ids=['%s-%dx%dx%d-%s-%s-%s' % (c[0].replace(' ', '_'), *c[1], *c[2:]) for c in CASES])
def test_every_op_of_the_inference_plan_matches_fp64(name, shape, dtype, fmt, extra, timing):
    model, plan = _plan(name, shape, dtype, extra)
    assert plan.workspace_bytes < plan.activation_bytes            # tensors share bytes
    if extra == 'stem4':
        assert plan._op_array[0].kind == nat.OP_STEM4
    if extra == 'side16':
        assert all(o.max_ctas == 16 for o in plan._op_array if o.branch > 0)
    x = _frames(fmt, *shape, channels=plan.in_channels, seed=sum(shape))
    want = Replay(plan, model, x, fmt).replay()
    for k, got in enumerate(product_run(plan, x, fmt)):
        assert_outputs_match('%s call %d' % (name, k + 1), plan, got, want)


@pytest.mark.gpu
@pytest.mark.parametrize('name', ['WIDERFACE_S', 'TL_L'])
def test_capacity_plan_below_its_size_matches_the_replayed_exact_plan(name, timing):
    """A reused capacity plan (CUDA graph) of 2 x 400 x 656 on frames of 399 x 655 and 257 x 130: cls / reg equal those of the plan built for
    the frame, replayed op by op, under the GroupNorm rule of the product run."""
    model = _model(name)
    cap = InferencePlan(model, 2, 400, 656, torch.device(DEV))
    for h, w in ((399, 655), (257, 130)):
        x = _frames('u8', 2, h, w, seed=h)
        exact = InferencePlan(model, 2, h, w, torch.device(DEV))
        want = Replay(exact, model, x, 'u8').replay()
        for k, got in enumerate(product_run(cap, x, 'u8')):
            assert cap.frame_P == exact.P
            assert_outputs_match('%s %dx%d call %d' % (name, h, w, k + 1), exact, got, want)


@pytest.fixture(scope='module')
def timing():
    state = dict(t0=time.time())
    yield state
    print('\nreplay: %.0f s; largest err / tol per op kind and output:' % (time.time() - state['t0']))
    for k in sorted(WORST):
        print('  %-40s %.3g' % (k, WORST[k]))


def test_the_cases_reach_every_inference_op_kind_in_both_dtypes():
    """The plans of CASES (host-side planning) hold, in bf16 and in fp16: STEM0, STEM4, CONV with a fused tail, a fused shortcut, a
    residual and GroupNorm statistics, GN_APPLY, and HEAD_FINAL with and without a GroupNorm; and every config of the deleted per-layer
    tests (every config, TL_S and the gray TL_S, on the wgmma kernels and the SIMT cross-check for TL_S)."""
    seen = set()
    for name, shape, dtype, fmt, extra in CASES:
        _, plan = _plan(name, shape, dtype, extra, device='cpu', create_native=False)
        for o in plan._op_array:
            feats = {KIND_NAMES[o.kind]}
            if o.kind == nat.OP_CONV:
                feats |= {'CONV tail'} if o.tail_cout else set()
                feats |= {'CONV shortcut'} if o.ds_cout else set()
                feats |= {'CONV residual'} if o.res_off >= 0 else set()
                feats |= {'CONV GroupNorm statistics'} if o.gn_groups else set()
            if o.kind == nat.OP_HEAD_FINAL:
                feats = {'HEAD_FINAL norm' if o.gn_groups else 'HEAD_FINAL no norm'}
            seen |= {(f, dtype) for f in feats}
    want = {'STEM0', 'STEM4', 'CONV', 'CONV tail', 'CONV shortcut', 'CONV residual', 'CONV GroupNorm statistics', 'GN_APPLY', 'HEAD_FINAL norm',
            'HEAD_FINAL no norm'}
    want = {(f, d) for f in want for d in ('bf16', 'fp16')}
    assert seen == want, sorted(want - seen)
    umma = {c[0] for c in CASES if c[4] != 'simt'}
    assert umma >= set(orc.CONFIGS) | {'TL_S', 'gray TL_S'} and {c[0] for c in CASES if c[4] == 'simt'} == {'TL_S', 'gray TL_S'}
    assert np.all([any(c[0] == n and c[2] == d for c in CASES) for n in NAMES for d in ('bf16', 'fp16')])
