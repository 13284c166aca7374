# -*- coding: utf-8 -*-
"""CPU tests: the C-ABI library loads and exports every declared symbol; host-side planning (op list, weight packing,
workspace liveness) is sound; entry points fail loudly without a GPU (there is no CPU fallback)."""
import ctypes as C
import os
import re

import pytest
import torch

from helpers import synth_model
from lfd import _native as nat
from lfd._engine import InferencePlan, pack_conv_weight, _Arena

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    hdr = open(os.path.join(ROOT, 'include', 'lfd_b200.h')).read()
    hdr = re.sub(r'/\*.*?\*/', '', hdr, flags=re.S)
    declared = set(re.findall(r'\b(lfd_[a-z0-9_]+)\s*\(', hdr))
    assert declared == set(nat.SYMBOLS), declared ^ set(nat.SYMBOLS)
    lib = nat.lib()
    for name in declared:
        assert hasattr(lib, name)
    assert lib.lfd_abi_version() == 5


def test_conv_query_is_host_only_and_rejects_unsupported():
    q = nat.conv_query(8, 90, 160, 64, 90, 160, 64, 3, 1)
    assert q['cc'] == 64 and q['weights_resident'] == 1 and q['stages'] >= 3 and q['num_tiles'] == 8 * 20 * 6
    q = nat.conv_query(8, 12, 20, 128, 12, 20, 128, 3, 1)      # 3x3x128x128 weights do not fit: streamed per stage
    assert q['weights_resident'] == 0 and q['stages'] >= 2 and q['smem_bytes'] <= 227 * 1024
    q = nat.conv_query(8, 360, 640, 64, 180, 320, 64, 3, 2)
    assert q['smem_bytes'] <= 227 * 1024 and q['stages'] >= 2
    with pytest.raises(nat.LfdError):
        nat.conv_query(1, 8, 8, 24, 8, 8, 64, 3, 1)            # Cin not a multiple of 16
    with pytest.raises(nat.LfdError):
        nat.conv_query(1, 8, 8, 64, 8, 8, 64, 5, 1)


@pytest.mark.skipif(torch.cuda.is_available(), reason='checks the no-GPU failure mode')
def test_entry_points_fail_loudly_without_gpu():
    lib = nat.lib()
    op = nat.Op()
    op.kind, op.N, op.H, op.W, op.Cin, op.Ho, op.Wo, op.Cout = nat.OP_GN_APPLY, 1, 4, 4, 128, 4, 4, 128
    op.gn_groups = 16
    h = C.c_void_p()
    rc = lib.lfd_plan_create(C.byref(op), 1, 1, 16, 1, 0, 256, 4096, 0, C.byref(h))
    assert rc == 2 and b'no CUDA device' in lib.lfd_last_error()
    rc = lib.lfd_nms(None, 3, 0.5, None, None, C.c_void_p(1), None)
    assert rc != 0
    model, _ = synth_model('WIDERFACE_XS')
    with pytest.raises(RuntimeError):
        model(torch.zeros(1, 3, 64, 64))


def test_pack_conv_weight_layout():
    cout, cin, k, cc = 32, 64, 3, 32
    w = torch.arange(cout * cin * k * k, dtype=torch.float32).reshape(cout, cin, k, k) % 251
    p = pack_conv_weight(w, cc).float()
    assert tuple(p.shape) == (cin // cc, k * k, cc // 8, cout, 8)
    for (c, tap, kc, n, j) in [(0, 0, 0, 0, 0), (1, 4, 3, 17, 5), (1, 8, 2, 31, 7), (0, 5, 1, 9, 3)]:
        ci = c * cc + kc * 8 + j
        assert p[c, tap, kc, n, j] == w[n, ci, tap // 3, tap % 3]


def test_arena_reuses_and_coalesces():
    a = _Arena(base=512)
    o1, o2, o3 = a.alloc(1000), a.alloc(3000), a.alloc(100)
    assert o1 == 512 and o2 == 512 + 1024 and o3 == o2 + 3072
    a.release(o1, 1000)
    a.release(o2, 3000)
    assert a.alloc(4000) == 512          # coalesced block reused
    assert a.alloc(10) == o3 + 256


# stem 1x1 convs are fused tails, the 4 shortcut convs are fused into their block's first conv; merged heads: the neck conv and the first
# tower conv of every level run as one kernel (5 levels: 5 + 10 convs -> 10)
@pytest.mark.parametrize('name,n_conv', [('WIDERFACE_S', 1 + 2 * 11 + 0 + 10), ('TT100K_L', 0 + 2 * 12 + 0 + 4 + 16)])
def test_planner_builds_expected_graph(name, n_conv):
    model, _ = synth_model(name)
    plan = InferencePlan(model, 2, 184, 248, torch.device('cpu'), create_native=False)
    rows = plan.describe()
    kinds = [r['kind'] for r in rows]
    assert kinds[0] == 'stem0' and kinds.count('stem0') == 1 and rows[0]['tail_cout'] == 64
    assert kinds.count('conv') == n_conv
    levels_fused = [r for r in rows if r['kind'] == 'conv' and r['ksize'] == 1 and r['tail_cout'] == 128 and r['Cout'] == 128]
    assert len(levels_fused) == (len(plan.level_sizes) if name.startswith('WIDERFACE') else 0)
    assert len([r for r in rows if r['ds_cout']]) == 4
    levels = len(plan.level_sizes)
    merged = name.startswith('WIDERFACE')
    assert kinds.count('head_final') == (levels if merged else 2 * levels)
    assert kinds.count('gn_apply') == (levels if merged else 2 * levels)
    # (the workspace placement and the ordering of every overlap: test_inference_plans_order_every_overlap)
    # branches: the per-level neck + head chains, and the shortcut convs on branch 7 where they cannot be fused into the block's first conv
    ops = plan._ops
    fused_sc = [o for o in ops if o.get('ds_cout')]
    branches = sorted(set(plan.tensor_branch.values()))
    assert branches == list(range(len(plan.level_sizes) + 1)) + ([] if fused_sc else [7])
    assert all(o['ksize'] == 3 and o['stride'] == 2 and o.get('out2') in plan.offsets for o in fused_sc)
    # shared = the level taps + per stage the block input read by the shortcut branch and the shortcut's output
    n_short = len([o for o in ops if o['branch'] == 7])
    assert n_short > 0 or fused_sc
    taps_and_inputs = set(o['inp'] for o in ops if o['branch'] == 7) | set(o['out'] for o in ops if o['branch'] == 7)
    assert plan.shared_tensors >= taps_and_inputs
    assert len(plan.shared_tensors) <= len(plan.level_sizes) + 2 * n_short
    # mid-graph dependencies: every shortcut conv waits for the main stream, and exactly one main-stream conv per shortcut waits for it
    assert all(o.get('wait_mask', 0) == 1 for o in ops if o['branch'] == 7)
    waiters = [o for o in ops if o.get('wait_mask', 0) == 1 << 7]
    assert len(waiters) == n_short and all(o['branch'] == 0 and o['res'] is not None for o in waiters)


@pytest.mark.parametrize('mode,n_fused', [('fast', 4), ('faster', 4), ('fastest', 0)])
def test_planner_accepts_every_block_mode(mode, n_fused):
    """SURVEY 8 row a4: FastBlock / FastestBlock are not used by any shipped config; the layer planner nevertheless builds a
    valid plan for them (same kernels: 3x3 and 1x1 convs).  FastestBlock's first conv has C/2 outputs, so its shortcut conv
    cannot ride on it and takes the auxiliary branch instead.  (Host logic only: the oracle restates the shipped configs.)"""
    from lfd.model.backbone import LFDResNet
    from lfd.model.neck import SimpleNeck
    from lfd.model.head import LFDHead
    from lfd.model.losses import FocalLoss, IoULoss
    from lfd.model import LFD
    bb = LFDResNet(block_mode=mode, stem_mode='fast', body_mode=None, input_channels=3, stem_channels=64, body_architecture=[2, 1, 1, 1],
                   body_channels=[64, 64, 64, 128], out_indices=((0, 1), (1, 0), (2, 0), (3, 0)), frozen_stages=-1,
                   activation_cfg=dict(type='ReLU', inplace=True), norm_cfg=dict(type='BatchNorm2d'), init_with_weight_file=None, norm_eval=False)
    neck = SimpleNeck(num_neck_channels=128, num_input_channels_list=bb.num_output_channels_list,
                      num_input_strides_list=bb.num_output_strides_list, norm_cfg=dict(type='BatchNorm2d'),
                      activation_cfg=dict(type='ReLU', inplace=True))
    head = LFDHead(num_classes=1, num_heads=4, num_input_channels=128, num_head_channels=128, num_conv_layers=2,
                   activation_cfg=dict(type='ReLU', inplace=True), norm_cfg=dict(type='GroupNorm', num_groups=16), share_head_flag=True,
                   merge_path_flag=True, classification_loss_type='FocalLoss', regression_loss_type='IoULoss')
    model = LFD(backbone=bb, neck=neck, head=head, num_classes=1, regression_ranges=((0, 16), (16, 32), (32, 64), (64, 128)),
                gray_range_factors=(0.9, 1.1), range_assign_mode='dist', point_strides=neck.num_output_strides_list,
                classification_loss_func=FocalLoss(), regression_loss_func=IoULoss(), distance_to_bbox_mode='sigmoid')
    plan = InferencePlan(model, 2, 184, 248, torch.device('cpu'), create_native=False)
    rows = plan.describe()
    assert sum(1 for r in rows if r['ds_cout']) == n_fused
    assert sum(1 for r in rows if r['kind'] == 'head_final') == 4
    per_block = {'fast': 3, 'faster': 2, 'fastest': 2}[mode]
    n_blocks = 5
    n_short = 4 - n_fused
    assert sum(1 for r in rows if r['kind'] == 'conv') == n_blocks * per_block + n_short + 2 * 4   # + (neck + first tower conv, one kernel) + second tower conv
    for o in plan._ops:
        if o.get('wait_mask') == 1 << 7:
            assert o['res'] is not None and o['branch'] == 0


def test_build_guard_rejects_large_stack_frames():
    """build.py fails the build when a conv_umma_kernel instantiation has a large stack frame (a role lambda whose closure
    landed in local memory made the stem kernel 2.5x slower, see conv_umma.cu LFD_LAMBDA_INLINE)."""
    import importlib.util
    spec = importlib.util.spec_from_file_location('lfd_build', os.path.join(ROOT, 'lfd-a-light-and-fast-detector_b200', 'build.py'))
    b = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(b)
    ok = 'ptxas info    : Function properties for _ZN3lfd16conv_umma_kernelILi4ELi4EEEvNS_14UmmaConvParamsE\n    16 bytes stack frame, 12 bytes spill stores, 24 bytes spill loads\n'
    b._check_stack_frames(ok)
    bad = ok.replace('16 bytes stack frame', '232 bytes stack frame')
    with pytest.raises(RuntimeError):
        b._check_stack_frames(bad)
    b._check_stack_frames(bad.replace('conv_umma_kernel', 'some_other_kernel'))


@pytest.mark.parametrize('name', ['WIDERFACE_L', 'TT100K_S', 'TL_L', 'TEST_FAST'])
def test_training_plan_level_chains_order_every_conflict(name):
    """The training planner puts every level's neck + head chain on its own branch (side stream) and derives the wait masks from the
    read / write / accumulate role of each operand.  Replay the fork / wait protocol of lfd_train_plan_run with vector clocks and check
    that every pair of ops that conflict on workspace bytes (write vs anything, accumulate vs read) is ordered, and that no read bytes are
    overwritten before their reader (plan_order.py)."""
    from lfd._train import TrainPlan
    from plan_order import check_training_ops
    model, _ = synth_model(name)
    model.train()
    plan = TrainPlan(model, 2, 128, 160, torch.device('cpu'), create_native=False)
    for which, ops in (('fwd', plan.fwd_ops), ('bwd', plan.bwd_ops)):
        branches = sorted({op.get('branch', 0) for op in ops})
        assert branches[0] == 0 and len(branches) == 1 + len(plan.level_sizes) and branches[-1] < nat.MAX_BRANCHES
        n_pairs = check_training_ops(plan, ops, (name, which))
        if which == 'bwd':
            assert n_pairs >= len(plan.level_sizes)                  # at least the taps' gradients: level chain writes, backbone accumulates
    # the backward starts every level chain before the backbone
    first_main = next(i for i, op in enumerate(plan.bwd_ops) if op.get('branch', 0) == 0 and op['kind'] not in (nat.TOP_ZERO,))
    assert all(op.get('branch', 0) == 0 for op in plan.bwd_ops[first_main:])


def test_plans_do_not_depend_on_the_environment(monkeypatch):
    """The planners and the library read no environment variable that picks a path inside a plan: with every former A/B switch set,
    the inference and training plans are the ones a clean environment gives (op fields, branches, wait masks, offsets, workspace size)."""
    import tl_s
    from lfd._train import TrainPlan
    cpu = torch.device('cpu')
    wf_s, tl = synth_model('WIDERFACE_S')[0], tl_s.synth_model()[0]
    wf_l, wf_l_frozen = synth_model('WIDERFACE_L')[0], synth_model('WIDERFACE_L')[0]
    wf_l_frozen._backbone._frozen_stages = 1
    wf_l.train(), wf_l_frozen.train()

    def plans():        # everything but pointers: the op dicts, the tensor offsets and the workspace size of each plan
        out =[InferencePlan(m, n, h, w, cpu, create_native=False) for m, n, h, w in
               ((wf_s, 2, 184, 248), (wf_s, 8, 720, 1280), (tl, 2, 184, 248))]       # WIDERFACE_S below and above the STEM4 gate
        out = [(p._ops, p.offsets, p.workspace_bytes) for p in out]
        for m in (wf_l, wf_l_frozen):
            p = TrainPlan(m, 2, 128, 160, cpu, create_native=False)
            out.append(([{k: v for k, v in op.items() if k != 'ptr'} for op in p.fwd_ops + p.bwd_ops], p._off, p.workspace_bytes))
        return out

    clean = plans()
    assert clean[0][0][0]['kind'] == nat.OP_STEM0 and clean[1][0][0]['kind'] == nat.OP_STEM4
    for name in ('NO_BRANCHES', 'NO_AUX', 'NO_TAIL', 'NO_FUSED_SHORTCUT', 'NO_STEM_FUSION', 'NO_NECK_TAIL', 'NO_REUSE', 'NO_PDL'):
        monkeypatch.setenv('LFD_B200_' + name, '1')
    monkeypatch.setenv('LFD_B200_TRAIN_BRANCHES', '0')
    monkeypatch.setenv('LFD_B200_GRAPH_PRIO', '0')
    monkeypatch.setenv('LFD_B200_FORCE_CC', '16')
    assert plans() == clean


def test_side_branch_cta_bounds_touch_only_side_branch_ops():
    """InferencePlan._set_side_ctas (what autotune / apply_side_ctas write into the op array): every op of a side branch gets its branch's
    bound (convs: persistent CTAs; GN_APPLY / HEAD_FINAL: the SM count their grids are sized from), main-stream ops stay unbounded."""
    model, _ = synth_model('WIDERFACE_S')
    plan = InferencePlan(model, 2, 184, 248, torch.device('cpu'), create_native=False)
    caps = {b: 16 * b for b in range(1, len(plan.level_sizes) + 1)}
    plan._set_side_ctas(caps)
    seen = set()
    for o, op in zip(plan._op_array, plan._ops):
        if op['branch'] == 0:
            assert o.max_ctas == 0
        else:
            assert o.max_ctas == caps[op['branch']]
            seen.add(op['kind'])
    assert seen == {nat.OP_CONV, nat.OP_GN_APPLY, nat.OP_HEAD_FINAL}
    plan._set_side_ctas({})
    assert all(o.max_ctas == 0 for o in plan._op_array)


def test_tune_branch_bounds_descent(monkeypatch):
    """The coordinate descent behind InferencePlan.autotune / TrainPlan.autotune, on a table of times and a fake clock (one second per
    measurement): branches in decreasing work, a bound kept only below 0.995x the best time so far, at most max_branches branches, no
    trial after the budget, and the log starts with the unbounded time."""
    import types
    import lfd._engine as eng
    clock = [0.0]
    monkeypatch.setattr(eng, 'time', types.SimpleNamespace(time=lambda: clock[0]))
    # kept: 99.0 < 0.995 x 100, 97.0, 90.0; marginal gains below 0.995x the best are dropped: 98.7 vs 99.0, 89.8 vs 90.0
    table = {(): 100.0, ((2, 64),): 99.0, ((2, 32),): 98.7, ((2, 64), (3, 64)): 97.0, ((2, 64), (3, 32)): 90.0,
             ((1, 64), (2, 64), (3, 32)): 95.0, ((1, 32), (2, 64), (3, 32)): 89.8}

    def measure(caps):
        clock[0] += 1.0
        return table.get(tuple(sorted((b, c) for b, c in caps.items() if c)), 1000.0)

    work = {1: 10, 2: 30, 3: 20}
    caps, log = eng.tune_branch_bounds(work, measure, (64, 32), 100.0)
    assert caps == {1: 0, 2: 64, 3: 32} and log[0] == ('all SMs', 100.0)
    assert log[1:] == [('branch %d <= %d CTAs' % (b, c), t) for b, c, t in [(2, 64, 99.0), (2, 32, 98.7), (3, 64, 97.0), (3, 32, 90.0),
                                                                            (1, 64, 95.0), (1, 32, 89.8)]]
    caps, log = eng.tune_branch_bounds(work, measure, (64, 32), 100.0, max_branches=2)
    assert caps == {1: 0, 2: 64, 3: 32} and len(log) == 5 and not any(l.startswith('branch 1 ') for l, _ in log)
    clock[0] = 0.0
    caps, log = eng.tune_branch_bounds(work, measure, (64, 32), 2.5)       # trials start at t = 1 and 2 only
    assert caps == {1: 0, 2: 64, 3: 0} and [l for l, _ in log] == ['all SMs', 'branch 2 <= 64 CTAs', 'branch 2 <= 32 CTAs']


def _inference_plans():
    """Every config, TL_S and the gray TL_S, at a small, an odd and the 8 x 720 x 1280 shape (WIDERFACE_S there plans a STEM4 op), with the
    fused stem forced on and off and on the SIMT cross-check (its shortcut convs run on branch 7)."""
    import tl_s
    from gray_models import gray_pair
    from oracle import lfd_oracle as orc
    models = [(name, synth_model(name)[0]) for name in sorted(orc.CONFIGS)] + [('TL_S', tl_s.synth_model()[0]), ('gray TL_S', gray_pair('TL_S')[0])]
    for name, model in models:
        # (below the STEM4 gate fuse_stem=False plans what the default plans; at 8 x 720 x 1280 the default fuses a 'faster' stem)
        for shape, variants in (((2, 184, 248), (dict(), dict(fuse_stem=True))), ((2, 186, 250), (dict(), dict(fuse_stem=True), dict(conv_impl=nat.CONV_SIMT))),
                                ((8, 720, 1280), (dict(), dict(fuse_stem=False)))):
            for kw in variants:
                yield '%s %s %s' % (name, shape, kw), model, InferencePlan(model, *shape, torch.device('cpu'), create_native=False, **kw)


def test_inference_plans_order_every_overlap():
    """plan_order.check_inference_plan on every plan of _inference_plans: the workspace bytes of every op record inside the workspace and
    aligned, every cross-branch overlap ordered by the executor's fork / wait rules, no bytes overwritten between their producer and a
    reader, disjoint GroupNorm statistics slots read from their producer, and the head's point ranges as level_geometry lays them out."""
    from plan_order import check_inference_plan
    seen_stem4 = False
    for what, model, plan in _inference_plans():
        n_pairs = check_inference_plan(plan, model, what)
        if len({o.branch for o in plan._op_array}) > 1:
            assert n_pairs > 0, what
        print('%-60s %3d ordered cross-branch overlapping pairs' % (what, n_pairs))
        seen_stem4 |= plan._op_array[0].kind == nat.OP_STEM4
        if what.startswith('WIDERFACE_S (2, 184, 248) {}'):
            caps = {b: 16 for b in range(1, len(plan.level_sizes) + 1)}
            plan._set_side_ctas(caps)
            assert check_inference_plan(plan, model, what + ' side CTAs') == n_pairs
    assert seen_stem4
