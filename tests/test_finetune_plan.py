# -*- coding: utf-8 -*-
"""Host-side planning of fine-tuning steps (frozen backbone stages, frozen parameters): the training planner runs the frozen
backbone prefix on the inference plan's ops and packing, keeps only the tensors the trainable part reads, and emits backward ops
only for what reaches a trainable parameter.  No GPU needed (create_native=False)."""
import pytest
import torch

import lfd._native as nat
from helpers import finetune_model, synth_model
from lfd._engine import InferencePlan
from lfd._train import TrainPlan, flat_parameters
from plan_order import check_training_ops

CPU = torch.device('cpu')
CASES = [(cfg, k) for cfg in ('WIDERFACE_L', 'WIDERFACE_S', 'TT100K_L', 'TL_L') for k in (1, 2, 'all')]


def freeze_head_branch(model):
    """Freeze one branch of the head by hand: the classification tower (or the merged tower) and the classification final conv."""
    cls_tower, _, fin_cls, _ = model._head.level_paths(0)
    for conv, norm in cls_tower:
        for p in list(conv.parameters()) + (list(norm.parameters()) if norm is not None else []):
            p.requires_grad = False
    for p in fin_cls.parameters():
        p.requires_grad = False
    return [p for p in model.parameters() if not p.requires_grad]


def _prefix_names(plan):
    return {op[k] for _, op in plan._prefix['ops'] for k in ('out', 'out2') if op.get(k) is not None}


def _weights(op, f32, b16):
    """The folded, packed operands an inference op points at (16-bit bit patterns and fp32 shifts)."""
    out = []
    cout, cin, k = op['Cout'], op['Cin'], op.get('ksize', 1)
    nw = 3 * 2 * cout * 8 if op['kind'] in (nat.OP_STEM0, nat.OP_STEM4) else cout * cin * k * k
    out += [b16[op['w_bf16']:op['w_bf16'] + nw], f32[op['shift']:op['shift'] + cout]]
    if op.get('tail_cout'):
        out += [b16[op['tail_w']:op['tail_w'] + cout * op['tail_cout']], f32[op['tail_shift']:op['tail_shift'] + op['tail_cout']]]
    if op.get('ds_cout'):
        out += [b16[op['ds_w']:op['ds_w'] + cin * op['ds_cout']], f32[op['ds_shift']:op['ds_shift'] + op['ds_cout']]]
    if op['kind'] == nat.OP_STEM4:
        out += [b16[op['s2_w']:op['s2_w'] + 9 * 64 * 64], f32[op['s2_shift']:op['s2_shift'] + 64],
                b16[op['s3_w']:op['s3_w'] + 64 * 64], f32[op['s3_shift']:op['s3_shift'] + 64]]
    return out


def _check_plan(plan, model, frozen_ids):
    pre_names = _prefix_names(plan) if plan._prefix is not None else set()
    kept = set(getattr(plan, 'prefix_outputs', {}))
    # the backward touches no prefix tensor but the taps / boundary it reads, and forms no gradient of any prefix tensor
    for op in plan.bwd_ops:
        for v in op.get('off', {}).values():
            if not isinstance(v, str):
                continue
            assert v != 'prefix_scratch' and (v not in pre_names or v in kept), (op['kind'], v)
            for n in pre_names:
                assert not v.startswith('d_' + n), (op['kind'], v)
    # no weight gradient (nor its scatter into .grad) for a frozen parameter; every trainable conv weight gets one
    stage_of = {name: key for key, name in plan._gstage.items()}
    for op in plan.bwd_ops:
        if op['kind'] in (nat.TOP_WGRAD, nat.TOP_WGRAD_STEM):
            assert stage_of[op['off'][5]] not in frozen_ids
    convs = [m for m in model.modules() if isinstance(m, torch.nn.Conv2d) and m.weight.requires_grad and m.out_channels >= 16
             and m.weight.shape[2] in (1, 3) and m not in _final_convs(model)]
    for c in convs:
        assert id(c.weight) in plan._gstage, c
    frozen_slots = {plan.flat.grad_ptr(p) for p in plan.flat.params if id(p) in frozen_ids}
    assert not any(d.dst in frozen_slots for d in plan._unpack.items)
    for op in plan.bwd_ops:
        for v in op.get('ptr', {}).values():
            assert not (isinstance(v, tuple) and v[0] == 'grad' and id(v[1]) in frozen_ids)
    # no backward op on a frozen-prefix layer, and the plan still orders every overlap, the recycled prefix scratch included
    assert check_training_ops(plan, plan.fwd_ops, 'fwd') >= 0
    assert check_training_ops(plan, plan.bwd_ops, 'bwd') >= 0


def _final_convs(model):
    out = set()
    for l in range(model._head._num_heads):
        _, _, fc, fr = model._head.level_paths(l)
        out |= {fc, fr}
    return out


@pytest.mark.parametrize('cfg,frozen_stages', CASES)
def test_frozen_stage_plan(cfg, frozen_stages, shape=(2, 128, 160)):
    model = finetune_model(cfg, frozen_stages, -1.0)
    frozen_ids = {id(p) for p in model.parameters() if not p.requires_grad}
    assert frozen_ids
    plan = TrainPlan(model, *shape, CPU, create_native=False)
    assert plan._prefix is not None
    n_units = 1 + sum(len(s) for s in model._backbone.stages()[:model._backbone._frozen_stages])
    assert len(plan._prefix['modules']) == n_units
    _check_plan(plan, model, frozen_ids)
    # the prefix runs on the inference ops (no BatchNorm statistics, no stored z) and only those
    infer = [op for op in plan.fwd_ops if op['kind'] == nat.TOP_INFER]
    assert len(infer) == len(plan._prefix['ops'])
    assert all(op.get('branch', 0) == 0 for op in infer)
    prefix_mods = {id(m) for u in plan._prefix['modules'] for m in u.modules()}
    assert not any(id(L.get('conv')) in prefix_mods for L in plan._layers)
    # workspace: smaller than the full training step's
    full_model, _ = synth_model(cfg)
    full_model.train()
    full = TrainPlan(full_model, *shape, CPU, create_native=False)
    print('%s frozen_stages=%s: workspace %.1f MB (all stages trainable: %.1f MB), %d / %d forward / backward ops (%d / %d)'
          % (cfg, frozen_stages, plan.workspace_bytes / 2 ** 20, full.workspace_bytes / 2 ** 20, len(plan.fwd_ops), len(plan.bwd_ops),
             len(full.fwd_ops), len(full.bwd_ops)))
    assert plan.workspace_bytes < full.workspace_bytes
    assert len(plan.bwd_ops) < len(full.bwd_ops)


@pytest.mark.parametrize('cfg,frozen_stages,shape', [(c, k, (2, 128, 160)) for c, k in CASES] + [('WIDERFACE_S', 1, (2, 656, 640)),
                                                                                                   ('WIDERFACE_L', 'all', (1, 186, 252))])
def test_prefix_ops_are_the_inference_plans(cfg, frozen_stages, shape):
    """Kinds, fusions (tails, fused shortcut, the four-conv stem where the inference plan picks it) and packed operand bytes of every
    prefix op equal those of the inference plan's op producing the same tensor."""
    model = finetune_model(cfg, frozen_stages, -1.0)
    plan = TrainPlan(model, *shape, CPU, create_native=False)
    model.eval()
    ref = InferencePlan(model, *shape, CPU, create_native=False)
    by_out = {op['out']: op for op in ref._ops if op.get('out') is not None}
    f32, b16 = plan._prefix['f32'], plan._prefix['b16']
    kinds = set()
    for top, op in plan._prefix['ops']:
        r = by_out[op['out']]
        kinds.add(op['kind'])
        for k in ('kind', 'H', 'W', 'Cin', 'Ho', 'Wo', 'Cout', 'ksize', 'stride', 'relu', 'cc', 'tail_cout', 'tail_relu', 'ds_cout', 'inp', 'res', 'out2',
                  's2_relu', 's3_relu'):
            assert op.get(k) == r.get(k), (op['out'], k, op.get(k), r.get(k))
        for a, b in zip(_weights(op, f32, b16), _weights(r, ref.params_f32, ref.params_bf16)):
            assert torch.equal(a, b), op['out']
        assert top['off'][1] == op['out'] and top['off'][0] == op.get('inp')
    if shape == (2, 656, 640):
        assert nat.OP_STEM4 in kinds
    # the descriptors handed to the native plan point at the staged operands
    for i, (top, op) in enumerate(plan._prefix['ops']):
        o = plan._prefix['arr'][i]
        assert o.kind == op['kind'] and o.weight == b16.data_ptr() + 2 * op['w_bf16'] and o.dtype == nat.DTYPE_BF16


@pytest.mark.parametrize('cfg', ['WIDERFACE_L', 'TT100K_L', 'TL_L'])
def test_hand_frozen_head_branch(cfg):
    """Parameters frozen by hand outside the backbone lose their own gradient ops only: the gradient still flows through them into the
    neck and the backbone, and there is no frozen prefix."""
    model, _ = synth_model(cfg)
    model.train()
    frozen = freeze_head_branch(model)
    frozen_ids = {id(p) for p in frozen}
    plan = TrainPlan(model, 2, 128, 160, CPU, create_native=False)
    assert plan._prefix is None
    _check_plan(plan, model, frozen_ids)
    stem_conv = model._backbone.stem_layers()[0][0]
    assert id(stem_conv.weight) in plan._gstage                # the backbone still trains
    cls_tower, _, fin_cls, _ = model._head.level_paths(0)
    for conv, _ in cls_tower:
        assert id(conv.weight) not in plan._gstage
    full_model, _ = synth_model(cfg)
    full_model.train()
    full = TrainPlan(full_model, 2, 128, 160, CPU, create_native=False)
    n = lambda p, k: sum(1 for op in p.bwd_ops if op['kind'] == k)
    assert n(plan, nat.TOP_WGRAD) < n(full, nat.TOP_WGRAD)
    assert n(plan, nat.TOP_CONV) == n(full, nat.TOP_CONV)       # every data gradient is still formed


def test_train_mode_norms_in_a_frozen_prefix_keep_the_training_forward():
    """requires_grad=False without eval(): the reference still normalises with batch statistics and updates the running statistics, so
    those layers stay on BN_STATS / BN_APPLY (no inference prefix) and only lose their backward."""
    model, _ = synth_model('WIDERFACE_L')
    model.train()
    for p in model._backbone._stem.parameters():
        p.requires_grad = False
    plan = TrainPlan(model, 2, 128, 160, CPU, create_native=False)
    assert plan._prefix is None
    stem = [L for L in plan._layers if L['name'].startswith('stem')]
    assert stem and all(not L['frozen'] for L in stem)
    names = {L['y'] for L in stem} | {L['z'] for L in stem}
    for op in plan.bwd_ops:
        for v in op.get('off', {}).values():
            assert not (isinstance(v, str) and v.startswith('d_') and v[2:] in names), v
    assert not any(op['kind'] == nat.TOP_WGRAD_STEM for op in plan.bwd_ops)


def test_no_trainable_parameter_raises():
    model, _ = synth_model('WIDERFACE_S')
    model.train()
    for p in model.parameters():
        p.requires_grad = False
    with pytest.raises(ValueError, match='trainable'):
        TrainPlan(model, 2, 128, 160, CPU, create_native=False)


def test_fused_sgd_runs_skip_frozen_slots():
    """FusedSGD steps over runs of the flat buffer: a frozen parameter's slots are in none of them (torch.optim.SGD skips a parameter
    without gradient: no weight decay, no momentum), and (un)freezing rebuilds the runs."""
    from lfd.execution.optim import FusedSGD
    model = finetune_model('WIDERFACE_L', 2, -1.0)
    flat = flat_parameters(model, allow_cpu=True)
    opt = FusedSGD(model, torch.optim.SGD(model.parameters(), lr=0.01, momentum=0.9, weight_decay=1e-4).param_groups)
    opt._flat = flat
    opt._make_runs()

    def covered():
        return [p for p, off in zip(flat.params, flat.offsets) if any(b <= off < e for b, e, _, _ in opt._runs)]
    assert {id(p) for p in covered()} == {id(p) for p in model.parameters() if p.requires_grad}
    for p in model._backbone._stem.parameters():
        p.requires_grad = True
    opt._make_runs()
    assert {id(p) for p in covered()} == {id(p) for p in model.parameters() if p.requires_grad}
