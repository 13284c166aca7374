# -*- coding: utf-8 -*-
"""The native training step through the drop-in API on the GPU (SURVEY section 8 rows a19 / g1, section 8e).

Everything in the step is hand-written CUDA: forward in train mode (BatchNorm batch statistics), label assignment, losses, the
backward of the whole conv stack (wgmma dgrad / wgrad, norm backward), the flat-bucket gradient all-reduce, clip + SGD.
The checker is tests/aten_train_reference.py: the SAME module graph evaluated by ATen in fp32 and differentiated by autograd --
the reference's arithmetic (lfd/model/lfd.py:511-542 through autograd)."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import synth
from aten_train_reference import train_forward as aten_train_forward
from helpers import rel_err, synth_model

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _freeze_norms(model):
    for m in model.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.eval()


def _pair(cfg, cls_bias=-2.0):
    a, _ = synth_model(cfg, cls_bias=cls_bias)
    b, _ = synth_model(cfg, cls_bias=cls_bias)
    return a.cuda().train(), b.cuda().train()


@pytest.mark.parametrize('cfg,frozen', [('WIDERFACE_XS', False), ('WIDERFACE_L', False), ('TT100K_S', False), ('WIDERFACE_S', True), ('TL_L', False),
                                        ('TEST_FAST', False)])
def test_native_train_forward_matches_aten(cfg, frozen):
    """Train-mode forward (batch statistics; `frozen`: BatchNorm modules in eval mode, as with norm_eval): native bf16 plan vs ATen fp32
    on the same weights -- outputs inside the bf16 drift of DESIGN.md gate C, identical wiring / layout, running statistics updated
    like nn.BatchNorm2d does."""
    model, ref = _pair(cfg)
    if frozen:
        _freeze_norms(model)
        _freeze_norms(ref)
    x = synth.synth_input(2, 184, 248).cuda()
    emu, _ = synth_model(cfg, cls_bias=-2.0)
    emu.cuda().train()
    if frozen:
        _freeze_norms(emu)
    with torch.no_grad():
        cls_n, reg_n = model(x)
        cls_n, reg_n = cls_n.clone(), reg_n.clone()
        cls_t, reg_t = aten_train_forward(ref, x)
        cls_e, reg_e = aten_train_forward(emu, x, emulate_bf16=True)
    assert cls_t.shape == cls_n.shape and reg_t.shape == reg_n.shape
    assert dict(model._head_indexes_to_feature_map_sizes) == dict(ref._head_indexes_to_feature_map_sizes)
    # against the same graph with the native rounding points (bf16-emulated) and against plain fp32: train mode stores z AND y per
    # layer as bf16 and re-normalises every layer to unit variance, so the drift is about twice the inference plan's
    for a, b, c in ((cls_n, cls_e, cls_t), (reg_n, reg_e, reg_t)):
        assert rel_err(a, b)[1] < 3e-2, ('vs bf16-emulated', rel_err(a, b))
        assert rel_err(a, c)[1] < 6e-2, ('vs fp32', rel_err(a, c))
        assert rel_err(a, c)[1] < 2.5 * max(rel_err(b, c)[1], 1e-2), ('drift vs the emulation\'s own drift', rel_err(a, c), rel_err(b, c))
    worst, worst_emu = 0.0, 0.0
    for (name, ba), (_, bb_), (_, be) in zip(model.named_buffers(), ref.named_buffers(), emu.named_buffers()):
        if ba.dtype.is_floating_point:
            worst = max(worst, float((ba - bb_).abs().max() / bb_.abs().max().clamp(min=1e-6)))
            worst_emu = max(worst_emu, float((be - bb_).abs().max() / bb_.abs().max().clamp(min=1e-6)))
        else:
            assert torch.equal(ba, bb_), name          # num_batches_tracked
    # running statistics: within the drift the bf16-emulated ATen graph itself shows against fp32 (the deepest stage has < 100 samples per
    # channel at this input size; tests/debug_bn_buffers.py prints the per-buffer table)
    assert worst < 2.0 * max(worst_emu, 1e-2), (worst, worst_emu)


@pytest.mark.parametrize('cfg', ['WIDERFACE_XS', 'WIDERFACE_L'])
def test_native_parameter_gradients_end_to_end(cfg):
    """loss.backward() through the native backward plan vs autograd over the ATen evaluation, END TO END.  Two 16-bit pipelines whose
    activations agree to ~1 % flip about that fraction of the ReLU masks, and every flipped element carries a full-size gradient error:
    the gradients of deep layers decorrelate at the 30-50 % level -- for ANY pair of bf16 pipelines: the ATen graph with the native
    rounding points (emulated) differs from ATen fp32 by as much as the native path does.  What is asserted end to end is therefore
    (a) losses agree, (b) the native gradients are as close to the fp32 ones as the emulation is (within 1.5x), (c) the layers next to
    the loss (final head convs) agree tightly.  The tight, per-element statement is test_gpu_train_step_per_op.py."""
    models = [synth_model(cfg, cls_bias=-2.0)[0].cuda().train() for _ in range(3)]
    n, h, w = 4, 192, 256
    x = synth.synth_input(n, h, w).cuda()
    ann = synth.synth_annotations(n, h, w, models[0]._num_classes, seed=3)
    lv = []
    for i, m in enumerate(models):
        out = m(x) if i == 0 else aten_train_forward(m, x, emulate_bf16=(i == 2))
        ld = m.get_loss(out, ann)
        if i:
            for p in m.parameters():
                p.grad = None
        ld['loss'].backward()
        lv.append(ld['loss_values']['loss'])
    assert abs(lv[0] - lv[1]) < 2e-2 * abs(lv[1]) and abs(lv[0] - lv[2]) < 2e-2 * abs(lv[2]), lv
    sq = [0.0, 0.0, 0.0]      # |native - fp32|^2, |emulated - fp32|^2, |fp32|^2 over all parameters
    for (name, p), (_, q), (_, r) in zip(*[m.named_parameters() for m in models]):
        assert p.grad is not None and torch.isfinite(p.grad).all(), name
        g, t, e = p.grad.double(), q.grad.double(), r.grad.double()
        sq[0] += float(((g - t) ** 2).sum()); sq[1] += float(((e - t) ** 2).sum()); sq[2] += float((t ** 2).sum())
        if 'classification_path' in name and name.endswith('weight'):
            assert float((g - t).norm() / t.norm()) < 5e-2, name
    nat, emu = (sq[0] / sq[2]) ** 0.5, (sq[1] / sq[2]) ** 0.5
    print('%s: whole-model gradient error vs fp32: native %.2f, bf16-emulated ATen %.2f' % (cfg, nat, emu))
    assert nat < 1.5 * emu + 0.05, (nat, emu)


def test_train_loop_reduces_the_loss():
    """Executor-style iterations on a fixed batch with the hook's native path: forward (train mode), native get_loss, backward,
    fused clip + SGD over the flat buffers -- every parameter receives a finite gradient and the loss goes down."""
    from lfd.execution.hooks import OptimizerHook
    from lfd.execution.optim import FusedSGD
    model, _ = synth_model('WIDERFACE_XS', cls_bias=-2.0)
    model.cuda().train()
    n, h, w = 4, 256, 256
    x = synth.synth_input(n, h, w).cuda()
    ann = synth.synth_annotations(n, h, w, 1, seed=3)
    opt = FusedSGD.from_torch(torch.optim.SGD(model.parameters(), lr=0.01, momentum=0.9, weight_decay=1e-4), model)
    hook = OptimizerHook(dict(max_norm=10, norm_type=2, duration=5), 10)

    class _Exec(object):
        config_dict = dict(model=model, optimizer=opt, epoch=0)
    losses = []
    for it in range(8):
        out = model(x)
        ld = model.get_loss(out, ann)
        _Exec.config_dict['loss'] = ld['loss']
        hook.after_train_iter(_Exec)
        if it == 0:
            for name, p in model.named_parameters():
                assert p.grad is not None and torch.isfinite(p.grad).all(), name
            assert float(_Exec.config_dict['grad_norm']) > 0
        losses.append(ld['loss_values']['loss'])
    assert all(np.isfinite(losses)), losses
    assert losses[-1] < 0.8 * losses[0], losses
    # the eval path picks the updated weights up
    model.eval()
    with torch.no_grad():
        cls, reg = model(x)
    assert torch.isfinite(cls).all() and torch.isfinite(reg).all()


def test_fused_sgd_state_dict_round_trip():
    from lfd.execution.optim import FusedSGD
    model, _ = synth_model('WIDERFACE_XS')
    model.cuda().train()
    topt = torch.optim.SGD(model.parameters(), lr=0.01, momentum=0.9, weight_decay=1e-4)
    opt = FusedSGD.from_torch(topt, model)
    opt.zero_grad()
    for p in model.parameters():
        p.grad.normal_()
    opt.step()
    sd = opt.state_dict()
    assert len(sd['state']) == len(list(model.parameters())) and sd['param_groups'][0]['lr'] == 0.01
    topt2 = torch.optim.SGD(model.parameters(), lr=0.5, momentum=0.9)
    topt2.load_state_dict(sd)          # the reference's optimizer reads it
    opt2 = FusedSGD.from_torch(topt2, model)
    opt2.load_state_dict(sd)
    opt2._sync()
    assert opt2.param_groups[0]['lr'] == 0.01 and torch.equal(opt2._mom, opt._mom)


def test_cuda_graph_training_step_matches_eager():
    model, ref = _pair('WIDERFACE_XS')
    ref.use_cuda_graph_training = True
    n, h, w = 2, 128, 160
    x = synth.synth_input(n, h, w).cuda()
    ann = synth.synth_annotations(n, h, w, 1, seed=5)
    grads = []
    for m in (model, ref):
        for it in range(3):          # the third pass of `ref` replays the captured graphs
            out = m(x)
            ld = m.get_loss(out, ann)
            m._flat_parameters.grad.zero_()
            ld['loss'].backward()
        grads.append(m._flat_parameters.grad.clone())
    assert float((grads[0] - grads[1]).abs().max()) <= 1e-3 * float(grads[0].abs().max())


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='needs 2 GPUs (NCCL)')
def test_ddp_two_ranks_match_one_rank_on_the_full_batch():
    """tests/run_train_ddp.py: 2 ranks (NCCL), each on half of the batch, global positive-count normalisation + SUM
    all-reduce of the flat gradient buffer == 1 rank on the whole batch."""
    env = dict(os.environ, MASTER_ADDR='127.0.0.1')
    cmd = [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', '2', '--master-addr', '127.0.0.1',
           '--master-port', '29517', os.path.join(ROOT, 'tests', 'run_train_ddp.py')]
    r = subprocess.run(cmd, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:]
    assert 'DDP_OK' in r.stdout, r.stdout[-3000:]


def test_train_plan_autotune_restores_the_model_state():
    """TrainPlan.autotune replays the forward / backward graphs to pick CTA bounds for the side-branch kernels; BatchNorm running
    statistics, num_batches_tracked, the gradient buffer and the plan outputs must come back bit-exact, and the next step must agree with
    an untuned twin."""
    model, twin = _pair('WIDERFACE_XS')
    x = synth.synth_input(2, 160, 192).cuda()
    ann = synth.synth_annotations(2, 160, 192, model._num_classes, seed=3)
    for m in (model, twin):
        m.get_loss(m(x), ann)['loss'].backward()
    torch.cuda.synchronize()
    plan = list(model._train_plans.values())[0]
    before = {k: v.clone() for k, v in model.state_dict().items()}
    g_before = model._flat_parameters.grad.clone()
    res = plan.autotune(candidates=(64,), budget_s=2.0)
    assert set(res) == {'fwd', 'bwd'}
    for k, v in model.state_dict().items():
        assert torch.equal(v, before[k]), k
    assert torch.equal(model._flat_parameters.grad, g_before)
    for m in (model, twin):
        m.zero_grad(set_to_none=False)
        m._flat_parameters.grad.zero_()
        m.get_loss(m(x), ann)['loss'].backward()
    torch.cuda.synchronize()
    a, b = model._flat_parameters.grad, twin._flat_parameters.grad
    assert float((a - b).norm() / b.norm()) < 2e-2           # (atomics order + bf16 re-rounding, as between any two runs)
