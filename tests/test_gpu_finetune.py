# -*- coding: utf-8 -*-
"""Fine-tuning on the GPU: LFDResNet(frozen_stages=k) and hand-frozen parameters through the native training step.

The frozen backbone prefix runs on the inference kernels (LFD_TOP_INFER ops) and must hand over bit-identical tensors to the inference
plan's; the backward covers the trainable part only; frozen parameters keep their values, BatchNorm buffers and a None .grad, as with
torch autograd + torch.optim.SGD."""
import os

import numpy as np
import pytest
import torch

import synth
from helpers import finetune_model, synth_model
from lfd._engine import InferencePlan
from lfd.execution.executor import Executor
from lfd.execution.optim import FusedSGD
from test_gpu_train_step_per_op import Replay

pytestmark = pytest.mark.gpu


def _input(fmt, n, h, w, seed=0):
    if fmt == 'f32':
        return synth.synth_input(n, h, w, seed=seed).cuda()
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (n, h, w, 3), generator=g, dtype=torch.uint8).cuda()


def _prefix_matches_inference(model, plan, x):
    """Every tensor the prefix hands over == the same tensor of an InferencePlan for the same model, input and shape (bit for bit)."""
    n = x.shape[0]
    h, w = (x.shape[1], x.shape[2]) if x.dtype == torch.uint8 else (x.shape[2], x.shape[3])
    was_training = model.training
    model.eval()
    ref = InferencePlan(model, n, h, w, x.device, reuse=False)          # keep every inference tensor readable after the forward
    ref.forward(x, use_graph=False)
    model.train(was_training)
    torch.cuda.synchronize()
    assert plan.prefix_outputs
    for name, (hh, ww, c) in plan.prefix_outputs.items():
        a = plan.tensor(name, hh, ww, c).view(torch.int16)
        b = ref.tensor(name).view(torch.int16)
        assert a.shape == b.shape and torch.equal(a, b), name
    return ref


@pytest.mark.parametrize('cfg,frozen_stages,shape,stem4', [('WIDERFACE_S', 1, (2, 656, 640), True), ('WIDERFACE_S', 2, (2, 128, 160), False),
                                                           ('WIDERFACE_L', 'all', (2, 186, 252), None), ('TT100K_L', 2, (1, 186, 252), None)])
@pytest.mark.parametrize('fmt', ['f32', 'u8'])
def test_prefix_tensors_equal_the_inference_plans(cfg, frozen_stages, shape, stem4, fmt):
    model = finetune_model(cfg, frozen_stages, -2.0).cuda()
    x = _input(fmt, *shape)
    plan = model.train_plan_for(*shape, x.device)
    kinds = {op['kind'] for _, op in plan._prefix['ops']}
    if stem4 is not None:
        assert (4 in kinds) == stem4, kinds                 # lfd._native.OP_STEM4, chosen by the inference plan's L2 gate
    plan.forward(x)
    _prefix_matches_inference(model, plan, x)


def _sgd(model, lr=0.02):
    return torch.optim.SGD(model.parameters(), lr=lr, momentum=0.9, weight_decay=1e-4)


def _frozen_state(model):
    frozen = {n: p.detach().clone() for n, p in model.named_parameters() if not p.requires_grad}
    bufs = {}
    for mn, m in model.named_modules():
        if isinstance(m, torch.nn.BatchNorm2d) and not m.training:
            for bn, b in m.named_buffers():
                bufs[mn + '.' + bn] = b.detach().clone()
    return frozen, bufs


def test_fused_sgd_steps_like_torch_sgd_with_frozen_parameters():
    """FusedSGD over the flat buffers vs torch.optim.SGD (momentum 0.9, weight decay 1e-4) on the same gradients: frozen parameters
    untouched and without momentum entry, trainable ones and their momentum buffers to the optimizer kernel test's bound."""
    model = finetune_model('WIDERFACE_L', 2, -2.0).cuda()
    twin = finetune_model('WIDERFACE_L', 2, -2.0).cuda()
    opt = FusedSGD.from_torch(_sgd(model), model)
    topt = _sgd(twin)
    opt.zero_grad()
    g = torch.Generator(device='cuda').manual_seed(1)
    for _ in range(3):
        for p, q in zip(model.parameters(), twin.parameters()):
            if p.requires_grad:
                gg = torch.randn(p.shape, device='cuda', generator=g)
                p.grad.copy_(gg)
                q.grad = gg.clone()
            else:
                assert p.grad is None
                q.grad = None
        opt.step()
        topt.step()
        for (name, p), q in zip(model.named_parameters(), twin.parameters()):
            if not p.requires_grad:
                assert torch.equal(p, q), name
            else:     # the bound test_gpu_train_kernel_configs.py holds FusedSGD to against torch.optim.SGD
                assert torch.allclose(p, q, rtol=1e-5, atol=1e-6), name
    sd, tsd = opt.state_dict(), topt.state_dict()
    assert set(sd['state']) == set(tsd['state'])
    for k, st in tsd['state'].items():
        assert torch.allclose(sd['state'][k]['momentum_buffer'], st['momentum_buffer'], rtol=1e-5, atol=1e-6), k
    assert len(sd['state']) == sum(1 for p in model.parameters() if p.requires_grad)


def _loader(n_batches, seed0, N=4, H=160, W=192):
    out = []
    for i in range(n_batches):
        x = synth.synth_input(N, H, W, seed=seed0 + i).numpy()
        ann = synth.synth_annotations(N, H, W, 1, seed=seed0 + 50 + i, max_boxes=6)
        meta = [dict(image_id=100 * i + j, resized_height=H, resized_width=W, resize_scale=1.0) for j in range(N)]
        out.append((x, ann, meta))
    return out


def _config(work_dir, epochs, frozen_stages, resume=None):
    model, _ = synth_model('WIDERFACE_XS', cls_bias=-2.0)
    model._backbone._frozen_stages = frozen_stages
    opt = _sgd(model)
    sched = torch.optim.lr_scheduler.MultiStepLR(opt, milestones=[1], gamma=0.5)
    return dict(work_dir=work_dir, log_path=None, model=model, optimizer=opt, lr_scheduler=sched, training_epochs=epochs, gpu_list=[0],
                train_data_loader=_loader(3, 10), val_data_loader=_loader(1, 90), evaluator=None, val_interval=1, save_interval=1,
                display_interval=1, optimizer_grad_clip_cfg=dict(max_norm=10, norm_type=2),
                warmup_setting=dict(by_epoch=False, warmup_mode='linear', warmup_loops=2, warmup_ratio=0.1), resume_path=resume, weight_path=None)


def test_executor_fine_tunes_with_frozen_stages_and_resumes(tmp_path):
    a = _config(os.path.join(str(tmp_path), 'a'), 2, frozen_stages=2)
    model = a['model']
    model.cuda().train()
    frozen0, bufs0 = _frozen_state(model)
    trainable0 = {n: p.detach().clone() for n, p in model.named_parameters() if p.requires_grad}
    assert frozen0 and bufs0 and trainable0
    ex = Executor(a)
    ex.run()
    model.train()
    frozen1, bufs1 = _frozen_state(model)
    assert set(frozen1) == set(frozen0)
    for k in frozen0:
        assert torch.equal(frozen0[k], frozen1[k]), k
    for k in bufs0:
        assert torch.equal(bufs0[k], bufs1[k]), k
    for n, p in model.named_parameters():
        if p.requires_grad:
            assert not torch.equal(p.detach(), trainable0[n]), n
        else:
            assert p.grad is None, n
    ck = torch.load(os.path.join(a['work_dir'], 'epoch_2.pth'), weights_only=False)
    tsgd = _sgd(model)
    frozen_ids = [i for i, p in enumerate(model.parameters()) if not p.requires_grad]
    assert set(ck['optimizer_state_dict']['state']) == set(range(len(list(model.parameters())))) - set(frozen_ids)
    tsgd.load_state_dict(ck['optimizer_state_dict'])                 # torch.optim.SGD reads it
    # interrupted after epoch 1 and resumed: same end state (the bound of test_gpu_executor.py)
    b = _config(os.path.join(str(tmp_path), 'b'), 2, frozen_stages=2, resume=os.path.join(a['work_dir'], 'epoch_1.pth'))
    exb = Executor(b)
    exb.run()
    worst = 0.0
    for (name, p), (_, q) in zip(a['model'].state_dict().items(), b['model'].state_dict().items()):
        if p.dtype.is_floating_point:
            worst = max(worst, float((p.float() - q.float()).abs().max() / p.float().abs().max().clamp(min=1e-6)))
        else:
            assert torch.equal(p, q), name
    assert worst < 2e-2, worst


def test_fine_tuning_reduces_the_loss():
    from lfd.execution.hooks import OptimizerHook
    model = finetune_model('WIDERFACE_S', 2, -2.0).cuda()
    n, h, w = 4, 256, 256
    x = synth.synth_input(n, h, w).cuda()
    ann = synth.synth_annotations(n, h, w, 1, seed=3)
    opt = FusedSGD.from_torch(_sgd(model, lr=0.01), model)
    hook = OptimizerHook(dict(max_norm=10, norm_type=2, duration=5), 10)

    class _Exec(object):
        config_dict = dict(model=model, optimizer=opt, epoch=0)
    losses = []
    for it in range(8):
        ld = model.get_loss(model(x), ann)
        _Exec.config_dict['loss'] = ld['loss']
        hook.after_train_iter(_Exec)
        losses.append(ld['loss_values']['loss'])
    assert all(np.isfinite(losses)) and losses[-1] < 0.8 * losses[0], losses


def test_new_prefix_weights_are_repacked_and_unfreezing_differentiates():
    """load_state_dict between two steps: the next step's prefix tensors equal a fresh InferencePlan's.  Unfreezing (frozen_stages -1 and
    train() again) gives a plan that differentiates the newly trainable layers, checked layer by layer."""
    model = finetune_model('WIDERFACE_S', 2, -2.0).cuda()
    n, h, w = 2, 160, 192
    x = synth.synth_input(n, h, w).cuda()
    ann = synth.synth_annotations(n, h, w, 1, seed=3)
    model.get_loss(model(x), ann)['loss'].backward()
    plan = model.train_plan_for(n, h, w, x.device)
    other, _ = synth_model('WIDERFACE_S', cls_bias=-2.0, seed=7)
    model.load_state_dict(other.state_dict())
    model.train()
    out = model(x)
    assert model.train_plan_for(n, h, w, x.device) is plan
    _prefix_matches_inference(model, plan, x)
    model.get_loss(out, ann)['loss'].backward()
    # unfreeze
    model._backbone._frozen_stages = -1
    for p in model.parameters():
        p.requires_grad = True
    model.train()
    model._flat_parameters.grad.zero_()
    replay = Replay(model, x, ann)          # the unfrozen step, every op checked per element (test_gpu_train_step_per_op.py)
    replay.replay()
    plan2 = replay.plan
    assert plan2 is not plan and plan2._prefix is None
    stem = model._backbone.stem_layers()[0][0]
    assert stem.weight.grad is not None and float(stem.weight.grad.abs().sum()) > 0


def test_cuda_graph_fine_tuning_step_matches_eager():
    model = finetune_model('WIDERFACE_S', 2, -2.0).cuda()
    ref = finetune_model('WIDERFACE_S', 2, -2.0).cuda()
    ref.use_cuda_graph_training = True
    n, h, w = 2, 128, 160
    x = synth.synth_input(n, h, w).cuda()
    ann = synth.synth_annotations(n, h, w, 1, seed=5)
    grads, prefix = [], []
    for m in (model, ref):
        for it in range(3):          # the third pass of `ref` replays the captured graphs
            out = m(x)
            ld = m.get_loss(out, ann)
            m._flat_parameters.grad.zero_()
            ld['loss'].backward()
        torch.cuda.synchronize()
        plan = m.train_plan_for(n, h, w, x.device)
        prefix.append({k: plan.tensor(k, *s).clone() for k, s in plan.prefix_outputs.items()})
        grads.append(m._flat_parameters.grad.clone())
    for k in prefix[0]:
        assert torch.equal(prefix[0][k], prefix[1][k]), k
    assert float((grads[0] - grads[1]).abs().max()) <= 1e-3 * float(grads[0].abs().max())
