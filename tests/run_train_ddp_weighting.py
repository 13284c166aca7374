# -*- coding: utf-8 -*-
"""Launched by torchrun with 2 ranks (tests/test_gpu_loss_weighting.py): tests/run_train_ddp.py with enable_classification_weight and
enable_regression_weight on.  The weight sum (the normaliser of both weighted losses) is summed over the ranks next to the positive count,
so three sharded iterations must leave every rank with the parameters one process obtains on the full batch.

    python -m torch.distributed.run --nproc-per-node 2 tests/run_train_ddp_weighting.py [nccl | gloo]

nccl puts rank r on GPU r; gloo runs both ranks on GPU 0 (the gradient and loss all-reduces work on CUDA tensors with either backend).
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [HERE, os.path.dirname(HERE), os.path.join(os.path.dirname(HERE), 'lfd-a-light-and-fast-detector_b200')]
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import synth  # noqa: E402
from helpers import synth_model  # noqa: E402
from run_train_ddp import run  # noqa: E402


def main():
    backend = sys.argv[1] if len(sys.argv) > 1 else 'nccl'
    rank = int(os.environ['RANK'])
    torch.cuda.set_device(int(os.environ['LOCAL_RANK']) if backend == 'nccl' else 0)
    n, h, w = 4, 192, 192
    batches = [(synth.synth_input(n, h, w, seed=10 + i), synth.synth_annotations(n, h, w, 1, seed=20 + i)) for i in range(3)]

    def fresh():
        m, _ = synth_model('WIDERFACE_XS', cls_bias=-2.0)
        m._enable_classification_weight = m._enable_regression_weight = True
        m.cuda().train()
        for mod in m.modules():
            if isinstance(mod, torch.nn.BatchNorm2d):
                mod.eval()
        return m

    ref = fresh()
    ref_losses = run(ref, batches, sharded=False)
    dist.init_process_group(backend)
    ddp = fresh()
    losses = run(ddp, batches, sharded=True)
    assert ddp.loss_globally_normalised
    t = torch.tensor(losses, dtype=torch.float64, device='cuda')
    dist.all_reduce(t)
    t /= dist.get_world_size()
    worst = 0.0
    for (name, a), (_, b) in zip(ref.named_parameters(), ddp.named_parameters()):
        worst = max(worst, float((a.detach() - b.detach()).abs().max() / a.detach().abs().max().clamp(min=1e-12)))
    ok = worst < 5e-3 and all(abs(float(t[i]) - ref_losses[i]) < 2e-3 * abs(ref_losses[i]) for i in range(len(ref_losses)))
    flat = torch.cat([p.detach().reshape(-1) for p in ddp.parameters()])
    other = flat.clone()
    dist.broadcast(other, src=0)
    same = bool((flat == other).all())
    flag = torch.tensor([1 if (ok and same) else 0], device='cuda')
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    if rank == 0:
        print('%s, weighted: losses full batch %s | logged by the ranks (global) %s | worst relative parameter difference %.2e | identical '
              'across ranks %s' % (backend, ['%.5f' % v for v in ref_losses], ['%.5f' % float(v) for v in t], worst, same))
        print('DDP_OK' if int(flag.item()) == 1 else 'DDP_MISMATCH')
    dist.barrier()
    dist.destroy_process_group()
    return 0 if int(flag.item()) == 1 else 1


if __name__ == '__main__':
    sys.exit(main())
