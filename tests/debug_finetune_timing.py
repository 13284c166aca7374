# -*- coding: utf-8 -*-
"""Step time of native fine-tuning with frozen backbone stages: WIDERFACE_L and WIDERFACE_S, 16 crops of 640 x 640 (uint8 frames, as
bench.py's training workload), LFDResNet(frozen_stages=k) for k in {-1, 1, 2, number of stages}.

One step = train-mode forward, label assignment + losses, backward, flat-bucket clip + SGD (the OptimizerHook's native path), CUDA
graphs on and side-branch CTA bounds autotuned, as in bench.py.  Per config the arms are timed in alternation within one session:
each round times every arm over a window of >= 0.5 s of device time (CUDA events); the median over the rounds is reported.

    python tests/debug_finetune_timing.py [--rounds 5] [--configs WIDERFACE_L,WIDERFACE_S]
"""
import argparse
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'lfd-a-light-and-fast-detector_b200'), os.path.join(ROOT, 'tests')):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

import synth  # noqa: E402
from helpers import build_model  # noqa: E402
import lfd._native as nat  # noqa: E402
from lfd.execution.hooks import OptimizerHook  # noqa: E402
from lfd.execution.optim import FusedSGD  # noqa: E402

N, H, W = 16, 640, 640


def card():
    name = torch.cuda.get_device_name()
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', str(torch.cuda.current_device())],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip()
    except Exception as e:
        q = 'power limit unavailable (%s)' % e
    return '%s | nvidia-smi: %s' % (name, q)


class Arm(object):
    def __init__(self, cfg, frozen_stages, pool, anns):
        torch.manual_seed(0)
        self.model = build_model(cfg)
        bb = self.model._backbone
        self.k = frozen_stages
        bb._frozen_stages = frozen_stages
        self.model.cuda().train()
        self.model.use_cuda_graph_training = True
        self.opt = FusedSGD.from_torch(torch.optim.SGD(self.model.parameters(), lr=0.001, momentum=0.9, weight_decay=1e-4), self.model)
        self.hook = OptimizerHook(dict(max_norm=10, norm_type=2), 10)
        self.pool, self.anns, self.i = pool, anns, 0
        model, opt = self.model, self.opt

        class _Exec(object):
            config_dict = dict(model=model, optimizer=opt, epoch=0)
        self.ex = _Exec
        self.step()
        torch.cuda.synchronize()
        for p_ in self.model._train_plans.values():
            p_.autotune()
        for _ in range(3):
            self.step()
        torch.cuda.synchronize()
        self.plan = list(self.model._train_plans.values())[-1]

    def step(self):
        i = self.i % len(self.pool)
        self.i += 1
        ld = self.model.get_loss(self.model(self.pool[i]), self.anns[i])
        self.ex.config_dict['loss'] = ld['loss']
        self.hook.after_train_iter(self.ex)

    def window(self, reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            self.step()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--configs', default='WIDERFACE_L,WIDERFACE_S')
    args = ap.parse_args()
    torch.cuda.set_device(0)
    print('card: %s' % card())
    print('workload: %d crops of %dx%d (uint8 NHWC), CUDA graphs, autotuned side branches; median of %d alternated rounds, windows >= 0.5 s'
          % (N, H, W, args.rounds))
    g = torch.Generator().manual_seed(2000)
    pool = [torch.randint(0, 256, (N, H, W, 3), generator=g, dtype=torch.uint8).cuda() for _ in range(4)]
    anns = [synth.synth_annotations(N, H, W, 1, seed=i, max_boxes=30) for i in range(4)]
    for cfg in args.configs.split(','):
        n_stages = len(build_model(cfg)._backbone.stages())
        arms = []
        for k in (-1, 1, 2, n_stages):
            arms.append(Arm(cfg, k, pool, anns))
        reps = {}
        for a in arms:
            t = a.window(3)
            reps[a.k] = max(3, int(math.ceil(500.0 / t)))
        times = {a.k: [] for a in arms}
        for _ in range(args.rounds):
            for a in arms:
                times[a.k].append(a.window(reps[a.k]))
        base = sorted(times[-1])[len(times[-1]) // 2]
        for a in arms:
            ts = sorted(times[a.k])
            med = ts[len(ts) // 2]
            n_infer = sum(1 for op in a.plan.fwd_ops if op['kind'] == nat.TOP_INFER)
            print('%-12s frozen_stages=%2d  step %7.2f ms (min %.2f, max %.2f)  %7.0f images/s  x%.2f vs -1  workspace %.2f GB  ops fwd %d (prefix %d) / bwd %d'
                  % (cfg, a.k, med, ts[0], ts[-1], N / (med / 1e3), base / med, a.plan.workspace_bytes / 1e9, len(a.plan.fwd_ops), n_infer,
                     len(a.plan.bwd_ops)))
        del arms
        torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
