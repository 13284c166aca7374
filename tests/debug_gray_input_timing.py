# -*- coding: utf-8 -*-
"""Timing of the gray modes of the training input kernel on one GPU, against the 3-channel modes, and of a WIDERFACE_L gray training
step fed by DataLoader(input_channels=1, model_normalizes=True) against the same step on a fixed uint8 gray batch.

    python tests/debug_gray_input_timing.py [--batch 16] [--crop 640] [--rounds 5] [--launches 50] [--steps 20]

The kernel arms run one after the other inside each round (CUDA events over --launches launches each), so every arm sees the same
conditions; the spread is over the rounds.  Sources are synthetic 1024x768 BGR images held in memory."""
import argparse
import ctypes as C
import os
import random
import subprocess
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [HERE, os.path.dirname(HERE), os.path.join(os.path.dirname(HERE), 'lfd-a-light-and-fast-detector_b200')]

import numpy as np  # noqa: E402
import torch  # noqa: E402

from debug_input_timing import SyntheticDataset  # noqa: E402


def _spread(v):
    return 'median %.3f (min %.3f, max %.3f)' % (float(np.median(v)), min(v), max(v))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=16)
    ap.add_argument('--crop', type=int, default=640)
    ap.add_argument('--workers', type=int, default=8)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--launches', type=int, default=50)
    ap.add_argument('--steps', type=int, default=20)
    a = ap.parse_args()
    from lfd import _native as nat
    from lfd.data_pipeline import DataLoader, RandomWithNegDatasetSampler, RandomBBoxCropRegionSampler, simple_widerface_train_pipeline
    from lfd.data_pipeline.data_loader.data_loader import source_window
    from lfd.data_pipeline.sampler.region_sampler import resize_plan
    print(subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True,
                         text=True).stdout.strip())
    random.seed(0), np.random.seed(0)
    per_round = max(3, a.steps // a.rounds)          # training steps per arm and round
    ds = SyntheticDataset(a.batch * (a.rounds * (per_round + 2) + 4), False)
    region = RandomBBoxCropRegionSampler(a.crop, (0.5, 1.5), 0.5)

    # 1. the input kernel on one staged batch of BGR windows, every output mode, alternated per round
    loader = DataLoader(ds, RandomWithNegDatasetSampler(ds, batch_size=a.batch), region, simple_widerface_train_pipeline, num_workers=a.workers)
    items = loader.plan(list(range(a.batch)))[0]
    descs, chunks, off = (nat.InputDesc * len(items))(), [], 0
    for j, (img, d, flip) in enumerate(items):
        h, w = img.shape[:2]
        mode, dh, dw = resize_plan(h, w, d.scale)
        wx, wy, ww, wh = source_window(h, w, d.scale, d.crop)
        win = np.ascontiguousarray(img[wy:wy + wh, wx:wx + ww]).reshape(-1)
        descs[j] = nat.InputDesc(off, 1.0 / d.scale, ww * 3, 3, wx, wy, ww, wh, w, h, dw, dh, mode, d.crop[0], d.crop[1], a.crop, a.crop, int(flip))
        chunks.append(np.pad(win, (0, (-win.size) % 16)))
        off += chunks[-1].size
    src = torch.from_numpy(np.concatenate(chunks)).cuda()
    dd = torch.frombuffer(bytearray(bytes(descs)), dtype=torch.uint8).cuda()
    m = (C.c_float * 3)(127.5, 127.5, 127.5)
    sc = (C.c_float * 3)(*[float(np.float32(1) / np.float32(127.5))] * 3)
    n, s = a.batch, a.crop
    arms = [('uint8 NHWC', nat.INPUT_OUT_U8_NHWC, (n, s, s, 3), torch.uint8), ('uint8 gray', nat.INPUT_OUT_U8_GRAY, (n, s, s), torch.uint8),
            ('fp32 NCHW', nat.INPUT_OUT_F32_NCHW, (n, 3, s, s), torch.float32), ('fp32 gray', nat.INPUT_OUT_F32_GRAY, (n, 1, s, s), torch.float32)]
    outs = {name: torch.empty(shape, dtype=dt, device='cuda') for name, _, shape, dt in arms}

    def launch(mode, out):
        nat.check(nat.lib().lfd_input_batch(nat.ptr(dd), n, nat.ptr(src), nat.ptr(out), mode, 0, s, s, m, sc, nat.stream_ptr()))

    for name, mode, _, _ in arms:
        for _ in range(5):
            launch(mode, outs[name])
    times = {name: [] for name, _, _, _ in arms}
    for _ in range(a.rounds):
        for name, mode, _, _ in arms:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.launches):
                launch(mode, outs[name])
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1) / a.launches)
    for name, _, _, _ in arms:
        moved = src.numel() + outs[name].numel() * outs[name].element_size()
        print('input kernel, %d BGR crops of %dx%d, %s: ms per batch %s; %.1f MB read + written' % (n, s, s, name, _spread(times[name]), moved / 1e6))

    # 2. WIDERFACE_L gray training step: fed by the gray loader, and on a fixed uint8 gray batch, alternated per round
    from gray_models import gray_pair
    from lfd.execution.optim import FusedSGD
    import synth
    model, _ = gray_pair('WIDERFACE_L', cls_bias=-2.0)
    model.cuda().train()
    gray_loader = DataLoader(ds, RandomWithNegDatasetSampler(ds, batch_size=a.batch), region, simple_widerface_train_pipeline,
                             num_workers=a.workers, model_normalizes=True, input_channels=1)
    model.set_input_transform(gray_loader.input_transform)
    opt = FusedSGD.from_torch(torch.optim.SGD(model.parameters(), lr=1e-3, momentum=0.9, weight_decay=1e-4), model)
    g = torch.Generator().manual_seed(3)
    fixed = (torch.randint(0, 256, (n, s, s), generator=g, dtype=torch.uint8).cuda(), synth.synth_annotations(n, s, s, 1, seed=3))

    def step(x, ann):
        opt.zero_grad()
        ld = model.get_loss(model(x), ann)
        ld['loss'].backward()
        opt.step(max_norm=35.0)

    def timed(batches, warm=2):
        count = 0
        for k, (x, ann) in enumerate(batches):
            if k == warm:
                torch.cuda.synchronize()
                t = time.perf_counter()
            step(x, ann)
            count += k >= warm
        torch.cuda.synchronize()
        return (time.perf_counter() - t) / count * 1e3

    batches = iter(gray_loader)
    fixed_ms, loader_ms = [], []
    for _ in range(a.rounds):
        fixed_ms.append(timed([fixed] * (per_round + 2)))
        loader_ms.append(timed(((x, ann) for _, (x, ann, _) in zip(range(per_round + 2), batches))))
        assert gray_loader.last_stats is not None
    st = gray_loader.last_stats
    print('WIDERFACE_L gray training step, batch %d at %dx%d: ms per step on a fixed uint8 gray batch %s; fed by the gray loader %s '
          '(%.2f MB to the device per batch)' % (n, s, s, _spread(fixed_ms), _spread(loader_ms), st['h2d_bytes'] / 1e6))


if __name__ == '__main__':
    main()
