# -*- coding: utf-8 -*-
"""Timing of the training input pipeline on one GPU: per batch, the host milliseconds for draws + decode and for the window copies,
the megabytes sent to the device and the input kernel's time (CUDA events over repeated launches); then the WIDERFACE_L training
step fed by the DataLoader against the same step fed a fixed synthetic uint8 batch.

    python tests/debug_input_timing.py [--batch 64] [--crop 480] [--workers 8] [--steps 20] [--jpeg]

Sources are synthetic 1024x768 BGR images held in memory (or as JPEG bytes with --jpeg, decoded by cv2 or turbojpeg)."""
import argparse
import os
import random
import subprocess
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [HERE, os.path.dirname(HERE), os.path.join(os.path.dirname(HERE), 'lfd-a-light-and-fast-detector_b200')]

import numpy as np  # noqa: E402
import torch  # noqa: E402


class SyntheticDataset(object):
    def __init__(self, n, jpeg, seed=0):
        rng = np.random.default_rng(seed)
        base = rng.integers(0, 256, (768, 1024, 3), dtype=np.uint8)
        self.samples = {}
        for i in range(n):
            img = np.roll(base, 37 * i, axis=1)
            s = {'bboxes': [[int(rng.integers(0, 900)), int(rng.integers(0, 650)), 40, 50]], 'bbox_labels': [0]}
            if jpeg:
                import cv2
                s['image_bytes'] = cv2.imencode('.jpg', img, [cv2.IMWRITE_JPEG_QUALITY, 90])[1].tobytes()
            else:
                s['image'] = img
            self.samples[i] = s

    def __len__(self):
        return len(self.samples)

    def __getitem__(self, i):
        return self.samples[i]

    def get_indexes(self):
        return list(self.samples.keys())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=64)
    ap.add_argument('--crop', type=int, default=480)
    ap.add_argument('--workers', type=int, default=8)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--jpeg', action='store_true')
    a = ap.parse_args()
    from lfd.data_pipeline import DataLoader, RandomWithNegDatasetSampler, RandomBBoxCropRegionSampler, simple_widerface_train_pipeline
    from helpers import synth_model
    import synth
    print(subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip())
    random.seed(0), np.random.seed(0)
    ds = SyntheticDataset(a.batch * (a.steps + 3), a.jpeg)
    loader = DataLoader(ds, RandomWithNegDatasetSampler(ds, batch_size=a.batch), RandomBBoxCropRegionSampler(a.crop, (0.5, 1.5), 0.5),
                        simple_widerface_train_pipeline, num_workers=a.workers)
    # 1. loader alone: host time per batch, bytes, kernel time
    stats, t0 = [], time.perf_counter()
    for k, (x, ann, meta) in enumerate(loader):
        stats.append(dict(loader.last_stats))
        if k == a.steps:
            break
    torch.cuda.synchronize()
    wall = (time.perf_counter() - t0) / (a.steps + 1)
    st = stats[2:]
    print('loader: %d images/batch, %s, %d workers: draws+decode %.2f ms, window copies %.2f ms, %.2f MB to the device per batch; '
          'wall %.1f ms per batch (%.0f images/s)' % (a.batch, 'JPEG' if a.jpeg else 'decoded', a.workers,
                                                       np.mean([s['draw_decode_ms'] for s in st]), np.mean([s['copy_ms'] for s in st]),
                                                       np.mean([s['h2d_bytes'] for s in st]) / 1e6, wall * 1e3, a.batch / wall))
    # 2. kernel time: one batch's windows staged on the device, the launch repeated between CUDA events
    import ctypes as C
    from lfd import _native as nat
    from lfd.data_pipeline.data_loader.data_loader import source_window
    from lfd.data_pipeline.sampler.region_sampler import resize_plan
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
    for mode_name, mode, shape, dt in (('uint8 NHWC', nat.INPUT_OUT_U8_NHWC, (a.batch, a.crop, a.crop, 3), torch.uint8),
                                       ('fp32 NCHW', nat.INPUT_OUT_F32_NCHW, (a.batch, 3, a.crop, a.crop), torch.float32)):
        out = torch.empty(shape, dtype=dt, device='cuda')
        launch = lambda: nat.check(nat.lib().lfd_input_batch(nat.ptr(dd), a.batch, nat.ptr(src), nat.ptr(out), mode, 0, a.crop, a.crop, m, sc,
                                                             nat.stream_ptr()))
        for _ in range(5):
            launch()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(50):
            launch()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 50
        moved = src.numel() + out.numel() * out.element_size()
        print('input kernel, %s: %.3f ms per batch of %d (%.0f GB/s over the %.1f MB read + written)' % (mode_name, ms, a.batch, moved / ms / 1e6, moved / 1e6))
    # 3. WIDERFACE_L training step fed by the loader against the same step on a fixed synthetic batch
    from lfd.execution.optim import FusedSGD
    model, _ = synth_model('WIDERFACE_L', cls_bias=-2.0)
    model.cuda().train()
    opt = FusedSGD.from_torch(torch.optim.SGD(model.parameters(), lr=1e-3, momentum=0.9, weight_decay=1e-4), model)
    fixed = (torch.from_numpy(np.ascontiguousarray(synth.synth_input(a.batch, a.crop, a.crop).numpy().transpose(0, 2, 3, 1) * 127.5 + 127.5)
                              .clip(0, 255).astype(np.uint8)).cuda(), synth.synth_annotations(a.batch, a.crop, a.crop, 1, seed=3))

    def step(x, ann):
        opt.zero_grad()
        ld = model.get_loss(model(x), ann)
        ld['loss'].backward()
        opt.step(max_norm=35.0)

    def timed(batches):
        n = 0
        for k, (x, ann) in enumerate(batches):
            if k == 3:
                torch.cuda.synchronize()
                t = time.perf_counter()
            step(x, ann)
            n += k >= 3
        torch.cuda.synchronize()
        return (time.perf_counter() - t) / n * 1e3

    fixed_ms = timed([fixed] * (a.steps + 3))
    loader_ms = timed(((x, ann) for k, (x, ann, _) in zip(range(a.steps + 3), loader)))
    print('WIDERFACE_L training step, batch %d at %dx%d: %.2f ms on a fixed batch (%.0f images/s), %.2f ms fed by the loader (%.0f images/s)'
          % (a.batch, a.crop, a.crop, fixed_ms, a.batch / fixed_ms * 1e3, loader_ms, a.batch / loader_ms * 1e3))


if __name__ == '__main__':
    main()
