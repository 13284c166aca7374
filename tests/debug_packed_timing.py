# -*- coding: utf-8 -*-
"""What packed camera frames gain end to end, on the card at hand (a script, not a test):

    python tests/debug_packed_timing.py [--seconds 1.0] [--rounds 3]

WIDERFACE_S at 1280x720, batch 8, CUDA graphs, autotuned; StreamingDetector(source_size=(1080, 1920)) from pinned host frames, the
frames resized on the device (s = 2/3), one batch submitted ahead of the collect of the previous one.  Arms:
  YUY2, BGRA, NV12 and BGR frames uploaded as they are and converted in the resize kernel;
  the host path users run today: cv2.cvtColor(YUY2 -> BGR) and cv2.cvtColor(BGRA -> BGR) of every frame on the host, then the BGR arm.
Arms alternate inside every measurement; a window is at least --seconds long and ends in a device synchronise.  Prints the card's name,
power limit and maximal SM clock first: an absolute number means nothing without them."""
import argparse
import os
import subprocess
import sys

import cv2
import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path[:0] = [HERE, ROOT, os.path.join(ROOT, 'lfd-a-light-and-fast-detector_b200')]

from debug_input_transform_timing import alternate, emit  # noqa: E402
from debug_resize_timing import pipelined  # noqa: E402
from helpers import synth_model  # noqa: E402
from lfd.pipeline import StreamingDetector  # noqa: E402
from nv12_oracle import nv12_frames  # noqa: E402
from packed_oracle import packed_frames  # noqa: E402

N, H, W = 8, 720, 1280
SH, SW = 1080, 1920


def host_frames(fmt):
    if fmt == 'nv12':
        return nv12_frames(N, SH, SW, seed=3)
    if fmt == 'bgr':
        return np.random.default_rng(3).integers(0, 256, (N, SH, SW, 3), dtype=np.uint8)
    return packed_frames(N, SH, SW, fmt, seed=3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--seconds', type=float, default=1.0)
    ap.add_argument('--rounds', type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('this script measures the GPU: no CUDA device')
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
    emit(dict(card=smi, torch_device=torch.cuda.get_device_name(0)))
    # (a low classification bias: the synthetic heads must not flood the post-process with candidates)
    model = synth_model('WIDERFACE_S', cls_bias=-6.0)[0].cuda().eval()
    steps, drains, h2d = {}, {}, {}
    for fmt in ('yuy2', 'bgra', 'nv12', 'bgr'):
        det = StreamingDetector(model, N, H, W, 0.5, 0.4, max_out=256, frame_format=fmt, source_size=(SH, SW))
        src = torch.from_numpy(host_frames(fmt)).pin_memory()
        steps[fmt], drains[fmt] = pipelined(det, lambda src=src: src)
        h2d[fmt] = det.h2d_bytes
    # the host path: cv2.cvtColor of every frame into a pinned BGR batch (one per batch in flight), then a BGR detector
    for fmt, code in (('yuy2', cv2.COLOR_YUV2BGR_YUY2), ('bgra', cv2.COLOR_BGRA2BGR)):
        det = StreamingDetector(model, N, H, W, 0.5, 0.4, max_out=256, frame_format='bgr', source_size=(SH, SW))
        src = host_frames(fmt)
        pinned = [torch.empty((N, SH, SW, 3), dtype=torch.uint8).pin_memory() for _ in range(det.depth)]
        turn = [0]

        def host_batch(src=src, code=code, pinned=pinned, turn=turn):
            out = pinned[turn[0] % len(pinned)]
            turn[0] += 1
            for i, f in enumerate(src):
                out[i] = torch.from_numpy(cv2.cvtColor(f, code))
            return out
        name = 'host cvtColor %s + bgr' % fmt
        steps[name], drains[name] = pipelined(det, host_batch)
        h2d[name] = det.h2d_bytes
    r = alternate(steps, a.seconds, a.rounds)
    for name in steps:
        drains[name]()
    for name, ms in r.items():
        emit(dict(arm=name, ms_per_batch=ms, images_per_s=[round(N / (m * 1e-3)) for m in ms], h2d_MB=round(h2d[name] / 1e6, 1)))
    emit(dict(cv2_threads=cv2.getNumThreads(), cpu_count=os.cpu_count()))


if __name__ == '__main__':
    main()
