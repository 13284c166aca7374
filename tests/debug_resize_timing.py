# -*- coding: utf-8 -*-
"""What resizing frames on the device costs, on the card at hand (a script, not a test):

    python tests/debug_resize_timing.py [--seconds 0.6] [--rounds 3]

WIDERFACE_S at 1280x720, batch 8, uint8 frames, CUDA graphs, autotuned:
  (a) lfd_resize_frames alone, device-resident sources: 3840x2160 BGR and NV12 (s = 1/3) and 1920x1080 BGR (s = 2/3) -> 1280x720;
  (b) the forward alone on 1280x720 frames (graph replay), and the resize + forward of plan.forward(resize_scale=) on each source;
  (c) end to end from pinned host frames, StreamingDetector(source_size=...) against the host path: cv2.resize of every frame on the host
      (cv2.cvtColor first for NV12), then StreamingDetector at 1280x720 -- per batch, pipelined (submit one batch ahead of collect).
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
from helpers import synth_model  # noqa: E402
from lfd import _native as nat  # noqa: E402
from lfd.pipeline import StreamingDetector  # noqa: E402
from nv12_oracle import nv12_frames  # noqa: E402

N, H, W = 8, 720, 1280
SOURCES = [('bgr', 2160, 3840), ('nv12', 2160, 3840), ('bgr', 1080, 1920)]


def host_frames(kind, h, w, seed=0):
    if kind == 'nv12':
        return nv12_frames(N, h, w, seed)
    rng = np.random.default_rng(seed)
    return rng.integers(0, 256, (N, h, w, 3), dtype=np.uint8)


def host_resized(kind, frames, out):
    """the host path: cv2 on every frame into the pinned uint8 [N, 720, 1280, 3] `out`"""
    for i, f in enumerate(frames):
        if kind == 'nv12':
            f = cv2.cvtColor(f, cv2.COLOR_YUV2BGR_NV12)
        out[i] = torch.from_numpy(cv2.resize(f, (W, H), interpolation=cv2.INTER_LINEAR) if f.shape[:2] != (H, W) else f)


def pipelined(det, batch_fn):
    """one batch submitted ahead of the collect of the previous one"""
    state = {'prev': None}

    def step():
        slot = det.submit(batch_fn())
        if state['prev'] is not None:
            det.collect(state['prev'])
        state['prev'] = slot

    def drain():
        if state['prev'] is not None:
            det.collect(state['prev'])
            state['prev'] = None
    return step, drain


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--seconds', type=float, default=0.6)
    ap.add_argument('--rounds', type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('this script measures the GPU: no CUDA device')
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
    emit(dict(card=smi, torch_device=torch.cuda.get_device_name(0)))
    # (a low classification bias: the synthetic heads must not flood the post-process with candidates)
    model = synth_model('WIDERFACE_S', cls_bias=-6.0)[0].cuda().eval()
    lib = nat.lib()
    dev = torch.device('cuda')
    plan = model.inference_plan(N, H, W, dev, exact=True)
    if not plan.autotuned:
        plan.autotune()
    x720 = torch.from_numpy(host_frames('bgr', H, W, seed=9)).cuda()
    stage = torch.empty((N, H, W, 3), dtype=torch.uint8, device=dev)
    srcs = {}
    for kind, h, w in SOURCES:
        srcs[(kind, h, w)] = torch.from_numpy(host_frames(kind, h, w, seed=h)).cuda()

    def resize_only(kind, h, w):
        x, s = srcs[(kind, h, w)], min(H / h, W / w)
        fmt = nat.INPUT_U8_NV12 if kind == 'nv12' else nat.INPUT_U8_NHWC
        return lambda: nat.check(lib.lfd_resize_frames(nat.ptr(x), fmt, 3, N, h, w, s, nat.ptr(stage), H, W, nat.stream_ptr()))

    # (a) the resize launch alone
    arms = {'%s %dx%d' % (k, w, h): resize_only(k, h, w) for k, h, w in SOURCES}
    r = alternate(arms, a.seconds, a.rounds)
    for (kind, h, w), (name, ms) in zip(SOURCES, r.items()):
        read = N * h * w * (1.5 if kind == 'nv12' else 3)
        emit(dict(part='a resize alone', source=name, ms=ms, source_MB=round(read / 1e6, 1), written_MB=round(N * H * W * 3 / 1e6, 1),
                  GBps_read_plus_written=round((read + N * H * W * 3) / (min(ms) * 1e-3) / 1e9, 1)))
    # (b) the forward alone, and resize + forward
    with torch.no_grad():
        arms = {'forward 1280x720': lambda: plan.forward(x720, use_graph=True)}
        for kind, h, w in SOURCES:
            x, s = srcs[(kind, h, w)], min(H / h, W / w)
            arms['resize+forward %s %dx%d' % (kind, w, h)] = (lambda x=x, s=s, kind=kind: plan.forward(
                x, use_graph=True, resize_scale=s, frame_format='nv12' if kind == 'nv12' else None))
        r = alternate(arms, a.seconds, a.rounds)
    for name, ms in r.items():
        emit(dict(part='b forward', arm=name, ms=ms))
    # (c) end to end from pinned host frames
    for kind, h, w in SOURCES:
        fmt = 'nv12' if kind == 'nv12' else 'bgr'
        src = torch.from_numpy(host_frames(kind, h, w, seed=3)).pin_memory()
        dev_det = StreamingDetector(model, N, H, W, 0.5, 0.4, max_out=256, frame_format=fmt, source_size=(h, w))
        host_det = StreamingDetector(model, N, H, W, 0.5, 0.4, max_out=256)
        pinned = [torch.empty((N, H, W, 3), dtype=torch.uint8).pin_memory() for _ in range(host_det.depth)]   # one per batch in flight
        src_np, turn = src.numpy(), [0]

        def host_batch():
            out = pinned[turn[0] % len(pinned)]
            turn[0] += 1
            host_resized(kind, src_np, out)
            return out
        dev_step, dev_drain = pipelined(dev_det, lambda: src)
        host_step, host_drain = pipelined(host_det, host_batch)
        r = alternate({'device resize (source_size)': lambda: dev_det.infer(src),
                       'host cv2 resize': lambda: host_det.infer(host_batch()),
                       'device resize, pipelined': dev_step,
                       'host cv2 resize, pipelined': host_step}, a.seconds, a.rounds)
        dev_drain()
        host_drain()
        for name, ms in r.items():
            emit(dict(part='c end to end', source='%s %dx%d' % (kind, w, h), arm=name, ms_per_batch=ms, h2d_MB=round(
                (dev_det.h2d_bytes if name.startswith('device') else host_det.h2d_bytes) / 1e6, 1)))
    emit(dict(cv2_threads=cv2.getNumThreads(), cpu_count=os.cpu_count()))


if __name__ == '__main__':
    main()
