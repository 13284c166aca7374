# -*- coding: utf-8 -*-
"""What a gray (1-channel) model costs against its 3-channel twin, on the card at hand (a script, not a test):

    python tests/debug_gray_timing.py [--seconds 0.6]

WIDERFACE-S 1280x720 batch 8 (the fused 'faster' stem, word loader), device-resident frames, CUDA-graph replay: the gray model on uint8
gray frames [N,H,W] and on NV12 frames (of which it reads the Y plane), against the twin on uint8 BGR frames [N,H,W,3].  Per arm: the stem
op (lfd_plan_profile, op 0, median of 20 per window) and the graph step.  Arms alternate inside every measurement; a window is at least
--seconds long and ends in a device synchronise.  Prints the card's name, power limit and maximal SM clock first: an absolute number means
nothing without them."""
import argparse
import os
import subprocess
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path[:0] = [HERE, ROOT, os.path.join(ROOT, 'lfd-a-light-and-fast-detector_b200')]

from debug_input_transform_timing import alternate, emit  # noqa: E402
from debug_nv12_timing import stem_ms  # noqa: E402
from gray_models import gray_pair, twin_u8  # noqa: E402
from lfd import _native as nat  # noqa: E402
from nv12_oracle import nv12_frames  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--seconds', type=float, default=0.6)
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'needs the GPU: there is nothing to time without it'
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
    emit(dict(card=smi))
    name, n, H, W = 'WIDERFACE_S', 8, 720, 1280
    gray, twin = (m.cuda() for m in gray_pair(name, cls_bias=-6.0))
    nv = torch.from_numpy(nv12_frames(n, H, W, seed=1)).cuda()
    y = nv[:, :H].contiguous()
    bgr = twin_u8(y, seed=2)
    gp, tp = gray.inference_plan(n, H, W, y.device), twin.inference_plan(n, H, W, y.device)
    tp.autotune()
    gp.apply_side_ctas(tp.side_ctas)             # the same side-branch bounds: only the stem's input differs
    arms = {'gray u8': (gp, y, nat.INPUT_U8_NHWC, None), 'gray nv12 (Y plane)': (gp, nv, nat.INPUT_U8_NV12, 'nv12'),
            'bgr u8 (twin)': (tp, bgr, nat.INPUT_U8_NHWC, None)}
    stem = gp._ops[0]
    r = {k: [] for k in arms}
    for _ in range(3):
        for k, (p, x, fmt, _) in arms.items():
            r[k].append(round(stem_ms(p, x, fmt), 4))
    emit(dict(what='stem op (lfd_plan_profile, median of 20 per window)', model=name, batch=n, size='%dx%d' % (W, H),
              op='STEM4' if stem['kind'] == nat.OP_STEM4 else 'STEM0', word_loader=W % 4 == 0,
              input_bytes={k: int(x[:, :H].numel()) for k, (_, x, _, _) in arms.items()}, ms=r))

    def step(p, x, f):
        return lambda: p.forward(x, use_graph=True, frame_format=f)
    with torch.no_grad():
        r = alternate({k: step(p, x, f) for k, (p, x, _, f) in arms.items()}, a.seconds)
    emit(dict(what='graph step, device-resident frames', model=name, batch=n, size='%dx%d' % (W, H), ms=r))


if __name__ == '__main__':
    main()
