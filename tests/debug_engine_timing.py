# -*- coding: utf-8 -*-
"""What running a model file through the C ABI costs against the Python plan it was exported from (a script, not a test):

    python tests/debug_engine_timing.py [--seconds 0.6]

WIDERFACE_S, 1280x720, batch 8, uint8 BGR frames resident on the device, autotuned export: one batch is
  engine -- lfd_engine_detect with use_graph (the forward's CUDA graph, then the post-process), the file's own kernels;
  plan   -- InferencePlan.forward(use_graph=True) and PostPlan.run on the same frames, the same work from Python.
The arms alternate, three windows each, every window at least --seconds long and ending in a device synchronise.  Both launch the same
kernels (the launch count is printed), so the expectation is equal times.  Prints the card's name, power limit and maximal SM clock
first: an absolute number means nothing without them."""
import argparse
import os
import subprocess
import sys
import tempfile

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path[:0] = [HERE, ROOT, os.path.join(ROOT, 'lfd-a-light-and-fast-detector_b200')]

from debug_input_transform_timing import alternate, emit  # noqa: E402
from engine_file import Engine  # noqa: E402
from helpers import synth_model  # noqa: E402
from lfd import _native as nat  # noqa: E402
from lfd.deployment import export_model  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--seconds', type=float, default=0.6)
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'needs the GPU: there is nothing to time without it'
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
    emit(dict(card=smi))
    name, n, H, W = 'WIDERFACE_S', 8, 720, 1280
    model = synth_model(name, cls_bias=-6.0)[0].cuda().eval()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, 'model.lfd')
        plan, post = export_model(model, path, n, H, W, classification_threshold=0.3)
        eng = Engine(open(path, 'rb').read())
    nat.check(eng.bind())
    x = torch.randint(0, 256, (n, H, W, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(1)).cuda()
    post.set_meta([W] * n, [H] * n, [1.0] * n)

    def python_plan():
        cls, reg = plan.forward(x, use_graph=True)
        post.run(cls, reg)

    with torch.no_grad():
        r = alternate({'engine': lambda: eng.detect_raw(x, nat.INPUT_U8_NHWC, H, W), 'plan': python_plan}, a.seconds)
    torch.cuda.synchronize()
    emit(dict(what='one batch: forward graph + post-process, device-resident uint8 frames', model=name, batch=n, size='%dx%d' % (W, H),
              launches=dict(engine=eng.num_launches(), plan=plan.num_launches), ms=r,
              range_ms={k: [min(v), max(v)] for k, v in r.items()}))


if __name__ == '__main__':
    main()
