# -*- coding: utf-8 -*-
"""What NV12 input costs and saves, on the card at hand (a script, not a test):

    python tests/debug_nv12_timing.py [--parent DIR [--bench-only]] [--seconds 0.6]

1. Device-resident frames, NV12 against the converted uint8 BGR frames, CUDA-graph replay: the stem op (lfd_plan_profile, op 0) and the
   graph step, for WIDERFACE_S 1280x720 batch 8 (fused stem, word loader), TL_L 1280x720 batch 8 (TrafficLight transform) and TT100K_L
   1920x1080 batch 16.
2. End to end from pinned host frames, the same configs: StreamingDetector(frame_format='nv12') against frame_format='bgr', per batch
   with one batch in flight and pipelined, and the host -> device copy of one batch alone (bytes, ms, GB/s).
3. --parent DIR (a built checkout of the parent commit): bench.py of both trees, alternated, three runs per arm, for WIDERFACE_S,
   TT100K_L, WIDERFACE_XS_4K and WIDERFACE_L_train, and --dump-outputs of the inference lines compared byte for byte
   (debug_input_transform_timing.py's comparison).

Arms alternate inside every measurement; a window is at least --seconds long and ends in a device synchronise.  Prints the card's name,
power limit and maximal SM clock first: an absolute number means nothing without them."""
import argparse
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path[:0] = [HERE, ROOT, os.path.join(ROOT, 'lfd-a-light-and-fast-detector_b200')]

from debug_input_transform_timing import alternate, bench_against, emit  # noqa: E402
from helpers import synth_model  # noqa: E402
from lfd import _native as nat  # noqa: E402
from nv12_oracle import nv12_frames, nv12_oracle  # noqa: E402
from test_input_transform_host import tl_val_pipeline  # noqa: E402

CASES = [('WIDERFACE_S', 8, 720, 1280, None), ('TL_L', 8, 720, 1280, tl_val_pipeline), ('TT100K_L', 16, 1080, 1920, None)]


def stem_ms(plan, x, fmt, reps=20):
    """median over `reps` eager profiled forwards of op 0's time (ms)."""
    ms = (C.c_float * nat.lib().lfd_plan_num_launches(plan.handle))()
    got = []
    for _ in range(reps):
        with torch.cuda.device(plan.device):
            nat.check(nat.lib().lfd_plan_profile(plan.handle, nat.ptr(x), fmt, nat.ptr(plan.workspace), nat.ptr(plan.cls_out), nat.ptr(plan.reg_out),
                                                 ms, nat.stream_ptr()))
        got.append(ms[0])
    return float(np.median(got))


def device_side(a):
    for name, n, H, W, pipeline in CASES:
        model = synth_model(name, cls_bias=-6.0)[0].cuda().eval()
        model.set_input_transform(pipeline)
        nv = nv12_frames(n, H, W, seed=1)
        dnv, dbgr = torch.from_numpy(nv).cuda(), torch.from_numpy(nv12_oracle(nv)).cuda()
        plan = model.inference_plan(n, H, W, dnv.device)
        if not plan.autotuned:
            plan.autotune()
        stem = plan._ops[0]
        r = {'nv12': [], 'bgr': []}
        for _ in range(3):
            r['nv12'].append(round(stem_ms(plan, dnv, nat.INPUT_U8_NV12), 4))
            r['bgr'].append(round(stem_ms(plan, dbgr, nat.INPUT_U8_NHWC), 4))
        emit(dict(what='stem op (lfd_plan_profile, median of 20 per window)', model=name, batch=n, size='%dx%d' % (W, H),
                  op='STEM4' if stem['kind'] == nat.OP_STEM4 else 'STEM0', word_loader=W % 4 == 0, ms=r))
        with torch.no_grad():
            r = alternate({'nv12': lambda: plan.forward(dnv, use_graph=True, frame_format='nv12'),
                           'bgr': lambda: plan.forward(dbgr, use_graph=True)}, a.seconds)
        emit(dict(what='graph step, device-resident frames', model=name, batch=n, size='%dx%d' % (W, H), ms=r))
        del plan


def end_to_end(a):
    from lfd.pipeline import StreamingDetector
    for name, n, H, W, pipeline in CASES:
        model = synth_model(name, cls_bias=-6.0)[0].cuda().eval()
        nvs = [nv12_frames(n, H, W, seed=10 * b) for b in range(3)]
        host = {'nv12': [torch.from_numpy(f).pin_memory() for f in nvs],
                'bgr': [torch.from_numpy(nv12_oracle(f)).pin_memory() for f in nvs]}
        dets = {f: StreamingDetector(model, n, H, W, 0.3, 0.3, input_pipeline=pipeline, frame_format=f) for f in ('nv12', 'bgr')}
        k = [0]

        def one(fmt):
            def run():
                k[0] += 1
                dets[fmt].infer(host[fmt][k[0] % 3])
            return run

        def pipelined(fmt):
            def run():
                d, fr = dets[fmt], host[fmt]
                s = [d.submit(fr[i % 3]) for i in range(2)]
                for i in range(8):
                    d.collect(s[i])
                    s.append(d.submit(fr[i % 3]))
                d.collect(s[8]), d.collect(s[9])
            return run

        def copy(fmt):
            def run():
                k[0] += 1
                dets[fmt].stage_input(0, host[fmt][k[0] % 3])
            return run

        r1 = alternate({f: one(f) for f in dets}, a.seconds, rounds=3)
        r2 = alternate({f: pipelined(f) for f in dets}, a.seconds, rounds=3)
        r2 = {f: [round(v / 10, 4) for v in vs] for f, vs in r2.items()}
        r3 = alternate({f: copy(f) for f in dets}, a.seconds, rounds=3)
        gbps = {f: [round(dets[f].h2d_bytes / (v * 1e-3) / 1e9, 2) for v in vs] for f, vs in r3.items()}
        emit(dict(what='end to end from pinned host frames, per batch', model=name, batch=n, size='%dx%d' % (W, H),
                  h2d_bytes={f: dets[f].h2d_bytes for f in dets}, one_in_flight_ms=r1, pipelined_ms=r2, h2d_copy_ms=r3, h2d_gbps=gbps))
        del dets


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--parent', default=None)
    ap.add_argument('--seconds', type=float, default=0.6)
    ap.add_argument('--bench-steps', type=int, default=200)
    ap.add_argument('--configs', default='WIDERFACE_S,TT100K_L,WIDERFACE_XS_4K,WIDERFACE_L_train', help='bench.py workloads compared with --parent')
    ap.add_argument('--bench-only', action='store_true', help='only the bench.py comparison with --parent')
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'needs the GPU: there is nothing to time without it'
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
    emit(dict(card=smi))
    if not a.bench_only:
        device_side(a)
        end_to_end(a)
    if a.parent:
        bench_against(a)


if __name__ == '__main__':
    main()
