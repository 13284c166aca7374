# -*- coding: utf-8 -*-
"""Measurement aid (GPU only): the fused four-conv stem (LFD_OP_STEM4) against the two-kernel path on WIDERFACE-S 720p x8.

    python tests/debug_stem_fusion.py [--rounds 3] [--steps 200] [--trace]

Alternates the fused and the two-kernel plan of the same model in one process and prints, per run: the per-op stem times
(lfd_plan_profile, eager, mean of 5), the CUDA-graph step time of the forward (events over --steps replays), the fused op's true
FLOPs and bytes with its achieved TFLOP/s, and the workspace of both plans.  The card, its power limit and maximum SM clock are
printed first (nvidia-smi, read-only query).  --trace (LFD_B200_TRACE=1 build) prints the clock64() phases of CTA 0 of the
fused kernel: patch wait, stem0/1 phase, plane barrier, stem2 MMAs, tail, store."""
import argparse
import ctypes as C
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path[:0] = [HERE, ROOT, os.path.join(ROOT, 'lfd-a-light-and-fast-detector_b200')]
import numpy as np  # noqa: E402
import torch  # noqa: E402

from helpers import synth_model  # noqa: E402
from lfd import _native as nat  # noqa: E402
from lfd._engine import InferencePlan  # noqa: E402

N, H, W = 8, 720, 1280


def stem4_work(n, h, w):
    """(flops, bytes) the fused kernel really does / moves: all four convs (stem0 with K = 27) at their own resolutions,
    the u8 image in, the stem3 map out, the weights once."""
    h1, w1 = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    h2, w2 = (h1 - 1) // 2 + 1, (w1 - 1) // 2 + 1
    px1, px2 = n * h1 * w1, n * h2 * w2
    flops = 2.0 * (px1 * 64 * 27 + px1 * 64 * 64 + px2 * 64 * 64 * 9 + px2 * 64 * 64)
    nbytes = n * h * w * 3 + px2 * 64 * 2 + 2 * (27 * 64 + 64 * 64 + 9 * 64 * 64 + 64 * 64)
    return flops, nbytes


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return 'nvidia-smi unavailable (%s)' % e


def profile_ops(plan, x, reps=5):
    n = plan.num_launches
    buf = (C.c_float * n)()
    acc = np.zeros(n)
    for r in range(reps + 1):
        nat.check(nat.lib().lfd_plan_profile(plan.handle, nat.ptr(x), nat.INPUT_U8_NHWC, nat.ptr(plan.workspace), nat.ptr(plan.cls_out),
                                             nat.ptr(plan.reg_out), buf, nat.stream_ptr()))
        if r:
            acc += np.frombuffer(buf, dtype=np.float32)
    return acc / reps


def step_ms(plan, x, steps):
    for _ in range(5):
        plan.forward(x, use_graph=True)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        plan.forward(x, use_graph=True)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def show_trace(plan, x):
    buf = torch.zeros((4, 32, 4), dtype=torch.int64, device='cuda')
    nat.lib().lfd_debug_set_trace(nat.ptr(buf))
    op = plan._op_array[0]
    nat.check(nat.lib().lfd_run_op(C.byref(op), nat.ptr(x), nat.INPUT_U8_NHWC, nat.ptr(plan.workspace), None, None, plan.P, plan.cls_channels,
                                   nat.CONV_UMMA, nat.stream_ptr()))
    torch.cuda.synchronize()
    nat.lib().lfd_debug_set_trace(None)
    t = buf.cpu().numpy().astype(np.int64)
    if not t.any():
        print('trace buffer empty: rebuild with LFD_B200_TRACE=1')
        return
    print('fused stem, CTA 0, cycles per tile (warpgroup: patch wait | stem0/1 | plane barrier | stem2 MMAs | tail | store):')
    for wg in range(2):
        ph = []
        for lt in range(2, 16):
            c, ep = t[1 + wg, lt], t[3, wg + 2 * lt]
            if c[0] == 0 or ep[2] == 0:
                break
            ph.append([c[1] - c[0], c[2] - c[1], c[3] - c[2], ep[3] - c[3], ep[0] - ep[3], ep[2] - ep[0]])
        if ph:
            m = np.mean(ph, axis=0)
            print('  wg%d (tiles 2..%d): %s  = %d' % (wg, 1 + len(ph), ' | '.join('%5d' % v for v in m), int(m.sum())))
    prod = [t[0, lt, 2] - t[0, lt, 1] for lt in range(2, 16) if t[0, lt, 2] > 0]
    if prod:
        print('  producer patch fill: %d cycles per tile' % int(np.mean(prod)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--steps', type=int, default=200)
    ap.add_argument('--trace', action='store_true')
    ap.add_argument('--shape', default='%dx%dx%d' % (N, H, W), help='NxHxW (the bench shape by default)')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('needs a GPU')
    print('card: %s' % card())
    n, h, w = (int(v) for v in args.shape.split('x'))
    model, _ = synth_model('WIDERFACE_S')
    model.cuda()
    dev = torch.device('cuda')
    plans = {'fused': InferencePlan(model, n, h, w, dev, fuse_stem=True), 'two-kernel': InferencePlan(model, n, h, w, dev, fuse_stem=False)}
    assert plans['fused']._ops[0]['kind'] == nat.OP_STEM4 and plans['two-kernel']._ops[0]['kind'] == nat.OP_STEM0
    g = torch.Generator().manual_seed(0)
    x = torch.randint(0, 256, (n, h, w, 3), dtype=torch.uint8, generator=g).cuda()
    flops, nbytes = stem4_work(n, h, w)
    print('shape %dx%dx%d: stem1 map %.1f MB' % (n, h, w, n * ((h - 1) // 2 + 1) * ((w - 1) // 2 + 1) * 128 / 1e6))
    for name, p in plans.items():
        print('%-10s workspace %.1f MB, %d launches' % (name, p.workspace_bytes / 1e6, p.num_launches))
    print('fused stem: %.1f GFLOP, %.1f MB per batch (true counts)' % (flops / 1e9, nbytes / 1e6))
    with torch.no_grad():
        for r in range(args.rounds):
            for name, p in plans.items():
                ops = profile_ops(p, x)
                stem = ops[:1] if name == 'fused' else ops[:2]
                ms = step_ms(p, x, args.steps)
                extra = '  -> %.0f TFLOP/s, %.0f GB/s' % (flops / (stem[0] * 1e-3) / 1e12, nbytes / (stem[0] * 1e-3) / 1e9) if name == 'fused' else ''
                print('round %d %-10s stem ops %s ms (sum %.3f)%s; graph step %.3f ms = %.0f images/s'
                      % (r, name, ' + '.join('%.3f' % v for v in stem), stem.sum(), extra, ms, n / (ms * 1e-3)))
        if args.trace:
            show_trace(plans['fused'], x)


if __name__ == '__main__':
    main()
