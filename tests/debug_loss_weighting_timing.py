# -*- coding: utf-8 -*-
"""Cost of enable_classification_weight / enable_regression_weight in the training loss, on WIDERFACE-L 640x640 with 16 crops (the
batch of bench.py --config WIDERFACE_L_train).

  unweighted  lfd_detection_loss: cls_loss_kernel + iou_loss_kernel (the two loss launches)
  weighted    lfd_loss_weight_sum (partials + final pass) + lfd_detection_loss_weighted with both switches on

Both arms run on the same device tensors: seeded network outputs of the WIDERFACE-L geometry and the targets of one assignment of
synthetic boxes.  Each arm is captured as one CUDA graph of `--iters` calls, so the host's launch rate does not enter the numbers;
graph replays are timed with CUDA events, windows alternating between the arms.  Also LFD.get_loss end to end (host included,
synchronised per window) with the switches off and on.

--dump DIR writes the gradients and loss sums of the unweighted call.  --pkg DIR imports lfd from another checkout's package directory
(whose library may predate the weighted entry points: only the unweighted arm runs then), so that two builds can be compared byte for
byte on the same inputs.

    python tests/debug_loss_weighting_timing.py [--windows 9] [--iters 200] [--out FILE.json] [--dump DIR] [--pkg DIR]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
_PKG = sys.argv[sys.argv.index('--pkg') + 1] if '--pkg' in sys.argv else os.path.join(os.path.dirname(HERE), 'lfd-a-light-and-fast-detector_b200')
sys.path[:0] = [HERE, os.path.dirname(HERE), os.path.abspath(_PKG)]
import numpy as np  # noqa: E402
import torch  # noqa: E402

import synth  # noqa: E402
from helpers import synth_model  # noqa: E402
from lfd import _native as nat  # noqa: E402


def gpu_info():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], stdout=subprocess.PIPE,
                              text=True, timeout=30).stdout.strip()
    except Exception as e:  # the numbers still stand; say what is missing
        return 'unknown (%s)' % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--windows', type=int, default=9)
    ap.add_argument('--iters', type=int, default=200)
    ap.add_argument('--out', default=None)
    ap.add_argument('--dump', default=None)
    ap.add_argument('--pkg', default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'needs a CUDA device'
    n, h, w = 16, 640, 640
    m, _ = synth_model('WIDERFACE_L', cls_bias=-2.0)
    m.cuda()
    ann = synth.synth_annotations(n, h, w, 1, seed=3, max_boxes=12)
    with torch.no_grad():
        m(synth.synth_input(1, h, w).cuda())                    # the level geometry of a 640x640 crop
    m.train()
    sizes = m._sizes()
    P = sum(a_ * b_ for a_, b_ in sizes)
    g = torch.Generator().manual_seed(2024)
    cls = (torch.randn(n, P, m._num_classes, generator=g) * 1.5 - 2.0).cuda()
    reg = torch.randn(n, P, 4, generator=g).cuda()
    cls_t, reg_t, label, counters, lv = m._assign(sizes, [b for b, _ in ann], [l for _, l in ann], cls.device)
    lc = nat.LossCfg()
    lc.N, lc.P, lc.C = cls.shape[0], cls.shape[1], m._num_classes
    lc.cls_mode, lc.reg_loss, lc.bbox_mode = nat.CLS_SIGMOID, nat.REG_IOU, nat.BBOX_SIGMOID
    lc.gamma, lc.alpha, lc.reg_eps, lc.smooth_l1_beta, lc.cls_weight, lc.reg_weight = 2.0, 0.25, 1e-6, 1.0, 1.0, 1.0
    gc, gr = torch.empty_like(cls), torch.empty_like(reg)
    sums = torch.empty(2, dtype=torch.float64, device='cuda')
    wsum = torch.empty(1, dtype=torch.float64, device='cuda')
    L = nat.lib()
    has_weighted = hasattr(L, 'lfd_detection_loss_weighted')
    if has_weighted:
        ws = torch.empty(int(L.lfd_loss_weight_sum_workspace_bytes(C.byref(lc))) // 8, dtype=torch.float64, device='cuda')
    common = [C.byref(lv), C.byref(lc)] + [nat.ptr(t) for t in (cls, reg, cls_t, reg_t, label, counters, gc, gr, sums)]

    def unweighted():
        nat.check(L.lfd_detection_loss(*common, nat.stream_ptr()))

    def weighted():
        nat.check(L.lfd_loss_weight_sum(C.byref(lc), nat.ptr(cls_t), nat.ptr(label), nat.ptr(ws), nat.ptr(wsum), nat.stream_ptr()))
        nat.check(L.lfd_detection_loss_weighted(*common, 1, 1, nat.ptr(wsum), nat.stream_ptr()))

    unweighted()
    torch.cuda.synchronize()
    if a.dump:
        os.makedirs(a.dump, exist_ok=True)
        for name, t in (('grad_cls', gc), ('grad_reg', gr), ('loss_sums', sums)):
            np.save(os.path.join(a.dump, name + '.npy'), t.cpu().numpy())
    arms = [('unweighted_us', unweighted)] + ([('weighted_us', weighted)] if has_weighted else [])
    graphs = {}
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        for name, fn in arms:
            for _ in range(3):                                 # warm-up outside the capture
                fn()
            stream.synchronize()
            graphs[name] = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graphs[name], stream=stream):
                for _ in range(a.iters):
                    fn()
    torch.cuda.synchronize()

    def window(name, iters):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        graphs[name].replay()
        e.record()
        e.synchronize()
        return s.elapsed_time(e) * 1e3 / iters       # us per call

    def get_loss_window(cw, rw, iters):
        m._enable_classification_weight, m._enable_regression_weight = cw, rw
        c, r = cls.detach().requires_grad_(True), reg.detach().requires_grad_(True)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(iters):
            m.get_loss((c, r), ann)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3 / iters    # ms per call

    for name, _ in arms:
        window(name, a.iters)
    gl = [('get_loss_off_ms', (False, False))] + ([('get_loss_on_ms', (True, True))] if has_weighted else [])
    for _, fl in gl:
        get_loss_window(fl[0], fl[1], 5)
    res = {name: [] for name, _ in arms + gl}
    for i in range(a.windows):
        for name, _ in (arms if i % 2 == 0 else arms[::-1]):
            res[name].append(window(name, a.iters))
        for name, fl in (gl if i % 2 == 0 else gl[::-1]):
            res[name].append(get_loss_window(fl[0], fl[1], 20))
    out = dict(gpu=gpu_info(), batch='WIDERFACE_L %dx%dx%d, P=%d, n_pos=%d' % (n, h, w, lc.P, int(counters[0])),
               **{k: dict(median=float(np.median(v)), min=float(np.min(v)), max=float(np.max(v))) for k, v in res.items()})
    print(json.dumps(out, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
