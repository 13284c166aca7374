"""TrafficLight LFD-S on the 48-wide conv kernel against the same weights zero-padded to a 64-channel model (which runs on the 64-wide
kernels and computes the same bits) and TL_L, graph-replayed at 1280x720 on u8 input, batch 8 and batch 1, in alternating windows of
>= 0.5 s; then lfd_plan_profile per op for the 48-wide layers against their padded counterparts.

    python tests/debug_tl_s_timing.py [--rounds 5] [--out DIR]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'lfd-a-light-and-fast-detector_b200'), os.path.join(ROOT, 'tests')]
import numpy as np  # noqa: E402
import torch  # noqa: E402

import tl_s  # noqa: E402
from helpers import synth_model  # noqa: E402
from lfd import _native as nat  # noqa: E402
from test_gpu_tl_s import _padded_model  # noqa: E402


def card():
    return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                          capture_output=True, text=True, timeout=30).stdout.strip()


def window_ms(plan, x, min_s=0.5):
    """Mean ms per graph replay over a window of at least min_s seconds."""
    n, total = 0, 0.0
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = 20
    while total < min_s * 1e3:
        e0.record()
        for _ in range(reps):
            plan.forward(x, use_graph=True)
        e1.record()
        torch.cuda.synchronize()
        total += e0.elapsed_time(e1)
        n += reps
        reps *= 2
    return total / n


def profile_ops(plan, x, reps=10):
    buf = (C.c_float * plan.num_launches)()
    acc = np.zeros(plan.num_launches)
    for r in range(reps + 1):
        nat.check(nat.lib().lfd_plan_profile(plan.handle, nat.ptr(x), nat.INPUT_U8_NHWC, nat.ptr(plan.workspace), nat.ptr(plan.cls_out),
                                             nat.ptr(plan.reg_out), buf, nat.stream_ptr()))
        if r:
            acc += np.frombuffer(buf, dtype=np.float32)
    return acc / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    dev = torch.device('cuda', 0)
    print('card:', card())
    s_model, sd = tl_s.synth_model()
    models = {'TL_S': s_model.to(dev), 'TL_S padded to 64': _padded_model(sd).to(dev), 'TL_L': synth_model('TL_L')[0].to(dev)}
    out = dict(card=card(), lines={})
    H, W = 720, 1280
    for N in (8, 1):
        x = torch.randint(0, 256, (N, H, W, 3), generator=torch.Generator().manual_seed(1), dtype=torch.uint8).to(dev)
        plans = {k: m.inference_plan(N, H, W, dev, exact=True) for k, m in models.items()}
        for p in plans.values():
            p.autotune()
        times = {k: [] for k in plans}
        with torch.no_grad():
            for p in plans.values():
                window_ms(p, x, 0.2)                               # warm-up
            for _ in range(a.rounds):
                for k, p in plans.items():                         # alternating windows
                    times[k].append(window_ms(p, x))
        for k, t in times.items():
            t = sorted(t)
            line = '%-18s batch %d: median %.4f ms per forward (min %.4f, max %.4f) -> %.0f images/s' % (k, N, t[len(t) // 2], t[0], t[-1],
                                                                                                          N / t[len(t) // 2] * 1e3)
            print(line)
            out['lines']['%s b%d' % (k, N)] = t
        if N == 8:
            s, p = plans['TL_S'], plans['TL_S padded to 64']
            ts, tp = profile_ops(s, x), profile_ops(p, x)
            assert len(s._ops) == len(p._ops) == s.num_launches == p.num_launches
            print('per op, TL_S (48-wide) vs padded (64-wide), batch 8, mean of 10 eager profiled passes:')
            rows = []
            for i, (o, q) in enumerate(zip(s._ops, p._ops)):
                if o['kind'] in (nat.OP_STEM0, nat.OP_CONV) and 48 in (o['Cin'], o['Cout']):
                    what = 'k%ds%d %d->%d%s%s' % (o['ksize'], o['stride'], o['Cin'], o['Cout'], ' tail %d' % o['tail_cout'] if o.get('tail_cout') else '',
                                                ' +shortcut' if o.get('ds_cout') else '')
                    rows.append((what, ts[i] * 1e3, tp[i] * 1e3))
                    print('  op %2d %-28s %7.1f us vs %7.1f us (%.2fx)' % (i, what, ts[i] * 1e3, tp[i] * 1e3, ts[i] / tp[i]))
            print('  sum of these ops: %.1f us vs %.1f us' % (sum(r[1] for r in rows), sum(r[2] for r in rows)))
            out['ops'] = rows
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, 'tl_s_timing.json'), 'w') as f:
            json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
