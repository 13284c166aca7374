# -*- coding: utf-8 -*-
"""Cost of varying frame sizes (needs a GPU): python tests/debug_variable_size_timing.py [--frames 200] [--out varsize_timing.json]

Per frame: `predict_for_single_image` on seeded 1024-wide uint8 frames whose heights vary as on WIDER FACE val, for WIDERFACE_L and
WIDERFACE_S, once with one plan per size (model.invalidate_plans() before every new size: what a plan per shape costs) and once with
the capacity plans (a new plan only at a new maximum).  Median and 95th percentile of the per-frame wall time (host clock around the
call, which ends in a device synchronise), the plans built, and the peak device memory of the pass.

Steady state: CUDA-graph replays of a 768 x 1024 frame on a 1024 x 1024 plan against a plan built for 768 x 1024, alternated in windows of
at least 0.5 s: what running below the capacity costs (the staging copy and the table update included)."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(HERE), os.path.join(os.path.dirname(HERE), 'lfd-a-light-and-fast-detector_b200'), HERE]

from helpers import synth_model  # noqa: E402
from lfd._engine import InferencePlan  # noqa: E402


def wider_heights(rng, n):
    """Heights of 1024-wide WIDER FACE val images: mostly 600 .. 1400, a few outside."""
    return np.clip(rng.normal(800, 220, size=n).round(), 320, 1536).astype(int)


def per_frame(name, frames, capacity):
    model, _ = synth_model(name, cls_bias=-2.0)
    model.cuda()
    model._classification_threshold = 0.5
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    times, built, seen = [], set(), set()
    for im in frames:
        if not capacity and im.shape[:2] not in seen:
            model.invalidate_plans()
        seen.add(im.shape[:2])
        t0 = time.perf_counter()
        model.predict_for_single_image(im, None)
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
        built |= set(model._plans)
    t = np.asarray(times) * 1e3
    return dict(median_ms=float(np.median(t)), p95_ms=float(np.percentile(t, 95)), mean_ms=float(t.mean()), plans_built=len(built),
                peak_mem_mb=torch.cuda.max_memory_allocated() / 2 ** 20)


def steady(name, seconds):
    model, _ = synth_model(name)
    model.cuda()
    dev = torch.device('cuda', 0)
    cap = InferencePlan(model, 1, 1024, 1024, dev)
    exact = InferencePlan(model, 1, 768, 1024, dev)
    x = torch.randint(0, 256, (1, 768, 1024, 3), dtype=torch.uint8, device=dev)
    for p in (cap, exact):
        for _ in range(3):
            p.forward(x, use_graph=True)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def window(p):
        reps, ms = 16, 0.0
        while True:
            e0.record()
            for _ in range(reps):
                p.forward(x, use_graph=True)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1)
            if ms >= seconds * 1e3:
                return ms / reps
            reps *= 2
    res = {'capacity_1024x1024': [], 'exact_768x1024': []}
    for _ in range(3):
        res['capacity_1024x1024'].append(window(cap))
        res['exact_768x1024'].append(window(exact))
    return {k: dict(ms_per_frame=sorted(v)[1], all=v) for k, v in res.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=200)
    ap.add_argument('--window', type=float, default=0.5)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA device')
    import subprocess
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
    rng = np.random.RandomState(2024)
    frames = [rng.randint(0, 256, size=(int(h), 1024, 3)).astype(np.uint8) for h in wider_heights(rng, a.frames)]
    out = dict(card=card, frames=a.frames, distinct_heights=len({f.shape[0] for f in frames}))
    for name in ('WIDERFACE_L', 'WIDERFACE_S'):
        out[name] = dict(plan_per_size=per_frame(name, frames, False), capacity_plan=per_frame(name, frames, True),
                         steady_state=steady(name, a.window))
    print(json.dumps(out, indent=1))
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
