# -*- coding: utf-8 -*-
"""What the input transform of the uint8 path costs and saves, on the card at hand (a script, not a test):

    python tests/debug_input_transform_timing.py [--parent DIR [--bench-only]] [--seconds 0.6]

1. TL_L and TL_S, 1280x720, batch 8 and 1, CUDA-graph replay: uint8 frames under the TrafficLight transform against the float32 NCHW
   tensor the host pipeline makes of them (device-resident input: the forward alone).
2. End to end from pinned host frames (TL_L): StreamingDetector(input_pipeline=p) against host normalisation (numpy) + float32 upload +
   forward + detect, per batch.
3. One TL_L training step (forward + loss + backward), uint8 batch against float32 batch.
4. --parent DIR (a built checkout of the parent commit): bench.py of both trees, alternated, three runs per arm, for WIDERFACE_S,
   TT100K_L, WIDERFACE_XS_4K and WIDERFACE_L_train, and --dump-outputs of the inference lines compared byte for byte.

Arms alternate inside every measurement; a window is at least --seconds long and ends in a device synchronise.  Prints the card's name,
power limit and maximal SM clock first: an absolute number means nothing without them."""
import argparse
import filecmp
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path[:0] = [HERE, ROOT, os.path.join(ROOT, 'lfd-a-light-and-fast-detector_b200')]

import synth  # noqa: E402
import tl_s  # noqa: E402
from helpers import synth_model  # noqa: E402
from test_input_transform_host import tl_val_pipeline  # noqa: E402


def emit(record):
    print(json.dumps(record), flush=True)


def window(fn, seconds):
    """ms per call over a window of at least `seconds` (host clock around work that ends in a synchronise)."""
    fn()
    torch.cuda.synchronize()
    n, t0 = 0, time.perf_counter()
    while True:
        for _ in range(10):
            fn()
        n += 10
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        if dt >= seconds:
            return dt / n * 1e3


def alternate(arms, seconds, rounds=3):
    """{arm: [ms per call, one per round]}, the arms taking turns."""
    out = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            out[k].append(round(window(fn, seconds), 4))
    return out


def host_f32(x8):
    return np.ascontiguousarray(np.stack([tl_val_pipeline({'image': f})['image'] for f in x8]).transpose(0, 3, 1, 2))


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
    H, W = 720, 1280
    for name in () if a.bench_only else ('TL_L', 'TL_S'):
        # (a low classification bias: the synthetic heads must not flood the post-process with candidates)
        model = (tl_s.synth_model(cls_bias=-6.0)[0] if name == 'TL_S' else synth_model(name, cls_bias=-6.0)[0]).cuda().eval()
        model.set_input_transform(tl_val_pipeline)
        for n in (8, 1):
            x8 = np.stack([synth.synth_image_u8(H, W, seed=i) for i in range(n)])
            d8, d32 = torch.from_numpy(x8).cuda(), torch.from_numpy(host_f32(x8)).cuda()
            plan = model.inference_plan(n, H, W, d8.device)
            if not plan.autotuned:
                plan.autotune()
            with torch.no_grad():
                r = alternate({'u8+transform': lambda: plan.forward(d8, use_graph=True), 'f32': lambda: plan.forward(d32, use_graph=True)}, a.seconds)
            emit(dict(what='forward, graph replay, device-resident input', model=name, batch=n, ms=r))
        if name != 'TL_L':         # (the synthetic TL_S head floods the post-process on these frames: its end-to-end line is not measured)
            continue
        # end to end from pinned host frames, batch 8
        from lfd.pipeline import StreamingDetector
        n = 8
        frames = [torch.from_numpy(np.stack([synth.synth_image_u8(H, W, seed=10 * b + i) for i in range(n)])).pin_memory() for b in range(3)]
        det = StreamingDetector(model, n, H, W, 0.3, 0.3, input_pipeline=tl_val_pipeline)
        k = [0]

        def streaming():
            k[0] += 1
            det.infer(frames[k[0] % 3])

        def host_path():
            k[0] += 1
            x = torch.from_numpy(host_f32(frames[k[0] % 3].numpy())).cuda()
            with torch.no_grad():
                out = model(x)
            model.detect(out, [H] * n, [W] * n, [1.0] * n, 0.3, 0.3)[3].cpu()

        def streaming_pipelined():
            s = [det.submit(frames[i % 3]) for i in range(2)]
            for i in range(8):
                det.collect(s[i])
                s.append(det.submit(frames[i % 3]))
            det.collect(s[8]), det.collect(s[9])

        r = alternate({'StreamingDetector(input_pipeline), one batch in flight': streaming, 'host normalise + f32 upload + forward + detect': host_path},
                      a.seconds, rounds=2)
        r['StreamingDetector(input_pipeline), pipelined, per batch'] = [round(window(streaming_pipelined, a.seconds) / 10, 4)]
        emit(dict(what='end to end from pinned host frames, per batch of 8', model=name, ms=r))
        del det
    if not a.bench_only:
        training_step(a)
    if a.parent:
        bench_against(a)


def training_step(a):
    n, h, w = 8, 640, 640
    ann = synth.synth_annotations(n, h, w, 1, seed=5)
    x8 = np.stack([synth.synth_image_u8(h, w, seed=i) for i in range(n)])
    model = synth_model('TL_L', cls_bias=-2.0)[0].cuda().train()
    model.set_input_transform(tl_val_pipeline)
    d8, d32 = torch.from_numpy(x8).cuda(), torch.from_numpy(host_f32(x8)).cuda()

    def step(x):
        ld = model.get_loss(model(x), ann)
        model._flat_parameters.grad.zero_()
        ld['loss'].backward()

    r = alternate({'u8+transform': lambda: step(d8), 'f32': lambda: step(d32)}, a.seconds)
    emit(dict(what='TL_L training step, 8 x 640 x 640, device-resident batch', ms=r))


def bench_against(a):
    if True:
        with tempfile.TemporaryDirectory() as tmp:
            for cfg in a.configs.split(','):
                res = {'this': [], 'parent': []}
                for rnd in range(3):
                    for arm, root in (('this', ROOT), ('parent', os.path.abspath(a.parent))):
                        cmd = [sys.executable, os.path.join(root, 'bench.py'), '--gpus', '1', '--steps', str(a.bench_steps), '--warmup', '10', '--config', cfg,
                               '--no-cpu-baseline']
                        dump = os.path.join(tmp, '%s_%s' % (arm, cfg))
                        if rnd == 0 and not cfg.endswith('_train'):
                            cmd += ['--dump-outputs', dump]
                        p = subprocess.run(cmd, capture_output=True, text=True, cwd=tmp)
                        line = [l for l in p.stdout.splitlines() if l.startswith('{')]
                        assert p.returncode == 0 and line, p.stderr[-2000:]
                        j = json.loads(line[-1])
                        res[arm].append({k: j[k] for k in j if k in ('value', 'metric', 'unit', 'ms_per_step', 'images_per_s', 'step_ms')})
                same = None
                if not cfg.endswith('_train'):
                    d1, d2 = (os.path.join(tmp, '%s_%s' % (arm, cfg)) for arm in ('this', 'parent'))
                    names = sorted(os.listdir(d1))
                    same = names == sorted(os.listdir(d2)) and bool(names) and all(filecmp.cmp(os.path.join(d1, f), os.path.join(d2, f), shallow=False) for f in names)
                emit(dict(what='bench.py, alternated with the parent', config=cfg, outputs_byte_identical=same, runs=res))


if __name__ == '__main__':
    main()
