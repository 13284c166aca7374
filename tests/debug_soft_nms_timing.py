"""Timing aid: device Soft-NMS (lfd.model.utils.soft_nms, one CTA) against the reference's compiled CPU soft_nms_cpu (oracle/_ref) on random
boxes at K = 1k / 4k / 8k, linear and gaussian; then lfd_postprocess_soft_nms on WIDERFACE_S outputs of a 1280x720 batch of 8 next to the
greedy lfd_postprocess.  Prints the card, its power limit and max SM clock with the numbers.

    python tests/debug_soft_nms_timing.py
"""
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'lfd-a-light-and-fast-detector_b200'), os.path.join(ROOT, 'tests')]
import numpy as np
import torch

from helpers import synth_model
from lfd.model.utils import soft_nms
from oracle import build_ref


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception as e:
        q = 'nvidia-smi unavailable (%s)' % e
    return q or torch.cuda.get_device_name(0)


def random_dets(n, rng):
    d = np.concatenate([rng.uniform(0, 1000, (n, 2)), rng.uniform(4, 120, (n, 2)), rng.uniform(0.01, 1, (n, 1))], 1).astype(np.float32)
    d[:, 2:4] += d[:, :2]
    return d


def gpu_ms(fn, reps=5):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def main():
    print('card: %s' % card())
    ref = build_ref.load_module()
    rng = np.random.RandomState(0)
    print('%6s %9s %8s %12s %12s' % ('K', 'method', 'rows', 'device ms', 'ref CPU ms'))
    for n in (1000, 4000, 8000):
        d = random_dets(n, rng)
        t = torch.from_numpy(d).cuda()
        for method, code in (('linear', 1), ('gaussian', 2)):
            rows = len(soft_nms(t, 0.3, method)[1])
            dev = gpu_ms(lambda: soft_nms(t, 0.3, method))
            cpu = float('nan')
            if ref is not None:
                t0 = time.perf_counter()
                ref.soft_nms(torch.from_numpy(d), 0.3, code, 0.5, 1e-3)
                cpu = (time.perf_counter() - t0) * 1e3
            print('%6d %9s %8d %12.2f %12.1f' % (n, method, rows, dev, cpu))
    # the post-process of a WIDERFACE_S 1280x720 batch of 8
    N, H, W = 8, 720, 1280
    model, _ = synth_model('WIDERFACE_S', cls_bias=-1.0)
    model.cuda().eval()
    plan = model.inference_plan(N, H, W, torch.device('cuda', 0))
    for i, hw in enumerate(plan.level_sizes):
        model._head_indexes_to_feature_map_sizes[i] = hw
    x = torch.randint(0, 256, (N, H, W, 3), generator=torch.Generator().manual_seed(1), dtype=torch.uint8).cuda()
    with torch.no_grad():
        cls, reg = plan.forward(x, use_graph=False)
    cls, reg = cls.float().contiguous(), reg.float().contiguous()
    for thr in (0.3, 0.2):
        for cfg in (dict(type='nms', iou_thr=0.3), dict(type='soft_nms', iou_thr=0.3, method='linear'),
                    dict(type='soft_nms', iou_thr=0.3, method='gaussian')):
            model._nms_cfg = cfg
            pp = model.post_plan(N, plan.level_sizes, cls.device)
            pp.set_meta([W] * N, [H] * N, [1.0] * N)
            ms = gpu_ms(lambda: pp.run(cls, reg, thr, 0.3))
            cnt = pp.count[:N].tolist()
            print('WIDERFACE_S %dx%d batch %d thr %.2f %-8s %-8s: %8.3f ms, candidates kept per image max %d' % (
                W, H, N, thr, cfg['type'], cfg.get('method', ''), ms, max(cnt)))


if __name__ == '__main__':
    main()
