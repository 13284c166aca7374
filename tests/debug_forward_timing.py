"""Timing aid for A/B runs of two library builds (LFD_B200_LIB): graph-replayed forward plan of one workload, CUDA events over many replays."""
import sys, os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'lfd-a-light-and-fast-detector_b200'), os.path.join(ROOT, 'tests')]
import torch
from helpers import synth_model

cfg = sys.argv[1] if len(sys.argv) > 1 else 'WIDERFACE_S'
N, H, W = (int(v) for v in (sys.argv[2:5] if len(sys.argv) > 4 else (8, 720, 1280)))
tag = sys.argv[5] if len(sys.argv) > 5 else ''
dev = torch.device('cuda', 0)
model, _ = synth_model(cfg)
model.to(dev).eval()
g = torch.Generator().manual_seed(1)
pool = [torch.randint(0, 256, (N, H, W, 3), generator=g, dtype=torch.uint8).to(dev) for _ in range(6)]
plan = model.inference_plan(N, H, W, dev)
if os.environ.get('TUNE'):
    print('autotune', plan.autotune())
with torch.no_grad():
    for r in range(3):
        for x in pool:
            plan.forward(x, use_graph=True, slot=0)
    torch.cuda.synchronize()
    best = []
    for rep in range(5):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(120):
            plan.forward(pool[i % 6], use_graph=True, slot=0)
        e1.record()
        torch.cuda.synchronize()
        best.append(e0.elapsed_time(e1) / 120)
best.sort()
print('%s %s forward %.4f ms (median of 5; min %.4f) -> %.0f img/s' % (cfg, tag, best[2], best[0], N / best[2] * 1e3))
