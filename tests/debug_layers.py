# -*- coding: utf-8 -*-
"""Debug aid (not a test): per-layer comparison of the native plan against the bf16-emulated oracle.

    python tests/debug_layers.py WIDERFACE_S [simt|umma]
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [HERE, os.path.dirname(HERE), os.path.join(os.path.dirname(HERE), 'lfd-a-light-and-fast-detector_b200')]
import torch  # noqa: E402

import synth  # noqa: E402
from helpers import load_golden, synth_model, rel_err  # noqa: E402
from lfd import _native as nat  # noqa: E402
from lfd._engine import InferencePlan  # noqa: E402
from oracle import lfd_oracle as orc  # noqa: E402


def oracle_key(name):
    import re
    m = re.match(r'stem(\d+)$', name)
    if m:
        return '_backbone._stem.%d' % (3 * int(m.group(1)))
    m = re.match(r's(\d+)b(\d+)_(c0|out|id)$', name)
    if m:
        sfx = {'c0': '._conv1', 'out': '._conv2', 'id': '._downsample.0'}[m.group(3)]
        return '_backbone.stage%s.%s%s' % (m.group(1), m.group(2), sfx)
    m = re.match(r'neck(\d+)$', name)
    if m:
        return '_neck.neck%s.0' % m.group(1)
    m = re.match(r'h(\d+)([mcr])_(raw|act)(\d+)$', name)
    if m:
        path = {'m': 'merge_path', 'c': 'classification_path', 'r': 'regression_path'}[m.group(2)]
        return '_head.head%s_%s.%d:%s' % (m.group(1), path, 3 * int(m.group(4)), m.group(3))
    return None


def main():
    name = sys.argv[1] if len(sys.argv) > 1 else 'WIDERFACE_S'
    impl = nat.CONV_SIMT if (len(sys.argv) > 2 and sys.argv[2] == 'simt') else nat.CONV_UMMA
    g = load_golden('forward_%s.pt' % name)
    model, sd = synth_model(name, cls_bias=g['cls_bias'], seed=g['seed'])
    model.cuda()
    x = synth.synth_input(g['N'], g['H'], g['W'])
    # reuse=False: every intermediate stays readable after the forward
    plan = InferencePlan(model, g['N'], g['H'], g['W'], torch.device('cuda'), impl, reuse=False)
    cls, reg = plan.forward(x.cuda(), use_graph=False)
    trace = {}
    ocls, oreg, _ = orc.forward(orc.CONFIGS[name], sd, x, emulate_bf16=True, trace=trace)
    for row in plan.describe():
        if row['out'] is None:
            continue
        key = oracle_key(row['out'])
        if key is None or key not in trace:
            print('%-14s (no oracle key %s)' % (row['out'], key))
            continue
        t = plan.tensor(row['out']).float().cpu().permute(0, 3, 1, 2)
        e = rel_err(t, trace[key])
        print('%-14s %-9s k%d s%d %3d->%3d %3dx%-3d  max %.2e rms %.2e %s' % (row['out'], row['kind'], row['ksize'], row['stride'], row['Cin'],
                                                                         row['Cout'], row['Ho'], row['Wo'], e[0], e[1], '' if e[0] < 2e-2 else '  <<<<'))
    print('cls', rel_err(cls.cpu(), ocls), 'reg', rel_err(reg.cpu(), oreg))


if __name__ == '__main__':
    main()
