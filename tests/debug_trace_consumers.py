# -*- coding: utf-8 -*-
"""Debug aid: the clock64() timeline of CTA 0 of one wgmma conv launch, with the columns the kernel stamps (LFD_B200_TRACE=1 build):
the producer per stage, each consumer warpgroup's MMA phase per tile and the epilogue of every tile store.

    python tests/debug_trace_consumers.py op0 op1 3x3s2 ...

opN = op N of the WIDERFACE-S 720p b8 plan with the two-launch stem (0 = fused stem0+stem1, 1 = fused stem2+stem3); other names are the stand-alone convs of
debug_trace.CASES.  The buffer layout is the one in conv_umma.cu (LFD_TRACE): [4 roles][32 entries][4 slots]."""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [HERE]
import torch  # noqa: E402

from debug_trace import CASES, trace_plan_op  # noqa: E402
from gpu_ops import run_conv  # noqa: E402
from lfd import _native as nat  # noqa: E402
from test_gpu_conv import _make  # noqa: E402


def rows(t):
    """(title, column names, [entries]) per stamped role; the epilogue entries of the two warpgroups are interleaved (2 * store + wg)."""
    out = [('producer (per stage)', 'wait_empty got_empty issued arrived_full (stem: stored next_fetch_issued)', t[0]),
           ('wg0 MMA phase (per tile)', 'wait_full got_full main_mma_done tail_mma_done', t[1]),
           ('wg1 MMA phase (per tile)', 'wait_full got_full main_mma_done tail_mma_done', t[2])]
    for wg in range(2):
        out.append(('wg%d epilogue (per store)' % wg, 'store_entry after_bulk_wait_read tma_issued -', t[3, wg::2]))
    return out


def show(t, title, n=12):
    t0 = int(t[t > 0].min())
    print('== %s' % (title,))
    for name, cols, r in rows(t):
        print('  %s  [%s]' % (name, cols))
        for i in range(min(n, r.shape[0])):
            if int(r[i].max()) == 0:
                break
            print('    %2d  %s' % (i, '  '.join('%7d' % (int(v) - t0 if int(v) > 0 else -1) for v in r[i])))


def main():
    args = sys.argv[1:] or ['op0', 'op1']
    for name in args:
        if name.startswith('op'):
            t, row = trace_plan_op(int(name[2:]))
            show(t, 'plan op %s %s' % (name, row))
            continue
        case = CASES[name]
        x, w, scale, shift, res = _make(case)
        buf = torch.zeros((4, 32, 4), dtype=torch.int64, device='cuda')
        run_conv(x, w, scale, shift, case[6], case[7], res=res)          # warm-up (weights / L2)
        nat.lib().lfd_debug_set_trace(nat.ptr(buf))
        _, _, q = run_conv(x, w, scale, shift, case[6], case[7], res=res)
        nat.lib().lfd_debug_set_trace(None)
        show(buf.cpu(), '%s %s plan=%s' % (name, case, q))


if __name__ == '__main__':
    main()
