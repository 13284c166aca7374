# -*- coding: utf-8 -*-
"""Debug aid: clock64() timeline of CTA 0 of one wgmma conv launch (producer / MMA issuer / epilogue per tile)."""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [HERE, os.path.dirname(HERE), os.path.join(os.path.dirname(HERE), 'lfd-a-light-and-fast-detector_b200')]
import torch  # noqa: E402

from gpu_ops import run_conv  # noqa: E402
from lfd import _native as nat  # noqa: E402
from test_gpu_conv import _make  # noqa: E402

CASES = {'3x3s1': (8, 90, 160, 64, 64, 3, 1, True, False, 0), '3x3s1res': (8, 90, 160, 64, 64, 3, 1, True, True, 0), 'flat': (8, 180, 320, 64, 64, 1, 1, True, False, 0),
         '3x3s2': (8, 180, 320, 64, 64, 3, 2, True, False, 0), 'stream': (8, 12, 20, 128, 128, 3, 1, True, False, 0)}


def trace_plan_op(index):
    """Timeline of op `index` of the WIDERFACE-S 720p b8 plan with the two-launch stem (0 = fused stem0+stem1, 1 = fused stem2+stem3)."""
    import ctypes as C
    from helpers import synth_model
    from lfd._engine import InferencePlan
    model, _ = synth_model('WIDERFACE_S')
    model.cuda()
    plan = InferencePlan(model, 8, 720, 1280, torch.device('cuda', 0), fuse_stem=False)
    x = torch.randint(0, 256, (8, 720, 1280, 3), dtype=torch.uint8, device='cuda')
    plan.forward(x, use_graph=False)
    torch.cuda.synchronize()
    buf = torch.zeros((4, 32, 4), dtype=torch.int64, device='cuda')
    nat.lib().lfd_debug_set_trace(nat.ptr(buf))
    op = plan._op_array[index]
    nat.check(nat.lib().lfd_run_op(C.byref(op), nat.ptr(x), nat.INPUT_U8_NHWC, nat.ptr(plan.workspace), None, None, plan.P, plan.cls_channels,
                                   nat.CONV_UMMA, nat.stream_ptr()))
    torch.cuda.synchronize()
    nat.lib().lfd_debug_set_trace(None)
    return buf.cpu(), plan.describe()[index]


def show(t, title):
    t0 = int(t[t > 0].min())
    rel = (t - t0).clamp(min=-1)
    print('== %s' % (title,))
    for role, rn, cols in ((0, 'producer', 'wait_empty got_empty issued arrived_full'), (1, 'mma', 'wait_tempty got_tempty first_full committed'),
                           (2, 'epilogue', 'wait_tfull got_tfull tmem_read_done stored'),
                           (3, 'epilogue detail', 'res_ready after_bar1 store_loop_done -')):
        print('  %s  [%s]' % (rn, cols))
        for i in range(12):
            if int(t[role, i].max()) == 0:
                break
            print('    %2d  %s' % (i, '  '.join('%7d' % int(v) for v in rel[role, i])))


def main():
    args = sys.argv[1:] or list(CASES)
    for name in [a for a in args if a.startswith('op')]:
        t, row = trace_plan_op(int(name[2:]))
        show(t, 'plan op %s %s' % (name, row))
    for name in [a for a in args if not a.startswith('op')]:
        case = CASES[name]
        x, w, scale, shift, res = _make(case)
        buf = torch.zeros((4, 32, 4), dtype=torch.int64, device='cuda')
        run_conv(x, w, scale, shift, case[6], case[7], res=res)          # warm-up (weights / L2)
        nat.lib().lfd_debug_set_trace(nat.ptr(buf))
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        out, _, q = run_conv(x, w, scale, shift, case[6], case[7], res=res)
        nat.lib().lfd_debug_set_trace(None)
        t = buf.cpu()
        t0 = int(t[t > 0].min())
        rel = (t - t0).clamp(min=-1)
        print('== %s %s plan=%s' % (name, case, q))
        for role, rn, cols in ((0, 'producer', 'wait_empty got_empty issued arrived_full'), (1, 'mma', 'wait_tempty got_tempty first_full committed'),
                               (2, 'epilogue', 'wait_tfull got_tfull tmem_read_done stored'),
                               (3, 'epilogue detail', 'res_ready after_bar1 store_loop_done -')):
            print('  %s  [%s]' % (rn, cols))
            for i in range(12):
                if int(t[role, i].max()) == 0:
                    break
                print('    %2d  %s' % (i, '  '.join('%7d' % int(v) for v in rel[role, i])))


if __name__ == '__main__':
    main()
