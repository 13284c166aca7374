# -*- coding: utf-8 -*-
"""Both plan kinds run on one executor (api.cu BranchExecutor): when an op on a side branch is rejected by its launcher (a host-side
status, before any kernel of it is enqueued), the call returns that status and every started branch is still joined into the caller's
stream: work enqueued on the caller's stream after the failed call sees everything the branch did before the failing op, and the
caller's stream keeps working.  The side-branch ops are GroupNorm applies bounded to one SM's worth of CTAs, so they run for a while
after the call returns and a missing join would let the caller's next op read their output before it is written.  With use_graph the
failing pass is the eager first pass of a graph request: it captures nothing, so the next call fails the same way."""
import ctypes as C

import pytest
import torch

import lfd._native as nat

pytestmark = pytest.mark.gpu

ERR_INVALID = 1
N, H, W, CH, GROUPS = 1, 512, 512, 128, 16
STATS_BYTES, ACT_BYTES = N * GROUPS * 2 * 8, N * H * W * CH * 2
IN_OFF, OUT_OFF = 256, 256 + ACT_BYTES


def _workspace():
    """Zero statistics and input, output filled with NaN bit patterns; GroupNorm apply writes relu(beta) = 0.5 everywhere."""
    ws = torch.zeros(OUT_OFF + ACT_BYTES, dtype=torch.uint8, device='cuda')
    ws[OUT_OFF:].fill_(0xFF)
    return ws, torch.ones(CH, device='cuda'), torch.full((CH,), 0.5, device='cuda')


def _check_joined(run, ws):
    rc = run()
    out = ws[OUT_OFF:].view(torch.bfloat16).clone()       # on the caller's stream, right after the failed call
    torch.cuda.current_stream().synchronize()
    assert rc == ERR_INVALID
    assert torch.equal(out, torch.full_like(out, 0.5))
    assert run() == ERR_INVALID                            # no graph was cached by the failed graph request


@pytest.mark.parametrize('use_graph', [0, 1])
def test_inference_plan_joins_branches_on_launch_error(use_graph):
    lib = nat.lib()
    ws, gamma, beta = _workspace()
    cls = torch.zeros((N, H * W, 1), device='cuda')
    reg = torch.zeros((N, H * W, 4), device='cuda')
    ops = (nat.Op * 3)()
    for o in ops:
        o.N, o.H, o.W, o.Cin, o.Ho, o.Wo, o.Cout, o.dtype, o.branch = N, H, W, CH, H, W, CH, nat.DTYPE_BF16, 1
        o.in_off, o.out_off, o.res_off, o.stats_off, o.ds_out_off = IN_OFF, -1, -1, -1, -1
    for g in ops[:2]:          # valid: GroupNorm apply (zero statistics) of a zero tensor, on 8 CTAs
        g.kind, g.gn_groups, g.out_off, g.stats_off, g.max_ctas = nat.OP_GN_APPLY, GROUPS, OUT_OFF, 0, 1
        g.gamma, g.beta = gamma.data_ptr(), beta.data_ptr()
    f = ops[2]                 # rejected by the launcher: a regression head has 4 outputs
    f.kind, f.Cout, f.n_cls, f.n_reg = nat.OP_HEAD_FINAL, 4, 1, 3
    h = C.c_void_p()
    nat.check(lib.lfd_plan_create(ops, 3, N, H * W, 1, 0, STATS_BYTES, ws.numel(), nat.CONV_UMMA, C.byref(h)))
    x = torch.zeros((N, 8, 8, 3), dtype=torch.uint8, device='cuda')
    try:
        _check_joined(lambda: lib.lfd_plan_forward(h, nat.ptr(x), nat.INPUT_U8_NHWC, nat.ptr(ws), nat.ptr(cls), nat.ptr(reg), use_graph,
                                                   nat.stream_ptr()), ws)
        assert b'n_reg' in lib.lfd_last_error()
    finally:
        lib.lfd_plan_destroy(h)


@pytest.mark.parametrize('use_graph', [0, 1])
def test_training_plan_joins_branches_on_launch_error(use_graph):
    lib = nat.lib()
    ws, gamma, beta = _workspace()
    ops = (nat.Top * 3)()
    for t in ops:
        t.N, t.H, t.W, t.Cout, t.groups, t.branch, t.eps, t.max_ctas = N, H, W, CH, GROUPS, 1, 1e-5, 1
        for j in range(8):
            t.off[j] = -1
        t.off[0], t.off[1], t.off[3] = IN_OFF, OUT_OFF, 0
    for g in ops[:2]:          # valid: GroupNorm apply, as above
        g.kind, g.ptr[0], g.ptr[1] = nat.TOP_GN_APPLY, gamma.data_ptr(), beta.data_ptr()
    ops[2].kind = nat.TOP_BN_APPLY     # rejected by the launcher: BatchNorm apply without gamma / beta
    h = C.c_void_p()
    nat.check(lib.lfd_train_plan_create(ops, 3, ws.numel(), C.byref(h)))
    try:
        _check_joined(lambda: lib.lfd_train_plan_run(h, None, nat.INPUT_U8_NHWC, nat.ptr(ws), use_graph, nat.stream_ptr()), ws)
        assert b'bn_apply' in lib.lfd_last_error()
    finally:
        lib.lfd_train_plan_destroy(h)
