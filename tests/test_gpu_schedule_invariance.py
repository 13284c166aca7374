# -*- coding: utf-8 -*-
"""Whole plans under forced schedules: every op of the plan bounded to m persistent CTAs (m = 1: one CTA walks every tile of
a layer; m = 5) gives the same stored bits as the plan as built.  Only the fp64 atomics of the GroupNorm statistics may add in
another order, so tensors downstream of a GroupNorm may show isolated 1-ulp flips."""
import pytest
import torch

import synth
from helpers import conv_outputs, downstream_of_gn, synth_model
from lfd import _native as nat
from lfd._engine import InferencePlan

pytestmark = pytest.mark.gpu

N, H, W = 2, 200, 328


def _run(plan, x):
    with torch.no_grad():
        cls, reg = plan.forward(x, use_graph=False)
    torch.cuda.synchronize()
    return {name: plan.tensor(name).clone() for name, _ in conv_outputs(plan)}, cls.clone(), reg.clone()


def _bound_every_op(plan, m):
    for o in plan._op_array:
        o.max_ctas = m
    old = plan.handle
    plan.handle = plan._create_handle()
    nat.lib().lfd_plan_destroy(old)


def _ulps(a, b):
    """Difference in bf16 spacings at the larger magnitude of the two."""
    a, b = a.float().cpu(), b.float().cpu()
    mag = torch.maximum(a.abs(), b.abs()).clamp(min=2.0 ** -126)
    return (a - b).abs() / torch.ldexp(torch.ones_like(mag), torch.frexp(mag)[1] - 1 - 7)


@pytest.mark.parametrize('name,fuse_stem', [('WIDERFACE_S', None), ('WIDERFACE_S', True), ('WIDERFACE_L', None), ('TT100K_L', None),
                                            ('TL_L', None), ('TEST_FAST', None)])
def test_plan_outputs_do_not_depend_on_the_grid(name, fuse_stem):
    model, _ = synth_model(name)
    model.cuda()
    plan = InferencePlan(model, N, H, W, torch.device('cuda'), fuse_stem=fuse_stem, reuse=False)   # every intermediate stays readable after the forward
    if fuse_stem:
        assert plan._ops[0]['kind'] == nat.OP_STEM4
    has_gn = any(op['kind'] == nat.OP_GN_APPLY or (op['kind'] == nat.OP_HEAD_FINAL and op.get('gn_groups')) for op in plan._ops)
    gn_tainted = downstream_of_gn(plan)
    x = synth.synth_input(N, H, W, seed=3).cuda()
    base, cls0, reg0 = _run(plan, x)
    for m in (1, 5):
        _bound_every_op(plan, m)
        outs, cls, reg = _run(plan, x)
        for tname, t0 in base.items():
            t = outs[tname]
            if tname not in gn_tainted:
                assert torch.equal(t.view(torch.int16), t0.view(torch.int16)), '%s max_ctas=%d: %s differs in %d elements' % (
                    name, m, tname, int((t != t0).sum()))
            else:
                u = _ulps(t, t0)
                assert float(u.max()) <= 1.0 and float((u > 0).float().mean()) <= 1e-3, '%s max_ctas=%d: %s (%d flips, max %g ulp)' % (
                    name, m, tname, int((u > 0).sum()), float(u.max()))
        if not has_gn:
            assert torch.equal(cls, cls0) and torch.equal(reg, reg0), '%s max_ctas=%d: head outputs differ' % (name, m)
        else:
            for a, b in ((cls, cls0), (reg, reg0)):
                d = (a - b).abs()
                assert float(d.max()) <= 2.0 ** -6 * float(b.abs().max()) and float((d > 0).float().mean()) <= 1e-2, (name, m, float(d.max()))
    assert name != 'TL_L' or not has_gn
