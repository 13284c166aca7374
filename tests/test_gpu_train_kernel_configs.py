# -*- coding: utf-8 -*-
"""The SIMT kernels of the training step (csrc/train.cu) and the optimizer, element-wise against float64 on the kernels' own 16-bit
operands, across their configuration space and under forced small grids (lfd_top.max_ctas 1 and 3) that make every thread walk its
batched grid-stride loops many times and every head-final-backward block run its cp.async ring through several refills.

Bounds are per element: a 16-bit output must be a faithful rounding of the float64 value widened by K * 2^-24 * S (train_op_ref
check_faithful), an fp32 / fp64 result must lie within K * 2^-24 * S (check_within).  The references and bounds live in train_op_ref.py,
shared with the op-by-op replay of whole training steps (test_gpu_train_step_per_op.py).  S is the sum of the magnitudes
of the terms, K the number of fp32 roundings a term can pass through, written next to each assert from the kernel's accumulation:
passes per thread, warp-shuffle levels, the 8 warp partials of a block, and fp32 atomics."""
import functools
import math

import pytest
import torch

from gpu_ops import DTYPES, conv_out, stem_input
from gpu_train_ops import (Workspace, bf16r, cdiv, desc_table, elementwise_blocks, gn_bwd_blocks, grid_sms, head_bwd_grid, make_top,
                           reduce_blocks, run_top, stem_wgrad_grid, assert_within)
from train_op_ref import (bn_apply_ref, bn_bwd_ref, bn_running_ref, bn_stats_ref, check_amb, check_faithful, check_within, conv_pack_ref,
                          gn_bwd_ref, head_activation, head_backward_ref, head_forward_ref)
from lfd import _native as nat

DEV = 'cuda'
GRIDS = [0, 1, 3]           # max_ctas: the default grid, and forced grids of 1 and 3 "SMs"
FORCED = [1, 3]
H100_SMS = 132              # the table test's stand-in for the SM count (the forced grids are below it on any H100)
EPS = 1e-5
MOM = float(torch.tensor(0.1, dtype=torch.float32))      # BatchNorm momentum as the kernel sees it (float)


def _sms(max_ctas):
    return grid_sms(max_ctas, nat.lib().lfd_device_sm_count())


# ================================================================================================ BatchNorm: sizes and grids
# N x H x W per channel count: about 43 k 16-byte chunks, odd H and W, N in {1, 3}
BN_SIZES = {8: (3, 119, 121), 16: (1, 147, 149), 32: (3, 59, 61), 64: (1, 73, 75), 128: (3, 29, 31), 256: (1, 37, 37)}


def _bn_grids(C, max_ctas, sms=H100_SMS):
    """-> chunks, [(kernel, blocks, loop depth)] of BN_STATS, BN_APPLY, NORM_BWD_REDUCE and NORM_BWD_APPLY (BatchNorm)."""
    N, H, W = BN_SIZES[C]
    chunks = N * H * W * (C // 8)
    s = grid_sms(max_ctas, sms)
    return chunks, [('bn_stats', reduce_blocks(chunks, s), 4), ('bn_apply', elementwise_blocks(chunks, s), 4),
                    ('norm_bwd_reduce', reduce_blocks(chunks, s), 2), ('norm_bwd_apply', elementwise_blocks(chunks, s), 2)]


# (C, relu, res, frozen, cancel): cancel = every other channel has |mean| = 16 std, where E[x^2] - E[x]^2 cancels
BN_CASES = [
    (8, 1, 0, 0, 0), (16, 0, 1, 0, 0), (32, 1, 1, 0, 0), (64, 1, 1, 0, 0), (128, 1, 1, 0, 0), (256, 0, 0, 0, 0),   # 64 / 128 res + relu: shipped
    (64, 1, 0, 0, 1), (256, 1, 1, 0, 1),
    (32, 0, 0, 1, 0), (128, 1, 0, 1, 0), (16, 1, 1, 1, 0),    # frozen; (128, relu, frozen): TL_L's conv + bias towers
]


def _bn_id(c):
    return 'C%d_relu%d_res%d_frozen%d%s' % (c[:4] + ('_cancel' if c[4] else '',))


# (C, relu, res, accumulate, up, frozen): up = 0, 'odd' (upH / upW = 2H - 1) or 'even' (2H)
NB_CASES = [
    (8, 1, 0, 0, 0, 0), (16, 0, 1, 0, 'odd', 0), (32, 1, 1, 1, 'even', 0), (64, 1, 1, 0, 0, 0), (128, 1, 1, 1, 0, 0), (256, 0, 0, 0, 'even', 0),
    (64, 0, 1, 1, 'odd', 0), (64, 1, 0, 0, 'even', 1), (128, 1, 0, 0, 0, 1), (32, 0, 1, 1, 0, 1), (256, 1, 1, 0, 'odd', 0),
]


def _nb_id(c):
    return 'C%d_relu%d_res%d_acc%d_up%s_frozen%d' % c


# (groups, N, H, W): C = 8 groups
GN_CASES = [(1, 1, 139, 143), (2, 3, 59, 61), (4, 2, 49, 51), (8, 1, 49, 53), (16, 3, 21, 23), (32, 2, 17, 19), (16, 1, 35, 37)]

# head final: (groups, n_cls, n_reg, N, H, W); the first 14 are deep enough for >= 4 tiles per block under the forced grids, the last
# three have HW < 64 (a single, partial tile)
HEAD_OUTS = [(1, 4), (0, 4), (1, 0), (5, 0), (2, 4), (45, 0), (60, 4)]


def _head_size(n_out, N):
    if n_out <= 5:
        return (53, 59) if N == 1 else (31, 33)       # 3127 / 1023 pixels: 49 / 16 tiles of 64
    return (77, 79) if N == 1 else (43, 47)           # 6083 / 2021 pixels: 48 / 16 tiles of 128


HEAD_CASES = [(g, nc, nr, N) + _head_size(nc + nr, N) for i, (nc, nr) in enumerate(HEAD_OUTS) for g, N in ((0, 1 + 2 * (i % 2)), (16, 3 - 2 * (i % 2)))] + \
             [(16, 1, 4, 2, 5, 9), (0, 60, 4, 1, 7, 7), (16, 45, 0, 3, 3, 11)]


def _head_id(c):
    return 'g%d_cls%d_reg%d_N%d_%dx%d' % c


# stem weight gradient: (Cout, path, fmt)
STEM_CASES = [(c, path, fmt) for c in (16, 32, 64) for path in ('simt', 'umma') for fmt in ('u8', 'f32')]
STEM_SIZE = (1, 99, 259)        # 50 x 130 outputs: 150 row segments of <= 64 pixels


def test_case_tables_cover_the_launchable_space():
    # BatchNorm: every power-of-two chunks-per-row count the launchers accept, each option on and off, the shipped combinations
    chans = {8 * 2 ** i for i in range(6)}
    assert {c[0] for c in BN_CASES} == chans and {c[0] for c in NB_CASES} == chans
    for i in range(1, 4):
        assert {c[i] for c in BN_CASES} == {0, 1}
    assert (64, 1, 1, 0, 0) in BN_CASES and (128, 1, 1, 0, 0) in BN_CASES and (128, 1, 0, 1, 0) in BN_CASES
    assert any(c[4] for c in BN_CASES)
    assert {c[1] for c in NB_CASES} == {0, 1} and {c[5] for c in NB_CASES} == {0, 1}
    assert {(c[2], c[3]) for c in NB_CASES} >= {(0, 0), (1, 0), (1, 1)} and {c[4] for c in NB_CASES} == {0, 'odd', 'even'}
    assert any(c[1] == 0 and c[4] for c in NB_CASES)                    # BN without ReLU feeding a stride-2 data gradient
    assert {g for g, _, _, _ in GN_CASES} == {1, 2, 4, 8, 16, 32} and {n for _, n, _, _ in GN_CASES} == {1, 2, 3}
    # head final: both kernels on both sides of n_out = 5, n_out = 64, both Scale-gradient paths, with and without GroupNorm
    assert {(c[0], c[1], c[2]) for c in HEAD_CASES if c[4] * c[5] >= 64} == {(g, nc, nr) for g in (0, 16) for nc, nr in HEAD_OUTS}
    assert max(nc + nr for _, nc, nr, _, _, _ in HEAD_CASES) == 64
    assert any(c[4] * c[5] < 64 for c in HEAD_CASES) and {c[3] for c in HEAD_CASES} >= {1, 3}
    for c in BN_SIZES.values():
        assert c[0] in (1, 3) and c[1] % 2 and c[2] % 2
    # forced grids: >= 6 passes per thread, and a remainder modulo both the stride and the batched stride
    for C in BN_SIZES:
        for m in FORCED:
            chunks, grids = _bn_grids(C, m)
            for name, blocks, depth in grids:
                stride = blocks * 256
                assert chunks // stride >= 6, (C, m, name, blocks)
                assert chunks % stride and chunks % (depth * stride), (C, m, name, blocks)
    for G, N, H, W in GN_CASES:
        for m in FORCED:
            chunks = H * W * G
            stride = gn_bwd_blocks(chunks, N, m) * 256
            assert chunks // stride >= 6 and chunks % stride and chunks % (2 * stride), (G, N, m)
    for g, nc, nr, N, H, W in HEAD_CASES:
        assert (H * W) % 64 and (H * W) % 128
        if H * W >= 64:
            for m in FORCED:
                bx, tiles = head_bwd_grid(H * W, nc + nr, N, m)
                assert tiles // bx >= 4, (g, nc, nr, N, m)
    N, H, W = STEM_SIZE
    for m in FORCED:
        blocks, n_seg = stem_wgrad_grid(N, conv_out(H, 3, 2), conv_out(W, 3, 2), m)
        assert n_seg // blocks >= 4
    for n in SQNORM_SIZES[:-1]:
        assert n % 4 or n < 4
    n = SQNORM_SIZES[-1]
    assert n % 4 == 3 and cdiv(n // 4, 4 * H100_SMS * 256) >= 3
    # packing: every (Cin, Cout, k, cc) the shipped configs' convs and data-gradient convs are packed with
    fwd, dgrad = _shipped_pack_configs()
    assert fwd <= set(PACK_FWD) and dgrad <= set(PACK_DGRAD), (fwd - set(PACK_FWD), dgrad - set(PACK_DGRAD))


# ================================================================================================ BatchNorm statistics and apply
@functools.lru_cache(maxsize=None)
def _bn_operands(case):
    C, relu, res, frozen, cancel = case
    N, H, W = BN_SIZES[C]
    g = torch.Generator().manual_seed(C * 100 + relu * 8 + res * 4 + frozen * 2 + cancel)
    sd = torch.rand((C,), generator=g) + 1.0                 # std in [1, 2), |mean| <= 0.5
    mu = torch.rand((C,), generator=g) - 0.5
    if cancel:
        mu[1::2] = 16.0 * sd[1::2] * torch.sign(torch.randn((C // 2,), generator=g))
    z = bf16r(torch.randn((N, H, W, C), generator=g) * sd + mu)
    r = bf16r(torch.randn((N, H, W, C), generator=g)) if res else None
    if frozen and C == 128:      # TL_L: conv + bias as a frozen BatchNorm with gamma 1, mean 0, var 1 - eps, beta = bias
        gamma, beta = torch.ones(C), torch.randn((C,), generator=g) * 0.3
        rm, rv = torch.zeros(C), torch.full((C,), 1.0 - EPS)
    else:
        gamma, beta = torch.rand((C,), generator=g) + 0.5, torch.randn((C,), generator=g) * 0.3
        rm, rv = mu + 0.1 * torch.randn((C,), generator=g), sd ** 2 * (torch.rand((C,), generator=g) + 0.5)
    return z, r, gamma, beta, rm, rv


def _run_bn(case, max_ctas):
    C, relu, res, frozen, cancel = case
    z, r, gamma, beta, rm, rv = _bn_operands(case)
    N, H, W = BN_SIZES[C]
    ws = Workspace(DEV)
    ws.add('z', z.to(torch.bfloat16))
    ws.add('y', torch.full((N, H, W, C), float('nan')).to(torch.bfloat16))
    if res:
        ws.add('res', r.to(torch.bfloat16))
    ws.add('sums', shape=(C, 2), dtype=torch.float64)
    ws.finalize()
    g_d, b_d, rm_d, rv_d = gamma.to(DEV), beta.to(DEV), rm.to(DEV), rv.to(DEV)
    geo = dict(N=N, H=H, W=W, Cout=C, eps=EPS, frozen=frozen, max_ctas=max_ctas)
    if not frozen:
        run_top(make_top(nat.TOP_BN_STATS, off={0: ws.off('z'), 3: ws.off('sums')}, **geo), ws)
    run_top(make_top(nat.TOP_BN_APPLY, relu=relu, momentum=0.1, off={0: ws.off('z'), 1: ws.off('y'), 2: ws.off('res') if res else -1,
                                                                      3: -1 if frozen else ws.off('sums')},
                     ptr={0: g_d.data_ptr(), 1: b_d.data_ptr(), 2: rm_d.data_ptr(), 3: rv_d.data_ptr()}, **geo), ws)
    return ws.get('sums').cpu(), ws.get('y').cpu(), rm_d.cpu(), rv_d.cpu()


@pytest.mark.gpu
@pytest.mark.parametrize('max_ctas', GRIDS)
@pytest.mark.parametrize('case', BN_CASES, ids=_bn_id)
def test_bn_stats_and_apply_match_fp64(case, max_ctas):
    C, relu, res, frozen, cancel = case
    z, r, gamma, beta, rm, rv = _bn_operands(case)
    N, H, W = BN_SIZES[C]
    M = N * H * W
    chunks, grids = _bn_grids(C, max_ctas, nat.lib().lfd_device_sm_count())
    if max_ctas:
        assert all(chunks // (b * 256) >= 6 for _, b, _ in grids)
    sums, y, rm_got, rv_got = _run_bn(case, max_ctas)
    what = 'BN %s max_ctas=%d' % (_bn_id(case), max_ctas)
    zd = z.double().reshape(M, C)
    sums_ref, sums_S, K_s = bn_stats_ref(zd, grids[0][1])
    if not frozen:
        check_within(sums, sums_ref, sums_S, K_s, what + ' sums')
    ref, S, K_y = bn_apply_ref(zd, r.double().reshape(M, C) if res else None, gamma, beta, EPS, relu, frozen, rm, rv, K_s)
    yg = y.reshape(M, C)
    if cancel:      # the channels with |mean| = 16 std: report the margin of the bound there
        odd = torch.arange(C) % 2 == 1
        m = check_faithful(yg[:, odd], ref[:, odd], S[:, odd], K_y, what + ' y (|mean| = 16 std)')
        print('%s: |mean| = 16 std channels: max err / tol %.3g' % (what, m))
    check_faithful(yg, ref, S, K_y, what + ' y')
    if frozen:      # eval-mode BatchNorm: the running statistics are read, never written
        assert torch.equal(rm_got, rm) and torch.equal(rv_got, rv), what
        return
    (want_m, S_m, K_m), (want_v, S_v, K_v) = bn_running_ref(zd, rm, rv, 0.1, K_s)
    check_within(rm_got, want_m, S_m, K_m, what + ' running_mean')
    check_within(rv_got, want_v, S_v, K_v, what + ' running_var')


# ================================================================================================ norm backward, BatchNorm
@functools.lru_cache(maxsize=None)
def _nb_operands(case):
    C, relu, res, acc, up, frozen = case
    N, H, W = BN_SIZES[C]
    g = torch.Generator().manual_seed(7000 + C * 10 + relu * 8 + res * 4 + acc * 2 + frozen)
    sd, mu = torch.rand((C,), generator=g) + 1.0, torch.rand((C,), generator=g) - 0.5
    z = bf16r(torch.randn((N, H, W, C), generator=g) * sd + mu)
    # an upstream gradient correlated with z and offset, so that both batch-statistics terms of dz are large
    dy = bf16r(0.5 * torch.randn((N, H, W, C), generator=g) + 0.7 * (z - mu) / sd + 0.3)
    y = bf16r(torch.randn((N, H, W, C), generator=g).clamp(min=0))          # the stored forward output: only its sign is read
    prev = bf16r(torch.randn((N, H, W, C), generator=g))
    gamma, beta = torch.rand((C,), generator=g) + 0.5, torch.randn((C,), generator=g) * 0.3
    rm, rv = mu + 0.1 * torch.randn((C,), generator=g), sd ** 2 * (torch.rand((C,), generator=g) + 0.5)
    if frozen and C == 128:
        gamma, rm, rv = torch.ones(C), torch.zeros(C), torch.full((C,), 1.0 - EPS)
    return z, dy, y, prev, gamma, beta, rm, rv


def _up_size(H, W, up):
    return (2 * H - 1, 2 * W - 1) if up == 'odd' else (2 * H, 2 * W)


def _run_norm_bwd(ws, geo, offs, ptr):
    run_top(make_top(nat.TOP_NORM_BWD_REDUCE, off={k: v for k, v in offs.items() if k < 5}, ptr=ptr, **geo), ws)
    run_top(make_top(nat.TOP_NORM_BWD_APPLY, off=offs, ptr=ptr, **geo), ws)


@pytest.mark.gpu
@pytest.mark.parametrize('max_ctas', GRIDS)
@pytest.mark.parametrize('case', NB_CASES, ids=_nb_id)
def test_bn_backward_matches_fp64(case, max_ctas):
    C, relu, res, acc, up, frozen = case
    z, dy, y, prev, gamma, beta, rm, rv = _nb_operands(case)
    N, H, W = BN_SIZES[C]
    M = N * H * W
    chunks, grids = _bn_grids(C, max_ctas, nat.lib().lfd_device_sm_count())
    if max_ctas:
        assert all(chunks // (b * 256) >= 6 for _, b, _ in grids)
    zd = z.double()
    fs = torch.stack([zd.reshape(M, C).sum(0), (zd * zd).reshape(M, C).sum(0)], -1)
    ws = Workspace(DEV)
    ws.add('z', z.to(torch.bfloat16))
    ws.add('dy', dy.to(torch.bfloat16))
    ws.add('y', y.to(torch.bfloat16))
    ws.add('fsums', fs)
    ws.add('bsums', shape=(C, 2), dtype=torch.float64)
    ws.add('dz', torch.full((N, H, W, C), float('nan')).to(torch.bfloat16))
    if res:
        ws.add('dres', prev.to(torch.bfloat16) if acc else torch.full((N, H, W, C), float('nan')).to(torch.bfloat16))
    if up:
        uh, uw = _up_size(H, W, up)
        ws.add('dzu', torch.full((N, uh, uw, C), float('nan')).to(torch.bfloat16))     # the launcher clears it
    ws.finalize()
    g_d, b_d, rm_d, rv_d = gamma.to(DEV), beta.to(DEV), rm.to(DEV), rv.to(DEV)
    dg_d, db_d = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV)
    geo = dict(N=N, H=H, W=W, Cout=C, groups=0, relu=relu, eps=EPS, frozen=frozen, accumulate=acc, max_ctas=max_ctas)
    if up:
        geo.update(upH=uh, upW=uw)
    offs = {0: ws.off('dy'), 1: ws.off('y') if relu else -1, 2: ws.off('z'), 3: -1 if frozen else ws.off('fsums'), 4: ws.off('bsums'),
            5: ws.off('dz'), 6: ws.off('dzu') if up else -1, 7: ws.off('dres') if res else -1}
    _run_norm_bwd(ws, geo, offs, {0: g_d.data_ptr(), 1: b_d.data_ptr(), 2: dg_d.data_ptr(), 3: db_d.data_ptr(), 4: rm_d.data_ptr(), 5: rv_d.data_ptr()})
    what = 'BN backward %s max_ctas=%d' % (_nb_id(case), max_ctas)
    r = bn_bwd_ref(zd.reshape(M, C), dy.double().reshape(M, C), y.double().reshape(M, C), fs, gamma, EPS, relu, frozen, rm, rv, grids[2][1])
    gm = r['g']
    dz = ws.get('dz').cpu()
    check_faithful(dz.reshape(M, C), *r['dz'], what=what + ' dz')
    check_within(ws.get('bsums').cpu(), *r['bsums'], what=what + ' sums')
    check_within(dg_d, *r['dgamma'], what=what + ' dgamma')
    check_within(db_d, *r['dbeta'], what=what + ' dbeta')
    if res:
        got = ws.get('dres').cpu().reshape(M, C)
        if acc:
            want = gm + prev.double().reshape(M, C)
            check_faithful(got, want, gm.abs() + prev.double().abs().reshape(M, C), 1, what + ' dres')    # prev + g, one fp32 add
        else:
            assert torch.equal(got.double(), gm), what + ' dres'
    if up:
        dzu = ws.get('dzu').cpu()
        assert torch.equal(dzu[:, ::2, ::2, :].contiguous().view(torch.int16), dz.view(torch.int16)), what + ' dz_up'
        mask = torch.ones(dzu.shape[:3], dtype=torch.bool)
        mask[:, ::2, ::2] = False
        assert bool((dzu[mask].view(torch.int16) == 0).all()), what + ' dz_up zeros'


# ================================================================================================ norm backward, GroupNorm
@functools.lru_cache(maxsize=None)
def _gn_operands(case):
    G, N, H, W = case
    C = 8 * G
    g = torch.Generator().manual_seed(9000 + G * 10 + N)
    mu = torch.randn((N, 1, 1, G, 1), generator=g) * 0.5
    sd = torch.rand((N, 1, 1, G, 1), generator=g) + 0.75
    z = bf16r((torch.randn((N, H, W, G, 8), generator=g) * sd + mu).reshape(N, H, W, C))
    dy = bf16r(0.5 * torch.randn((N, H, W, C), generator=g) + 0.7 * ((z.reshape(N, H, W, G, 8) - mu) / sd).reshape(N, H, W, C) + 0.3)
    gamma, beta = torch.rand((C,), generator=g) + 0.5, torch.randn((C,), generator=g) * 0.3
    return z, dy, gamma, beta


@pytest.mark.gpu
@pytest.mark.parametrize('max_ctas', GRIDS)
@pytest.mark.parametrize('case', GN_CASES, ids=lambda c: 'g%d_N%d_%dx%d' % c)
def test_gn_backward_matches_fp64(case, max_ctas):
    G, N, H, W = case
    C, HW = 8 * G, H * W
    z, dy, gamma, beta = _gn_operands(case)
    blocks = gn_bwd_blocks(HW * G, N, _sms(max_ctas))
    if max_ctas:
        assert HW * G // (blocks * 256) >= 6
    zd = z.double().reshape(N, HW, G, 8)
    fs = torch.stack([zd.sum((1, 3)), (zd * zd).sum((1, 3))], -1)           # [N][G][2]
    ws = Workspace(DEV)
    ws.add('z', z.to(torch.bfloat16))
    ws.add('dy', dy.to(torch.bfloat16))
    ws.add('fsums', fs)
    ws.add('bsums', shape=(C * 2 + N * G * 2,), dtype=torch.float64)
    ws.add('dz', torch.full((N, H, W, C), float('nan')).to(torch.bfloat16))
    ws.finalize()
    g_d, b_d = gamma.to(DEV), beta.to(DEV)
    dg_d, db_d = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV)
    geo = dict(N=N, H=H, W=W, Cout=C, groups=G, relu=1, eps=EPS, max_ctas=max_ctas)
    offs = {0: ws.off('dy'), 2: ws.off('z'), 3: ws.off('fsums'), 4: ws.off('bsums'), 5: ws.off('dz')}
    _run_norm_bwd(ws, geo, offs, {0: g_d.data_ptr(), 1: b_d.data_ptr(), 2: dg_d.data_ptr(), 3: db_d.data_ptr()})
    what = 'GN backward %s max_ctas=%d' % ('g%d_N%d_%dx%d' % case, max_ctas)
    r = gn_bwd_ref(zd, dy.double().reshape(N, HW, G, 8), fs, gamma, beta, EPS, blocks)
    check_amb(r['amb'], what)
    check_faithful(ws.get('dz').cpu().reshape(N, HW, G, 8), *r['dz'], what=what + ' dz')
    bs = ws.get('bsums').cpu()
    check_within(bs[:C * 2].view(C, 2), *r['bsums'][0], what=what + ' channel sums')
    check_within(bs[C * 2:].view(N, G, 2), *r['bsums'][1], what=what + ' group sums')
    check_within(dg_d, *r['dgamma'], what=what + ' dgamma')
    check_within(db_d, *r['dbeta'], what=what + ' dbeta')


# ================================================================================================ head final, forward and backward
@functools.lru_cache(maxsize=None)
def _head_operands(case, dtype='bf16'):
    groups, nc, nr, N, H, W = case
    C, HW, no = 128, H * W, nc + nr
    rnd = DTYPES[dtype][1]
    g = torch.Generator().manual_seed(3000 + groups * 100 + nc * 5 + nr + N)
    if groups:
        raw = rnd(torch.randn((N, HW, C), generator=g) * 1.5 + 0.3)
    else:
        raw = rnd(torch.randn((N, HW, C), generator=g).clamp(min=0))      # no norm layers: the input is the activated tensor
    gamma, beta = torch.rand((C,), generator=g) + 0.5, torch.randn((C,), generator=g) * 0.3
    w = rnd(torch.randn((no, C), generator=g) * 0.1)
    bias = torch.randn((no,), generator=g) * 0.5
    scale = torch.cat([torch.ones(nc), torch.full((nr,), 1.3)])
    shift = (bias * scale).float()                                       # PACK_SCALE_SHIFT: bias * scale in fp32
    point_off, cls_stride = 20, nc + 3
    P = point_off + HW + 37
    gcls = torch.randn((N, P, cls_stride), generator=g)
    greg = torch.randn((N, P, 4), generator=g)
    xs = raw.double().reshape(N, HW, 16, 8)
    stats = torch.stack([xs.sum((1, 3)), (xs * xs).sum((1, 3))], -1)
    return raw, gamma, beta, w, bias, scale, shift, gcls, greg, stats, point_off, cls_stride, P


def _head_activation(raw, gamma, beta, stats, groups, dtype='bf16'):
    """-> (a, a_other, amb) of train_op_ref.head_activation on the case's GroupNorm(16, 128)."""
    return head_activation(raw, gamma, beta, stats, 16 if groups else 0, EPS, dtype)


def _check_head_outputs(cls_o, reg_o, ref, S, K, nc, point_off, HW, what):
    sl = slice(point_off, point_off + HW)
    if nc:
        check_within(cls_o[:, sl, :nc], ref[..., :nc], S[..., :nc], K, what + ' cls')
        assert bool(torch.isnan(cls_o[:, sl, nc:]).all()), what + ': cls channels past n_cls written'
        assert bool(torch.isnan(cls_o[:, :point_off]).all() and torch.isnan(cls_o[:, point_off + HW:]).all()), what + ': cls rows outside the level written'
    if ref.shape[-1] > nc:
        check_within(reg_o[:, sl], ref[..., nc:], S[..., nc:], K, what + ' reg')
        assert bool(torch.isnan(reg_o[:, :point_off]).all() and torch.isnan(reg_o[:, point_off + HW:]).all()), what + ': reg rows outside the level written'


@pytest.mark.gpu
@pytest.mark.parametrize('max_ctas', GRIDS)
@pytest.mark.parametrize('case', HEAD_CASES, ids=_head_id)
def test_head_final_forward_and_backward_match_fp64(case, max_ctas):
    groups, nc, nr, N, H, W = case
    C, HW, no = 128, H * W, nc + nr
    raw, gamma, beta, w, bias, scale, shift, gcls, greg, stats, point_off, cls_stride, P = _head_operands(case)
    bx, tiles = head_bwd_grid(HW, no, N, _sms(max_ctas))
    T = cdiv(tiles, bx)                      # most tiles a block walks
    if max_ctas and HW >= 64:
        assert tiles // bx >= 4
    ws = Workspace(DEV)
    ws.add('raw', raw.to(torch.bfloat16))
    ws.add('stats', stats)
    ws.add('stage', torch.cat([w.reshape(-1), scale, shift, bias]))
    ws.add('dstage', shape=(no * C + no,), dtype=torch.float32)
    ws.add('dscale', shape=(1,), dtype=torch.float32)
    ws.add('dact', torch.full((N, HW, C), float('nan')).to(torch.bfloat16))
    ws.finalize()
    g_d, b_d = gamma.to(DEV), beta.to(DEV)
    cls_o, reg_o = torch.full((N, P, cls_stride), float('nan'), device=DEV), torch.full((N, P, 4), float('nan'), device=DEV)
    gcls_d, greg_d = gcls.to(DEV), greg.to(DEV)
    geo = dict(N=N, H=H, W=W, Cout=C, groups=groups, n_cls=nc, n_reg=nr, P=P, point_off=point_off, cls_stride=cls_stride, eps=EPS, max_ctas=max_ctas)
    nptr = {0: g_d.data_ptr(), 1: b_d.data_ptr()} if groups else {}
    run_top(make_top(nat.TOP_HEAD_FINAL, off={0: ws.off('raw'), 3: ws.off('stats') if groups else -1, 4: ws.off('stage')},
                     ptr={**nptr, 2: cls_o.data_ptr(), 3: reg_o.data_ptr()}, **geo), ws)
    run_top(make_top(nat.TOP_HEAD_FINAL_BWD, off={0: ws.off('raw'), 1: ws.off('dact'), 3: ws.off('stats') if groups else -1, 4: ws.off('stage'),
                                                 5: ws.off('dstage'), 6: ws.off('dscale')},
                     ptr={**nptr, 2: gcls_d.data_ptr(), 3: greg_d.data_ptr()}, **geo), ws)
    what = 'head final %s max_ctas=%d' % (_head_id(case), max_ctas)
    a, a_b, amb = _head_activation(raw, gamma, beta, stats, groups)
    check_amb(amb, what)
    ref, S, K = head_forward_ref(a, a_b, w, scale, shift)
    _check_head_outputs(cls_o.cpu(), reg_o.cpu(), ref, S, K, nc, point_off, HW, what)
    # backward: h_o = g_o * scale_o (one rounding); dact = sum_o h_o W_o; dW = sum_pix h a; db = sum_pix h; dScale = sum g (W . a + b)
    up = torch.cat([gcls[:, point_off:point_off + HW, :nc], greg[:, point_off:point_off + HW, :nr]], -1).double()     # [N][HW][no]
    r = head_backward_ref(a, a_b, up, w, scale, bias, nc, bx, tiles, N)
    check_faithful(ws.get('dact').cpu(), *r['dact'], what=what + ' dact')
    ds = ws.get('dstage').cpu()
    check_within(ds[:no * C].view(no, C), *r['dW'], what=what + ' dW')
    check_within(ds[no * C:], *r['dbias'], what=what + ' dbias')
    if nr:
        check_within(ws.get('dscale').cpu(), *r['dscale'], what=what + ' dScale')
    else:
        assert float(ws.get('dscale').cpu()[0]) == 0.0


# inference ops that already honour max_ctas: GN apply and head final at both storage types on a single-SM grid
@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ['bf16', 'fp16'])
def test_inference_gn_apply_matches_fp64(dtype):
    tdt, rnd, _, code = DTYPES[dtype]
    N, H, W, G = 3, 31, 33, 16
    C, HW = 8 * G, H * W
    g = torch.Generator().manual_seed(41)
    x = rnd(torch.randn((N, HW, C), generator=g) * 1.5 + 0.3)
    gamma, beta = torch.rand((C,), generator=g) + 0.5, torch.randn((C,), generator=g) * 0.3
    xs = x.double().reshape(N, HW, G, 8)
    stats = torch.stack([xs.sum((1, 3)), (xs * xs).sum((1, 3))], -1)
    bx = min(cdiv(HW * G, 256), cdiv(8, N))           # gn_apply_launch with one SM
    assert HW * G // (bx * 256) >= 6
    ws = Workspace(DEV)
    ws.add('stats', stats)
    ws.add('in', x.to(tdt))
    ws.add('out', torch.full((N, HW, C), float('nan')).to(tdt))
    ws.finalize()
    g_d, b_d = gamma.to(DEV), beta.to(DEV)
    op = nat.Op()
    op.kind, op.dtype, op.N, op.H, op.W, op.Cin, op.Cout, op.gn_groups = nat.OP_GN_APPLY, code, N, H, W, C, C, G
    op.in_off, op.out_off, op.stats_off, op.res_off, op.ds_out_off = ws.off('in'), ws.off('out'), ws.off('stats'), -1, -1
    op.gamma, op.beta, op.max_ctas = g_d.data_ptr(), b_d.data_ptr(), 1
    _run_op(op, ws)
    a, a_b, amb = _head_activation(x, gamma, beta, stats, 16, dtype)
    got = ws.get('out').cpu().double()
    bad = (got != a) & (got != a_b)
    assert not bool(bad.any()), '%s GN apply: %d elements differ from the exact emulation' % (dtype, int(bad.sum()))


def _run_op(op, ws, cls=None, reg=None, P=0, cls_channels=0):
    import ctypes as C_
    with torch.cuda.device(ws.device):
        nat.check(nat.lib().lfd_run_op(C_.byref(op), None, 0, nat.ptr(ws.buf), nat.ptr(cls), nat.ptr(reg), P, cls_channels, nat.CONV_UMMA,
                                       nat.stream_ptr()))
        torch.cuda.synchronize()


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', ['bf16', 'fp16'])
@pytest.mark.parametrize('case', [c for c in HEAD_CASES if c[3] == 3 and c[1] + c[2] in (5, 6, 45, 64)], ids=_head_id)
def test_inference_head_final_matches_fp64(case, dtype):
    groups, nc, nr, N, H, W = case
    tdt, rnd, _, code = DTYPES[dtype]
    C, HW, no = 128, H * W, nc + nr
    raw, gamma, beta, w, bias, scale, shift, gcls, greg, stats, point_off, cls_stride, P = _head_operands(case, dtype)
    tiles, bx = cdiv(HW, 128), min(cdiv(4, N), cdiv(HW, 128))           # head_final_launch with one SM
    assert tiles // bx >= 4 or HW < 64
    ws = Workspace(DEV)
    ws.add('stats', stats)
    ws.add('in', raw.to(tdt))
    ws.finalize()
    w_d, sc_d, sh_d, g_d, b_d = w.to(DEV), scale.to(DEV), shift.to(DEV), gamma.to(DEV), beta.to(DEV)
    cls_o, reg_o = torch.full((N, P, cls_stride), float('nan'), device=DEV), torch.full((N, P, 4), float('nan'), device=DEV)
    op = nat.Op()
    op.kind, op.dtype, op.N, op.H, op.W, op.Cin, op.Cout, op.gn_groups = nat.OP_HEAD_FINAL, code, N, H, W, C, no, groups
    op.n_cls, op.n_reg, op.point_off = nc, nr, point_off
    op.in_off, op.out_off, op.stats_off, op.res_off, op.ds_out_off = ws.off('in'), -1, ws.off('stats') if groups else -1, -1, -1
    op.weight, op.scale, op.shift, op.max_ctas = w_d.data_ptr(), sc_d.data_ptr(), sh_d.data_ptr(), 1
    if groups:
        op.gamma, op.beta = g_d.data_ptr(), b_d.data_ptr()
    _run_op(op, ws, cls_o, reg_o, P, cls_stride)
    a, a_b, _ = _head_activation(raw, gamma, beta, stats, groups, dtype)
    ref, S, K = head_forward_ref(a, a_b, w, scale, shift)
    _check_head_outputs(cls_o.cpu(), reg_o.cpu(), ref, S, K, nc, point_off, HW, 'inference head final %s %s' % (_head_id(case), dtype))


# ================================================================================================ parameter packing
# (Cin, Cout, k, cc) of the forward and data-gradient packs of the shipped configs (a superset is fine: see the table test)
PACK_FWD = [(16, 32, 3, 16), (32, 32, 1, 32), (32, 32, 3, 32), (32, 64, 1, 32), (32, 64, 3, 32), (64, 32, 3, 32), (64, 32, 3, 64),
            (64, 64, 1, 64), (64, 64, 3, 32), (64, 64, 3, 64), (64, 128, 1, 64), (64, 128, 3, 16), (128, 128, 1, 64), (128, 128, 3, 16)]
PACK_DGRAD = [(32, 32, 1, 32), (32, 32, 3, 32), (32, 64, 1, 64), (32, 64, 3, 64), (64, 32, 3, 32), (64, 64, 1, 64), (64, 64, 3, 64),
              (64, 128, 1, 64), (64, 128, 3, 32), (128, 128, 1, 64), (128, 128, 3, 16)]


def _shipped_pack_configs():
    """Every (Cin, Cout, k, cc) conv_query gives the convs of the shipped configs that are packed with PACK_CONV_FWD (all but the
    stem and the final head convs), and their data-gradient convs (PACK_CONV_DGRAD; ones the wgmma kernel cannot run are skipped,
    as the training planner refuses them)."""
    from oracle import lfd_oracle as orc
    from helpers import build_model
    fwd, dgrad = set(), set()
    for name in orc.CONFIGS:
        model = build_model(name)
        head = model._head
        final = {id(c) for l in range(head._num_heads) for c in head.level_paths(l)[2:4]}
        for m in model.modules():
            if not isinstance(m, torch.nn.Conv2d) or m.in_channels == 3 or id(m) in final:
                continue
            k, s, ci, co = m.kernel_size[0], m.stride[0], m.in_channels, m.out_channels
            ho = conv_out(64, k, s)
            fwd.add((ci, co, k, nat.conv_query(2, 64, 64, ci, ho, ho, co, k, s)['cc']))
            try:
                dgrad.add((ci, co, k, nat.conv_query(2, 64, 64, co, 64, 64, ci, k, 1)['cc']))
            except nat.LfdError:
                pass
    return fwd, dgrad


@pytest.mark.gpu
def test_pack_table_matches_index_formulas():
    """One PACK table with every kind and entries of very different n: each entry writes exactly its n elements."""
    from lfd._engine import pack_conv_weight, pack_stem_weight
    g = torch.Generator().manual_seed(51)
    descs, checks, keep = [], [], []

    def dst(n, dtype):
        t = torch.full((n + 300,), float('nan'), device=DEV).to(dtype)       # 300 sentinels past the end
        keep.append(t)
        return t

    for dgrad, table in ((0, PACK_FWD), (1, PACK_DGRAD)):
        for ci, co, k, cc in table:
            w = torch.randn((co, ci, k, k), generator=g)
            wd, o = w.to(DEV), dst(w.numel(), torch.bfloat16)
            keep.append(wd)
            descs.append(nat.PackDesc(kind=nat.PACK_CONV_DGRAD if dgrad else nat.PACK_CONV_FWD, Cout=co, Cin=ci, k=k, cc=cc, n=w.numel(),
                                      src=wd.data_ptr(), dst=o.data_ptr()))
            want = conv_pack_ref(w, cc, dgrad)
            if not dgrad:
                assert torch.equal(want, pack_conv_weight(w, cc).reshape(-1))
            checks.append(('%s %s' % ('dgrad' if dgrad else 'fwd', (ci, co, k, cc)), o, want))
    for co in (32, 64):
        w = torch.randn((co, 3, 3, 3), generator=g)
        wd, o = w.to(DEV), dst(3 * 2 * co * 8, torch.bfloat16)
        keep.append(wd)
        descs.append(nat.PackDesc(kind=nat.PACK_STEM, Cout=co, Cin=3, k=3, n=3 * 2 * co * 8, src=wd.data_ptr(), dst=o.data_ptr()))
        checks.append(('stem %d' % co, o, pack_stem_weight(w).reshape(-1)))
    hw = torch.randn((1001,), generator=g)
    hwd, o = hw.to(DEV), dst(1001, torch.float32)
    keep.append(hwd)
    descs.append(nat.PackDesc(kind=nat.PACK_ROUND_F32, n=1001, src=hwd.data_ptr(), dst=o.data_ptr()))
    checks.append(('round', o, bf16r(hw)))
    bias, sc = torch.randn((5,), generator=g), torch.tensor([1.7])
    bd, scd = bias.to(DEV), sc.to(DEV)
    keep += [bd, scd]
    for name, src, src2, b_eff, s_eff in (('no scale', bd, None, bias, torch.ones(5)), ('no bias', None, scd, torch.zeros(5), sc.expand(5))):
        o1, o2, o3 = dst(5, torch.float32), dst(5, torch.float32), dst(5, torch.float32)
        descs.append(nat.PackDesc(kind=nat.PACK_SCALE_SHIFT, n=5, src=0 if src is None else src.data_ptr(), src2=0 if src2 is None else src2.data_ptr(),
                                  dst=o1.data_ptr(), dst2=o2.data_ptr(), dst3=o3.data_ptr()))
        checks += [('scale ' + name, o1, s_eff.float()), ('shift ' + name, o2, (b_eff * s_eff).float()), ('bias ' + name, o3, b_eff.float())]
    max_n = max(d.n for d in descs)
    table = desc_table(descs, DEV)
    ws = Workspace(DEV).finalize()
    run_top(make_top(nat.TOP_PACK, n_desc=len(descs), max_n=max_n, ptr={0: table.data_ptr()}), ws)
    for what, o, want in checks:
        got = o.cpu()
        n = want.numel()
        assert torch.equal(got[:n].float(), want.float()), what
        assert bool(torch.isnan(got[n:].float()).all()), what + ': written past n'


@pytest.mark.gpu
def test_unpack_table_matches_index_formulas():
    g = torch.Generator().manual_seed(52)
    descs, checks, keep = [], [], []
    for ci, co, k in ((32, 64, 3), (64, 32, 1), (128, 64, 3), (48, 16, 1)):
        kk = k * k
        stage = torch.randn((kk, ci, co), generator=g)              # [tap][ci][co]
        grad = torch.randn((co, ci, k, k), generator=g)
        sd, gd = stage.to(DEV), grad.to(DEV)
        keep.append(sd)
        descs.append(nat.UnpackDesc(kind=nat.UNPACK_CONV, Cout=co, Cin=ci, kk=kk, n=grad.numel(), src=sd.data_ptr(), dst=gd.data_ptr()))
        idx = torch.arange(grad.numel())
        tap, r = idx % kk, idx // kk
        cin, cout = r % ci, r // ci
        checks.append(('conv %s' % ((ci, co, k),), gd, grad.reshape(-1) + stage.reshape(-1)[(tap * ci + cin) * co + cout]))
    a, b = torch.randn((777,), generator=g), torch.randn((777 + 100,), generator=g)
    ad, bd = a.to(DEV), b.to(DEV)
    keep.append(ad)
    descs.append(nat.UnpackDesc(kind=nat.UNPACK_ADD, n=777, src=ad.data_ptr(), dst=bd.data_ptr()))
    checks.append(('add', bd, torch.cat([b[:777] + a, b[777:]])))
    table = desc_table(descs, DEV)
    ws = Workspace(DEV).finalize()
    run_top(make_top(nat.TOP_UNPACK, n_desc=len(descs), max_n=max(d.n for d in descs), ptr={0: table.data_ptr()}), ws)
    for what, got, want in checks:
        assert torch.equal(got.cpu().reshape(-1), want.reshape(-1)), what


# ================================================================================================ stem weight gradient
@pytest.mark.gpu
@pytest.mark.parametrize('max_ctas', GRIDS)
@pytest.mark.parametrize('cout,path,fmt', STEM_CASES)
def test_stem_wgrad_matches_fp64(cout, path, fmt, max_ctas):
    N, H, W = STEM_SIZE
    Ho, Wo = conv_out(H, 3, 2), conv_out(W, 3, 2)
    blocks, n_seg = stem_wgrad_grid(N, Ho, Wo, _sms(max_ctas))
    if max_ctas:
        assert n_seg // blocks >= 4
    g = torch.Generator().manual_seed(cout + (path == 'simt') * 7 + (fmt == 'u8') * 3)
    img = torch.randint(0, 256, (N, H, W, 3), generator=g, dtype=torch.uint8) if fmt == 'u8' else torch.randn((N, 3, H, W), generator=g)
    x = stem_input(img, fmt)                                              # normalised and rounded as the kernels do (R0)
    dz = bf16r(torch.randn((N, Ho, Wo, cout), generator=g))
    ws = Workspace(DEV)
    ws.add('dz', dz.to(torch.bfloat16))
    ws.add('ds', shape=(32, cout), dtype=torch.float32)
    ws.add('x27', shape=(N, Ho, Wo, 32), dtype=torch.bfloat16)
    ws.finalize()
    offs = {1: ws.off('dz'), 5: ws.off('ds')}
    if path == 'umma':
        offs[0] = ws.off('x27')
    run_top(make_top(nat.TOP_WGRAD_STEM, N=N, H=H, W=W, Cin=3, Ho=Ho, Wo=Wo, Cout=cout, ksize=3, stride=2, max_ctas=max_ctas,
                     impl=nat.WGRAD_SIMT if path == 'simt' else nat.WGRAD_UMMA, off=offs), ws,
            input=img.to(DEV).contiguous(), fmt=nat.INPUT_U8_NHWC if fmt == 'u8' else nat.INPUT_F32_NCHW)
    stage = ws.get('ds').cpu()
    assert float(stage[27:].abs().max()) == 0.0
    got = stage[:27].reshape(9, 3, cout).permute(2, 1, 0).reshape(cout, 3, 3, 3)
    xd, dzd = x.double().permute(0, 3, 1, 2), dz.double().permute(0, 3, 1, 2)
    ref = torch.nn.grad.conv2d_weight(xd, (cout, 3, 3, 3), dzd, stride=2, padding=1)
    S = torch.nn.grad.conv2d_weight(xd.abs(), (cout, 3, 3, 3), dzd.abs(), stride=2, padding=1)
    # SIMT: one fp32 chain per (tap, ci, co) and block over its segments' pixels, then one atomic per block; the wgmma path's fp32
    # accumulators see at most every pixel of the batch, plus one atomic per CTA
    K = cdiv(n_seg, blocks) * 64 + blocks if path == 'simt' else N * Ho * Wo + 4 * _sms(max_ctas)
    assert_within(got, ref, S, K, 'stem wgrad %d %s %s max_ctas=%d' % (cout, path, fmt, max_ctas))


# ================================================================================================ gradient norm and SGD
SQNORM_SIZES = [1, 3, 5, 4 * 1001 + 3, 3 * 4 * 4 * H100_SMS * 256 + 7]     # the last: several passes of the default grid, n % 4 = 3


@pytest.mark.gpu
@pytest.mark.parametrize('n', SQNORM_SIZES)
def test_grad_sqnorm_matches_fp64(n):
    g = torch.randn((n,), generator=torch.Generator().manual_seed(n))
    gd = g.to(DEV)
    sq = torch.full((1,), float('nan'), dtype=torch.float64, device=DEV)
    nat.check(nat.lib().lfd_grad_sqnorm(nat.ptr(gd), n, nat.ptr(sq), nat.stream_ptr()))
    torch.cuda.synchronize()
    sms = nat.lib().lfd_device_sm_count()
    blocks = max(1, min(cdiv(n // 4, 256), 4 * sms))
    # 4 fmas per float4 pass (+1 for the n % 4 tail), 5 shuffle levels; the 8 warp sums and the atomics are fp64
    K = 4 * cdiv(n // 4, blocks * 256) + 1 + 5
    want = (g.double() ** 2).sum()
    assert_within(sq.cpu(), want.reshape(1), want.reshape(1), K, 'sqnorm n=%d' % n)


# (momentum, dampening, nesterov, weight decay, max_norm, grad_scale): max_norm 0 = no clipping, 1e9 = clipping inactive
SGD_CASES = [(0.0, 0.0, 0, 1e-4, 0.0, 1.0), (0.9, 0.0, 1, 5e-4, 1e9, 1.0), (0.9, 0.1, 0, 1e-4, 5.0, 1.0), (0.8, 0.0, 0, 0.0, 1e9, 0.5),
             (0.9, 0.0, 1, 1e-4, 5.0, 0.25)]


@pytest.mark.gpu
@pytest.mark.parametrize('case', SGD_CASES, ids=lambda c: 'm%g_d%g_nest%d_wd%g_clip%g_gs%g' % c)
def test_sgd_step_matches_fp64(case):
    mom, damp, nest, wd, max_norm, gs = case
    n, lr = 100003, 0.05
    gen = torch.Generator().manual_seed(61)
    p0, g0, m0 = torch.randn((n,), generator=gen), torch.randn((n,), generator=gen) * 0.1, torch.randn((n,), generator=gen) * 0.1
    pd, gd, md = p0.to(DEV), g0.to(DEV), m0.to(DEV)
    sq = torch.zeros(1, dtype=torch.float64, device=DEV)
    if max_norm > 0:
        nat.check(nat.lib().lfd_grad_sqnorm(nat.ptr(gd), n, nat.ptr(sq), nat.stream_ptr()))
    nat.check(nat.lib().lfd_sgd_step(nat.ptr(pd), nat.ptr(gd), nat.ptr(md), n, lr, mom, damp, wd, nest, max_norm, gs, nat.ptr(sq), nat.stream_ptr()))
    torch.cuda.synchronize()
    what = 'sgd %s' % (case,)
    # include/lfd_b200.h: g *= grad_scale * min(1, max_norm / (|grad_scale| * ||g|| + 1e-6)); d = g + wd p; b = mom m + (1 - damp) d;
    # d = nesterov ? d + mom b : b; p -= lr d
    p, g, m = p0.double(), g0.double(), m0.double()
    f = lambda v: float(torch.tensor(v, dtype=torch.float32))             # the float arguments as the kernel receives them
    lr_, mom_, damp_, wd_, gs_ = f(lr), f(mom), f(damp), f(wd), f(gs)
    coef = gs_
    if max_norm > 0:
        total = math.sqrt(float((g * g).sum())) * abs(gs_)
        coef *= min(1.0, f(max_norm) / (total + f(1e-6)))
        if max_norm < 1e9:
            assert coef < gs_ * 0.9, 'the clipping case must clip'
    gs2 = g * coef
    d = gs2 + wd_ * p
    Sd = gs2.abs() + abs(wd_) * p.abs()
    if mom:
        b = mom_ * m + (1 - damp_) * d
        Sb = mom_ * m.abs() + abs(1 - damp_) * Sd
        d, Sd = (d + mom_ * b, Sd + mom_ * Sb) if nest else (b, Sb)
        assert_within(md.cpu(), b, Sb, 10, what + ' momentum')        # coef (~5 roundings), g * coef, fma wd, (1 - damp) *, fma
    else:
        assert torch.equal(md.cpu(), m0), what + ': momentum buffer written without momentum'
    assert_within(gd.cpu(), gs2, gs2.abs(), 6, what + ' clipped gradient')
    assert_within(pd.cpu(), p - lr_ * d, p.abs() + lr_ * Sd, 12, what + ' parameters')


def _split_groups(params):
    a = [p for i, p in enumerate(params) if i % 3]
    b = [p for i, p in enumerate(params) if not i % 3]
    return a, b


GROUP_A = dict(lr=0.02, momentum=0.9, weight_decay=1e-4, nesterov=True, dampening=0.0)
GROUP_B = dict(lr=0.05, momentum=0.8, weight_decay=5e-4, dampening=0.1)


@pytest.mark.gpu
def test_fused_sgd_matches_torch_sgd_with_two_groups():
    """FusedSGD over the flat buffers against torch.optim.SGD: two parameter groups with different hyper-parameters, Nesterov in
    one and dampening in the other (torch starts a momentum buffer as the undamped gradient); then the state_dict round trip."""
    from helpers import synth_model
    from lfd.execution.optim import FusedSGD
    model, _ = synth_model('WIDERFACE_XS')
    model.cuda().train()
    params = list(model.parameters())
    ref = [p.detach().cpu().clone().requires_grad_(True) for p in params]
    ra, rb = _split_groups(ref)
    topt = torch.optim.SGD([dict(params=ra, **GROUP_A), dict(params=rb, **GROUP_B)], lr=0.1)
    pa, pb = _split_groups(params)
    opt = FusedSGD.from_torch(torch.optim.SGD([dict(params=pa, **GROUP_A), dict(params=pb, **GROUP_B)], lr=0.1), model)
    gen = torch.Generator().manual_seed(71)

    def step():
        grads = [torch.randn(p.shape, generator=gen) for p in params]
        opt.zero_grad()
        for p, r, gr in zip(params, ref, grads):
            p.grad.copy_(gr)
            r.grad = gr.clone()
        opt.step()
        topt.step()
        torch.cuda.synchronize()

    def compare(what, tref):
        for i, (p, r) in enumerate(zip(params, ref)):
            group = 'B' if i % 3 == 0 else 'A'
            assert torch.allclose(p.detach().cpu(), r.detach(), rtol=1e-5, atol=1e-6), '%s: parameter %d (group %s) differs by %g' % (
                what, i, group, float((p.detach().cpu() - r.detach()).abs().max()))
        sd = opt.state_dict()
        index = {id(r): i for i, r in enumerate(ra + rb)}
        assert len(sd['state']) == len(tref.state)
        for r, st in tref.state.items():
            got = sd['state'][index[id(r)]]['momentum_buffer'].cpu()
            assert torch.allclose(got, st['momentum_buffer'], rtol=1e-5, atol=1e-6), what + ': momentum buffer'

    for s in range(3):
        step()
        compare('step %d' % s, topt)
    # the checkpoint loads into torch.optim.SGD; one more step on each agrees
    sd = opt.state_dict()
    ref2 = [r.detach().clone().requires_grad_(True) for r in ref]
    r2a, r2b = _split_groups(ref2)
    topt2 = torch.optim.SGD([dict(params=r2a, **GROUP_A), dict(params=r2b, **GROUP_B)], lr=0.1)
    topt2.load_state_dict(sd)
    ref, ra, rb, topt = ref2, r2a, r2b, topt2
    step()
    compare('step after the state_dict round trip', topt)
    # like torch.optim.SGD, an optimizer that never stepped has no momentum buffers to save
    fresh = FusedSGD.from_torch(torch.optim.SGD([dict(params=pa, **GROUP_A), dict(params=pb, **GROUP_B)], lr=0.1), model)
    assert fresh.state_dict()['state'] == {}, 'momentum buffers saved before the first step'
