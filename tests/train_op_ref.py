# -*- coding: utf-8 -*-
"""float64 references and per-element bounds of the SIMT training ops (csrc/train.cu), shared by the op-level configuration tests
(test_gpu_train_kernel_configs.py) and the op-by-op replay of whole training steps (test_gpu_train_step_per_op.py).

Every function takes the op's operands as float64 tensors (on any device; the replay keeps them on the GPU), the op's lfd_top fields
and the grid its launcher uses (gpu_train_ops mirrors), and returns (ref, S, K) per output: a 16-bit output must be a faithful rounding
of ref widened by K * 2^-24 * S (check_faithful), an fp32 / fp64 one must lie within K * 2^-24 * S of ref (check_within).

Nothing here assumes a property of the data, because activations of a real step have dead channels (variance 0), channels whose mean is
many standard deviations, float rstd values that depend on fma contraction, and pre-activations that round to either side of 0:
- the error the BatchNorm statistics carry into the normalised output is propagated through rstd per channel (bn_apply_ref);
- both float rstd values a compiler may produce are emulated (mean_rstd_f32), and K carries one more float rounding for the choice;
- a GroupNorm ReLU decision whose fp32 pre-activation lies within its rounding bound of 0 may go either way: such elements are counted
  (`amb`) and either branch is accepted, the group and channel sums widened by their terms."""
import math
from fractions import Fraction

import torch

from gpu_ops import ulp16

U = 2.0 ** -24          # one fp32 rounding


def f32(x):
    """float64 tensor -> the nearest float32 values, as float64."""
    return x.float().double()


def fma_f32(a, b, c):
    """fmaf(a, b, c) on float32 operands held in float64: the product is exact in float64, the sum keeps its sign."""
    return f32(a * b + c)


def cdiv(a, b):
    return -(-a // b)


def passes(chunks, blocks):
    """Most passes any thread makes over a grid-stride loop of `chunks` 16-byte items with `blocks` blocks of 256 threads."""
    return cdiv(chunks, blocks * 256)


def shuffle_levels(C):
    return 5 - int(math.log2(C // 8))      # block_reduce_groups: xor offsets cpr .. 16


def _report(what, got, ref, tol, ok):
    if bool(ok.all()):
        return
    bad = ~ok
    i = tuple(torch.nonzero(bad)[0].tolist())
    err = (got - ref).abs()
    raise AssertionError('%s: %d / %d elements off; first at %s: got %r want %r (tol %g); max err / tol %g'
                         % (what, int(bad.sum()), got.numel(), i, float(got[i]), float(ref[i]), float(tol[i]),
                            float((err / tol.clamp(min=1e-300)).max())))


def check_faithful(out, refs, S, K, what, dtype='bf16'):
    """|out - ref| <= ulp16(ref) + K * 2^-24 * S per element, for at least one of `refs` (a tensor or a tuple of admissible references).
    -> max err / tol (the margin)."""
    refs = refs if isinstance(refs, (tuple, list)) else (refs,)
    o = out.to(refs[0].device).double()
    best, tol0 = None, None
    ok = torch.zeros(o.shape, dtype=torch.bool, device=o.device)
    for r in refs:
        tol = ulp16(r, dtype) + K * U * S
        e = (o - r).abs()
        ratio = e / tol.clamp(min=1e-300)
        ratio = torch.where(e == 0, torch.zeros_like(ratio), ratio)
        best = ratio if best is None else torch.minimum(best, ratio)
        ok |= e <= tol
        tol0 = tol if tol0 is None else tol0
    _report(what, o, refs[0], tol0, ok)
    return float(best.max()) if best.numel() else 0.0


def check_within(got, ref, S, K, what):
    """|got - ref| <= K * 2^-24 * S per element (an fp32 / fp64 accumulation).  -> max err / tol."""
    g = got.to(ref.device).double()
    e = (g - ref).abs()
    tol = K * U * S
    _report(what, g, ref, tol, e <= tol)
    r = e / tol.clamp(min=1e-300)
    return float(torch.where(e == 0, torch.zeros_like(r), r).max()) if r.numel() else 0.0


def check_amb(amb, what, frac=1e-4):
    """Recomputed ReLU decisions that may go either way: they need a pre-activation within a few fp32 roundings of 0, so they are rare."""
    n, k = amb.numel(), int(amb.sum())
    assert k <= max(1.0, frac * n), '%s: %d of %d recomputed ReLU decisions are within rounding of 0' % (what, k, n)
    return k


# ------------------------------------------------------------------------------------------------ statistics
def mean_rstd_f32(s1, s2, count, eps):
    """The kernels' mean and rstd from float64 sums (train.cu mean_rstd_from_sums, conv_simt.cu gn_mean_rstd): (float)(s1 / count) and
    (float)(1 / sqrt(max(s2 / count - m * m, 0) + (double)eps)).  The variance line may be compiled with or without an fma, so both
    float rstd values are returned: (mean, rstd, rstd_fma), equal almost everywhere."""
    shape = s1.shape
    s1, s2 = s1.double().reshape(-1), s2.double().reshape(-1)
    m = s1 / count
    q = s2 / count
    var_sep = (q - m * m).clamp(min=0)
    var_fma = torch.tensor([float(Fraction(a) - Fraction(b) ** 2) for a, b in zip(q.tolist(), m.tolist())], dtype=torch.float64,
                           device=s1.device).clamp(min=0)
    epsd = float(torch.tensor(eps, dtype=torch.float32))
    r_sep, r_fma = f32(1.0 / torch.sqrt(var_sep + epsd)), f32(1.0 / torch.sqrt(var_fma + epsd))
    return f32(m).reshape(shape), r_sep.reshape(shape), r_fma.reshape(shape)


def frozen_mean_rstd(rm, rv, eps):
    """Eval-mode BatchNorm: float running mean, (float)(1 / sqrt((double)running_var + (double)eps))."""
    epsd = float(torch.tensor(eps, dtype=torch.float32))
    return f32(rm.double()), f32(1.0 / torch.sqrt(f32(rv.double()) + epsd))


# ------------------------------------------------------------------------------------------------ BatchNorm forward
def bn_stats_ref(z, blocks):
    """BN_STATS: per-channel (sum z, sum z^2) of z [M, C] in fp64 atomics over fp32 block partials.  -> (ref [C, 2], S [C, 2], K)."""
    M, C = z.shape
    K = passes(M * C // 8, blocks) + shuffle_levels(C) + 8 + 1     # per-thread fp32 chain, shuffle levels, 8 warp partials, the cast
    s1, s2, a1 = z.sum(0), (z * z).sum(0), z.abs().sum(0)
    return torch.stack([s1, s2], -1), torch.stack([a1, s2], -1), K


def bn_apply_ref(z, res, gamma, beta, eps, relu, frozen, rm=None, rv=None, K_s=0):
    """BN_APPLY: y = relu?(gamma * (z - mean) * rstd + beta (+ res)) of z [M, C]; batch statistics of z (their sums carry K_s fp32
    roundings) or, frozen, the running ones.  -> (ref, S, K).

    The kernel forms sc = gamma * rstd, shift = fmaf(-mean, sc, beta), y = fmaf(z, sc, shift) (+ res): 6 roundings on the terms of
    S0 = (|z| + |mean|) |sc| + |beta| (+ |res|), plus one for the fma-dependent rstd.  Batch statistics add, per element, the error of
    the mean (K_s roundings of E|z|, times |sc|) and that of rstd: the sums' error moves the variance by at most
    dv = K_s 2^-24 (E[z^2] + 2 |mean| E|z|), so rstd lies in [1 / sqrt(var + dv + eps), 1 / sqrt(max(var - dv, 0) + eps)] -- exact
    interval arithmetic, valid for a dead channel (var = 0) and for |mean| >> std alike.  S carries those terms scaled to K."""
    M = z.shape[0]
    epsd = float(torch.tensor(eps, dtype=torch.float32))
    g, b = gamma.double(), beta.double()
    K = 7
    if frozen:
        mean, rstd = frozen_mean_rstd(rm, rv, eps)
        sc = g * rstd
        extra = torch.zeros_like(z)
    else:
        mean = z.sum(0) / M
        var = ((z - mean) ** 2).sum(0) / M
        rstd = 1.0 / torch.sqrt(var + epsd)
        sc = g * rstd
        e_abs, e_sq = z.abs().sum(0) / M, (z * z).sum(0) / M
        dv = K_s * U * (e_sq + 2 * mean.abs() * e_abs)
        r_lo, r_hi = 1.0 / torch.sqrt(var + dv + epsd), 1.0 / torch.sqrt((var - dv).clamp(min=0) + epsd)
        d_rstd = torch.maximum(r_hi - rstd, rstd - r_lo)
        extra = K_s * U * e_abs * sc.abs() * (1 + 2 * d_rstd / rstd) + (z - mean).abs() * g.abs() * d_rstd
        K = max(K, K_s)
    ref = (z - mean) * sc + b
    S = (z.abs() + mean.abs()) * sc.abs() + b.abs()
    if res is not None:
        ref, S = ref + res, S + res.abs()
    if relu:
        ref = ref.clamp(min=0)
    return ref, S + extra / (K * U), K


def bn_running_ref(z, rm, rv, momentum, K_s):
    """Running statistics after a train-mode BN_APPLY: (1 - m) r + m stat in float, the unbiased batch variance.  The batch mean moves by
    K_s roundings of E|z|, the variance by K_s roundings of E[z^2] + 2 |mean| E|z|.  -> ((ref, S, K) of the mean, (ref, S, K) of the var)."""
    M = z.shape[0]
    mom = float(torch.tensor(momentum, dtype=torch.float32))
    mean = z.sum(0) / M
    var = ((z - mean) ** 2).sum(0) / M
    var_u = var * M / (M - 1)
    a1, s2 = z.abs().sum(0), (z * z).sum(0)
    d_mean = K_s * U * a1 / M
    d_var = K_s * U * (s2 + 2 * mean.abs() * a1) / M * M / (M - 1)
    rm, rv = rm.double(), rv.double()
    want_m, want_v = (1 - mom) * rm + mom * mean, (1 - mom) * rv + mom * var_u
    # 4 float roundings of (1 - m) r + m stat; the statistics' own error enters once, through m
    return ((want_m, (1 - mom) * rm.abs() + mom * mean.abs() + mom * d_mean / U / 4, 4),
            (want_v, (1 - mom) * rv.abs() + mom * var_u + mom * d_var / U / 4, 4))


# ------------------------------------------------------------------------------------------------ norm backward
def bn_bwd_ref(z, dy, y, fsums, gamma, eps, relu, frozen, rm, rv, blocks):
    """NORM_BWD_REDUCE + NORM_BWD_APPLY of a BatchNorm on [M, C] tensors: the kernels' zhat from the stored forward sums (or the
    running statistics), the mask from the stored output y.  -> dict of (ref, S, K): 'bsums' [C, 2] (sum g, sum g zhat), 'dz', 'dgamma',
    'dbeta'; and 'g' = dy * mask (the residual gradient, exact in bf16)."""
    M, C = z.shape
    if frozen:
        mean, rstd = frozen_mean_rstd(rm, rv, eps)
        rstd_b = rstd
    else:
        mean, rstd, rstd_b = mean_rstd_f32(fsums[:, 0], fsums[:, 1], float(M), eps)
    zh = f32(f32(z - mean) * rstd)
    gm = dy * ((y > 0).double() if relu else 1.0)
    S1, S2 = gm.sum(0), (gm * zh).sum(0)
    A1, A2 = gm.abs().sum(0), (gm * zh).abs().sum(0)
    ga = gamma.double()
    fma = int(not torch.equal(rstd, rstd_b))       # the other rstd moves zhat and rstd by one float rounding each
    K_r = passes(M * C // 8, blocks) + shuffle_levels(C) + 8 + 1 + 2 * fma
    if frozen:
        ref, S = ga * rstd * gm, (ga * rstd * gm).abs()
    else:
        ref = ga * rstd * (gm - (S1 / M + zh * S2 / M))
        S = (ga * rstd).abs() * (gm.abs() + (A1 + zh.abs() * A2) / M)
    # sums (K_r), S / M, zh * S2 / M + S1 / M, g - ., gamma * rstd, *; parameter gradients: the sums cast to float and added by one block
    return dict(bsums=(torch.stack([S1, S2], -1), torch.stack([A1, A2], -1), K_r), dz=(ref, S, K_r + 6), dgamma=(S2, A2, K_r + 1),
                dbeta=(S1, A1, K_r + 1), g=gm)


def gn_mask(zh, zh_b, ga, be):
    """The GroupNorm ReLU decision fmaf(zhat, gamma, beta) > 0, recomputed -> (on, amb): `amb` where the other rstd flips it or the
    pre-activation is within two fp32 roundings of its terms of 0 (either branch is then a correct execution)."""
    v, v_b = fma_f32(zh, ga, be), fma_f32(zh_b, ga, be)
    near = (zh * ga + be).abs() <= 2 * U * ((zh * ga).abs() + be.abs())
    return v > 0, ((v > 0) != (v_b > 0)) | near


def gn_bwd_ref(z, dy, fsums, gamma, beta, eps, blocks):
    """NORM_BWD_REDUCE + NORM_BWD_APPLY of GroupNorm(G, 8 G) + ReLU on [N, HW, G, 8] tensors, fsums [N, G, 2]; `blocks` per image.
    -> dict: 'dz' = ((ref, ref_other), S, K), the two references differing only at the ambiguous elements; 'dgamma', 'dbeta' (ref, S, K)
    per channel; 'bsums' = ((ref [C, 2], S, K), (ref [N, G, 2], S, K)); 'amb' the ambiguous-decision mask."""
    N, HW, G, _ = z.shape
    C, Mg = 8 * G, HW * 8
    mean, rstd, rstd_b = mean_rstd_f32(fsums[..., 0], fsums[..., 1], float(Mg), eps)
    mean, rstd, rstd_b = mean.reshape(N, 1, G, 1), rstd.reshape(N, 1, G, 1), rstd_b.reshape(N, 1, G, 1)
    zh, zh_b = f32(f32(z - mean) * rstd), f32(f32(z - mean) * rstd_b)
    ga, be = gamma.double().reshape(G, 8), beta.double().reshape(G, 8)
    on, amb = gn_mask(zh, zh_b, ga, be)
    fma = int(not torch.equal(rstd, rstd_b))
    gm = dy * (on | amb).double()                                         # the ambiguous elements taken as on
    gd = dy * amb.double()                                                # ... whose terms the sums may or may not hold
    T1, T2 = (gm * ga).sum((1, 3), keepdim=True), (gm * ga * zh).sum((1, 3), keepdim=True)
    A1, A2 = (gm * ga).abs().sum((1, 3), keepdim=True), (gm * ga * zh).abs().sum((1, 3), keepdim=True)
    D1, D2 = (gd * ga).abs().sum((1, 3), keepdim=True), (gd * ga * zh).abs().sum((1, 3), keepdim=True)
    K_r = passes(HW * G, blocks) + shuffle_levels(C) + 8 + 2 + 2 * fma     # + the g * gamma product
    K = K_r + 6
    base = T1 / Mg + zh * T2 / Mg
    ref_on, ref_off = rstd * (gm * ga - base), rstd * (gm * ga * (~amb).double() - base)
    S = rstd * ((gm * ga).abs() + (A1 + zh.abs() * A2) / Mg) + rstd * (D1 + zh.abs() * D2) / Mg / (K * U)
    gz = gm * zh
    dgam, dbet = gz.sum((0, 1)).reshape(C), gm.sum((0, 1)).reshape(C)
    Sg = gz.abs().sum((0, 1)).reshape(C) + (gd * zh).abs().sum((0, 1)).reshape(C) / ((K_r + 1) * U)
    Sb = gm.abs().sum((0, 1)).reshape(C) + gd.abs().sum((0, 1)).reshape(C) / ((K_r + 1) * U)
    ST = torch.cat([A1 + D1 / (K_r * U), A2 + D2 / (K_r * U)], -1).reshape(N, G, 2)
    Sc = torch.stack([gm.abs().sum((0, 1)).reshape(C) + gd.abs().sum((0, 1)).reshape(C) / (K_r * U),
                      gz.abs().sum((0, 1)).reshape(C) + (gd * zh).abs().sum((0, 1)).reshape(C) / (K_r * U)], -1)
    return dict(dz=((ref_on, ref_off), S, K), dgamma=(dgam, Sg, K_r + 1), dbeta=(dbet, Sb, K_r + 1), amb=amb,
                bsums=((torch.stack([dbet, dgam], -1), Sc, K_r), (torch.cat([T1, T2], -1).reshape(N, G, 2), ST, K_r)))


# ------------------------------------------------------------------------------------------------ GroupNorm apply and head final
def head_activation(raw, gamma, beta, stats, groups, eps, dtype='bf16'):
    """a = round16(relu(fmaf((x - mean) * rstd, gamma, beta))) as GN_APPLY / HEAD_FINAL / HEAD_FINAL_BWD form it, raw [N, HW, C].
    -> (a, a_other, amb): a_other takes the other branch at the ambiguous decisions and the other float rstd everywhere; an exact kernel
    matches one of the two per element.  groups = 0: the tower has no norm layers, raw is already the activation."""
    from gpu_ops import DTYPES
    rnd = lambda t: t.float().to(DTYPES[dtype][0]).double()
    N, HW, C = raw.shape
    if not groups:
        a = rnd(raw.clamp(min=0))
        return a, a, torch.zeros(a.shape, dtype=torch.bool, device=a.device)
    x = raw.double().reshape(N, HW, groups, C // groups)
    mean, rstd, rstd_b = mean_rstd_f32(stats[..., 0], stats[..., 1], float(HW * C // groups), eps)
    mean, rstd, rstd_b = mean.reshape(N, 1, groups, 1), rstd.reshape(N, 1, groups, 1), rstd_b.reshape(N, 1, groups, 1)
    ga, be = gamma.double().reshape(groups, -1), beta.double().reshape(groups, -1)
    zh, zh_b = f32(f32(x - mean) * rstd), f32(f32(x - mean) * rstd_b)
    _, amb = gn_mask(zh, zh_b, ga, be)
    # (the emulated fmaf keeps the exact sign, so for a given rstd the decision is exact; the other rstd may flip it)
    a, a_b = rnd(fma_f32(zh, ga, be).clamp(min=0)), rnd(fma_f32(zh_b, ga, be).clamp(min=0))
    return a.reshape(N, HW, C), a_b.reshape(N, HW, C), amb.reshape(N, HW, C)


def head_forward_ref(a, a_b, w, scale, shift):
    """HEAD_FINAL: out = scale * (W . a) + shift over a [.., C].  K = 16 fp32 fmas per channel slice + 3 shuffle adds + 1 fma; the
    activations the kernel may hold instead (a_b) differ from a at few elements by a few bf16 ulps of values near 0, which S covers."""
    wd = w.double()
    ref = (a @ wd.t()) * scale.double() + shift.double()
    S = ((a.abs() + (a - a_b).abs() / (20 * U)) @ wd.abs().t()) * scale.double().abs() + shift.double().abs()
    return ref, S, 20


def head_backward_ref(a, a_b, up, w, scale, bias, n_cls, bx, tiles, N):
    """HEAD_FINAL_BWD on a [N, HW, C], up [N, HW, n_out] (the loss gradients at the level's points), bx blocks per image over `tiles`
    tiles.  -> dict of (ref, S, K): 'dact' (bf16), 'dW' [n_out, C], 'dbias', 'dscale' [1] (when there are regression rows)."""
    no, C = w.shape
    nr = no - n_cls
    T = cdiv(tiles, bx)
    h = up * scale.double()
    wd = w.double()
    da = (a - a_b).abs()
    small = no <= 5
    ppt = 2 if small else 4                  # pixels per thread per tile
    n_atom = bx * N                          # fp32 atomics onto the staging, one per block
    if small:       # registers over all tiles, 2 shuffles, 8 warp partials through shared memory
        K_w, K_b = 1 + (ppt + 1) * T + 2 + 8 + n_atom, 1 + ppt + T + 2 + 8 + n_atom
        K_sc = 16 + 3 + 2 + 2 * ppt * T * 2 + 2 + 8 + n_atom
    else:           # per tile: 4-pixel sums, 2 shuffles, one shared-memory atomic per warp (8 per tile)
        K_w = K_b = 1 + ppt + 2 + 8 * T + n_atom
        K_sc = 16 + 3 + 2 + nr * ppt * T + 32 + n_atom       # 32 slice-0 threads add into one shared float
    hf, af, daf = h.reshape(-1, no), a.reshape(-1, C), da.reshape(-1, C)
    out = dict(dact=(h @ wd, h.abs() @ wd.abs(), no + 1),
               dW=(hf.t() @ af, hf.abs().t() @ (af.abs() + daf / (K_w * U)), K_w),
               dbias=(hf.sum(0), hf.abs().sum(0), K_b))
    if nr:
        u = af @ wd[n_cls:].t() + bias.double()[n_cls:]                     # [pix][n_reg]: W . a + b
        ur = up.reshape(-1, no)[:, n_cls:]
        Su = (af.abs() + daf / (K_sc * U)) @ wd[n_cls:].abs().t() + bias.double()[n_cls:].abs()
        out['dscale'] = ((ur * u).sum().reshape(1), (ur.abs() * Su).sum().reshape(1), K_sc)
    return out


# ------------------------------------------------------------------------------------------------ packing
def conv_pack_ref(w, cc, dgrad):
    """Index formula of the packed operand [Kin/cc][k*k][cc/8][Nout][8]: forward Kin = Cin, Nout = Cout, W[n][kch][tap]; data
    gradient Kin = Cout, Nout = Cin, W[kch][n][k*k - 1 - tap]."""
    Cout, Cin, k, _ = w.shape
    kk = k * k
    nout = Cin if dgrad else Cout
    idx = torch.arange(w.numel(), device=w.device)
    j, r = idx % 8, idx // 8
    n, r = r % nout, r // nout
    kc, r = r % (cc // 8), r // (cc // 8)
    tap, c = r % kk, r // kk
    kch = c * cc + kc * 8 + j
    wf = w.reshape(-1)
    v = wf[(kch * Cin + n) * kk + (kk - 1 - tap)] if dgrad else wf[(n * Cin + kch) * kk + tap]
    return v.to(torch.bfloat16)
