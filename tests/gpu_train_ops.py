# -*- coding: utf-8 -*-
"""Helpers that drive single native TRAINING ops through the C-ABI (lfd_run_top) for the GPU parity tests."""
import ctypes as C

import torch

from gpu_ops import Workspace  # noqa: F401  (the training tests' workspace)
from lfd import _native as nat


def make_top(kind, **kw):
    t = nat.Top()
    t.kind = kind
    for i in range(8):
        t.off[i] = -1
    for k, v in kw.items():
        if k == 'off':
            for i, o in v.items():
                t.off[i] = o
        elif k == 'ptr':
            for i, p in v.items():
                t.ptr[i] = p
        else:
            setattr(t, k, v)
    return t


def run_top(t, ws, input=None, fmt=0):
    with torch.cuda.device(ws.device):
        nat.check(nat.lib().lfd_run_top(C.byref(t), nat.ptr(input), fmt, nat.ptr(ws.buf), nat.stream_ptr()))
        torch.cuda.synchronize()


def desc_table(descs, device):
    """ctypes structs -> device byte tensor (the PACK / UNPACK tables live in device memory)."""
    arr = (type(descs[0]) * len(descs))(*descs)
    raw = bytes(memoryview(arr).cast('B'))
    return torch.frombuffer(bytearray(raw), dtype=torch.uint8).to(device)


# ------------------------------------------------------------------------------------------------ grids of the SIMT training launches
# Mirrors of the block counts in csrc/train.cu.  `sms` is what launch_top passes them: the device's SM count, or lfd_top.max_ctas
# when that is smaller (api.cu bounded_sms).
def grid_sms(max_ctas, sm_count):
    return max_ctas if 0 < max_ctas < sm_count else sm_count


def cdiv(a, b):
    return -(-a // b)


def elementwise_blocks(chunks, sms):          # bn_apply, norm_bwd_apply (BN)
    return max(1, min(cdiv(chunks, 1024), 8 * sms))


def reduce_blocks(chunks, sms):               # bn_stats, norm_bwd_reduce (BN)
    return max(1, min(cdiv(chunks, 2048), 4 * sms))


def gn_bwd_blocks(hw_chunks, N, sms):         # norm_bwd_{reduce,apply} (GN): blocks per image
    return min(elementwise_blocks(hw_chunks, sms), cdiv(4 * sms, N))


def head_bwd_grid(HW, n_out, N, sms):         # head_final_bwd: (blocks per image, tiles per image)
    tiles = cdiv(HW, 64 if n_out <= 5 else 128)
    return max(1, min(cdiv(4 * sms, N), tiles)), tiles


def stem_wgrad_grid(N, Ho, Wo, sms):          # wgrad_stem (SIMT): (blocks, 64-pixel row segments)
    n_seg = N * Ho * cdiv(Wo, 64)
    return min(4 * sms, n_seg), n_seg


def assert_within(got, ref, S, K, what=''):
    """Per element |got - ref| <= K * 2^-24 * S: an fp32 (or fp64) result of an accumulation of terms whose magnitudes sum to S,
    each term passing through at most K fp32 roundings."""
    g = got.detach().cpu().double()
    err = (g - ref).abs()
    tol = K * 2.0 ** -24 * S
    bad = ~(err <= tol)
    if bool(bad.any()):
        i = tuple(torch.nonzero(bad)[0].tolist())
        raise AssertionError('%s: %d / %d elements off; first at %s: got %r want %r (tol %g); max err / tol %g'
                             % (what, int(bad.sum()), g.numel(), i, float(g[i]), float(ref[i]), float(tol[i]),
                                float((err / tol.clamp(min=1e-300)).max())))
