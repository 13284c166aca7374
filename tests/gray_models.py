# -*- coding: utf-8 -*-
"""Gray (1-channel) models and their 3-channel twins, for the tests of the gray input path.

The rule those tests check: a gray model with stem weights W1 gives, bit for bit, the outputs of the 3-channel model whose stem weights are
[W1, 0, 0] (channel 0 = the first byte of a BGR pixel, no channel swap) on any frame whose channel 0 is the gray frame."""
import copy

import torch
import torch.nn as nn

import tl_s
from helpers import synth_model


def gray_pair(name, cls_bias=-1.0, seed=666):
    """-> (gray model, 3-channel twin), both in eval mode on the host.  The twin is the synthetic model of config `name` (tl_s for TL_S)
    with channels 1 and 2 of its stem conv's weight zeroed; the gray model is a copy of it whose stem conv is a 1-channel conv holding the
    twin's channel 0.  Every other parameter and buffer is the same."""
    twin = tl_s.synth_model(cls_bias, seed)[0] if name == 'TL_S' else synth_model(name, cls_bias, seed)[0]
    bb = twin._backbone
    conv = bb._stem[0]
    with torch.no_grad():
        conv.weight[:, 1:] = 0
    gray = copy.deepcopy(twin)
    g = nn.Conv2d(1, conv.out_channels, kernel_size=3, stride=2, padding=1, bias=conv.bias is not None)
    with torch.no_grad():
        g.weight.copy_(conv.weight[:, :1])
        if conv.bias is not None:
            g.bias.copy_(conv.bias)
    gray._backbone._stem[0] = g
    gray._backbone._input_channels = 1
    return gray.eval(), twin.eval()


def twin_u8(gray_u8, seed=0):
    """uint8 gray frames [N, H, W] -> BGR frames [N, H, W, 3] whose byte 0 is the gray frame and whose bytes 1 and 2 are random."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(0, 256, tuple(gray_u8.shape) + (3,), generator=g, dtype=torch.uint8).to(gray_u8.device)
    x[..., 0] = gray_u8
    return x.contiguous()


def twin_f32(gray_f32):
    """float32 gray frames [N, 1, H, W] -> [N, 3, H, W] with planes 1 and 2 = 0."""
    n, _, h, w = gray_f32.shape
    x = torch.zeros((n, 3, h, w), dtype=torch.float32, device=gray_f32.device)
    x[:, :1] = gray_f32
    return x
