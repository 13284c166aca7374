# -*- coding: utf-8 -*-
"""A model file run through the C ABI alone (lfd_engine_*), with torch tensors as the caller's device buffers: what a C program does,
for the tests and the timing script to compare with InferencePlan / PostPlan."""
import ctypes as C

import torch

from lfd import _native as nat
from lfd._engine import stage_nv12


class Engine(object):
    def __init__(self, data, device='cuda', poison=None):
        lib = nat.lib()
        self.handle = C.c_void_p()
        nat.check(lib.lfd_engine_open(data, len(data), C.byref(self.handle)))
        self.desc = d = nat.EngineDesc()
        nat.check(lib.lfd_engine_info(self.handle, C.byref(d)))
        self.N, self.H, self.W = d.N, d.H, d.W

        def buf(n):
            t = torch.empty(max(int(n), 1), dtype=torch.uint8, device=device)
            if poison is not None:
                t.fill_(poison)
            return t
        self.weights, self.workspace, self.post_ws = buf(d.weights_bytes), buf(d.workspace_bytes), buf(d.post_workspace_bytes)
        self.dets = torch.empty((d.N, d.cap, 5), dtype=torch.float32, device=device)
        self.labels = torch.empty((d.N, d.cap), dtype=torch.int32, device=device)
        self.count = torch.empty((d.N + 1,), dtype=torch.int32, device=device)
        self.cls = torch.empty((d.N, d.P, d.cls_channels), dtype=torch.float32, device=device)
        self.reg = torch.empty((d.N, d.P, 4), dtype=torch.float32, device=device)
        self.stage = {}

    def bind(self, workspace_bytes=None):
        """-> lfd_engine_bind's return code."""
        ws = self.desc.workspace_bytes if workspace_bytes is None else workspace_bytes
        with torch.cuda.device(self.weights.device):
            return nat.lib().lfd_engine_bind(self.handle, nat.ptr(self.weights), self.desc.weights_bytes, nat.ptr(self.workspace), ws,
                                             nat.ptr(self.post_ws), self.desc.post_workspace_bytes, nat.stream_ptr())

    def num_launches(self):
        return nat.lib().lfd_engine_num_launches(self.handle)

    def op(self, i):
        o, src, level = nat.Op(), C.c_int32(), C.c_int32()
        nat.check(nat.lib().lfd_engine_op(self.handle, i, C.byref(o), C.byref(src), C.byref(level)))
        return o, src.value, level.value

    def capacity_input(self, x, fmt, h, w):
        """x: the frames (float32 [N,3,h,w], uint8 [N,h,w,3] or NV12 [N,3h/2,w]) -> the same frames in the capacity layout."""
        if (h, w) == (self.H, self.W):
            return x
        if fmt not in self.stage:
            shape = {nat.INPUT_F32_NCHW: (self.N, 3, self.H, self.W), nat.INPUT_U8_NHWC: (self.N, self.H, self.W, 3),
                     nat.INPUT_U8_NV12: (self.N, self.H * 3 // 2, self.W)}[fmt]
            self.stage[fmt] = torch.zeros(shape, dtype=torch.float32 if fmt == nat.INPUT_F32_NCHW else torch.uint8, device=x.device)
        s = self.stage[fmt]
        if fmt == nat.INPUT_U8_NV12:
            stage_nv12(s, x, h, w)
        elif fmt == nat.INPUT_U8_NHWC:
            s[:, :h, :w].copy_(x)
        else:
            s[:, :, :h, :w].copy_(x)
        return s

    def detect_raw(self, x, fmt, h, w, use_graph=True, outputs=True):
        """lfd_engine_detect on x (already in the capacity layout) -> its return code."""
        with torch.cuda.device(self.weights.device):
            return nat.lib().lfd_engine_detect(self.handle, nat.ptr(x), fmt, h, w, nat.ptr(self.dets), nat.ptr(self.labels), nat.ptr(self.count),
                                               nat.ptr(self.cls) if outputs else None, nat.ptr(self.reg) if outputs else None,
                                               int(bool(use_graph)), nat.stream_ptr())

    def detect(self, x, fmt, h, w, use_graph=True, outputs=True):
        """-> (cls [N,P,C'], reg [N,P,4] of the frame (None without outputs), dets, labels, count [N + 1]), the engine's buffers."""
        nat.check(self.detect_raw(self.capacity_input(x, fmt, h, w), fmt, h, w, use_graph, outputs))
        return self.dets, self.labels, self.count

    def frame_outputs(self, P):
        n, c = self.N, self.desc.cls_channels
        return self.cls.view(-1)[:n * P * c].view(n, P, c), self.reg.view(-1)[:n * P * 4].view(n, P, 4)

    def __del__(self):
        try:
            if self.handle:
                nat.lib().lfd_engine_close(self.handle)
                self.handle = None
        except Exception:
            pass


def rows(dets, labels, count):
    """predict_for_single_image's rows of every image: [label, score, x, y, w, h] with w = x2 - x1 + 1, h = y2 - y1 + 1 in float32."""
    from lfd.model.lfd import LFD
    n = count.shape[0] - 1
    return LFD._rows(dets, labels, count[:n], count[n:], dets.shape[1])
