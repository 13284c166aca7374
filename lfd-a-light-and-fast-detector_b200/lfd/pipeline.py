# -*- coding: utf-8 -*-
"""StreamingDetector -- end-to-end batched inference from HOST frames to HOST detections.

Pipelined over three streams: the host->device copy of batch i+1 (copy stream) overlaps the forward of batch i (forward
stream), whose score / decode / NMS and the small device->host read of the results (post stream) in turn overlap the
forward of batch i+1.  This is the serving-side
counterpart of the reference's `predict_for_single_image` (lfd/model/lfd.py:544-655), which moves one image at a time
and synchronises after every stage.
"""
import math
import os
import torch

from . import _native as nat


def bind_host_to_gpu_numa_node(device):
    """Restrict this process to the CPU cores of the NUMA node the GPU hangs off (sysfs), so that host buffers pinned afterwards
    are first-touched on that node and the H2D DMA does not cross the inter-socket link.  One process per GPU (the layout of
    bench.py / the Executor), so the affinity is per GPU.  Returns the node (None when the topology cannot be read)."""
    import os
    try:
        props = torch.cuda.get_device_properties(device)
        bdf = '%04x:%02x:%02x.0' % (props.pci_domain_id, props.pci_bus_id, props.pci_device_id)
        node = int(open('/sys/bus/pci/devices/%s/numa_node' % bdf).read().strip())
        if node < 0:
            return None
        cpus = set()
        for part in open('/sys/devices/system/node/node%d/cpulist' % node).read().strip().split(','):
            lo, _, hi = part.partition('-')
            cpus.update(range(int(lo), int(hi or lo) + 1))
        allowed = os.sched_getaffinity(0) & cpus
        if allowed:
            os.sched_setaffinity(0, allowed)
            return node
    except Exception:
        pass
    return None


class ForwardPostPipeline(object):
    """Software pipeline over batches on two streams: forward(i+1) starts as soon as forward(i) is done, while the (small,
    latency-bound) score / decode / NMS kernels of batch i run next to it.  The forward writes alternating output slots; a
    slot is rewritten only after its post-process has finished.  The post-process buffers are single: `consume(results)`
    is called with the post stream current, enqueue device->host copies (or anything else that reads them) there."""

    def __init__(self, model, plan, post, score_thr, iou_thr, frame_format=None, resize_scale=None):
        """frame_format: of the device inputs, passed to plan.forward (None: float32 NCHW or uint8 BGR by dtype, 'nv12': NV12 frames,
        'yuy2' / 'uyvy' / 'bgra' / 'rgba': packed camera frames);
        resize_scale: passed to plan.forward as well (the inputs are frames of another size, resized on the forward stream)."""
        self.model, self.plan, self.post = model, plan, post
        self.frame_format, self.resize_scale = frame_format, resize_scale
        self.score_thr, self.iou_thr = float(score_thr), float(iou_thr)
        dev = plan.device
        with torch.cuda.device(dev):
            self.fwd_stream = torch.cuda.Stream(device=dev)
            # highest priority the device offers (torch maps out-of-range values to it): the post-process kernels are tiny and
            # latency-bound; with a priority above the forward graph's nodes their CTAs are placed at the first kernel boundary of the
            # NEXT batch's forward instead of queueing behind its persistent CTAs
            self.post_stream = torch.cuda.Stream(device=dev, priority=-100)
        self.n_slots = 2                # output pairs of the plan: the forward of batch i+1 writes one while batch i is post-processed
        self.fwd_done = [torch.cuda.Event() for _ in range(self.n_slots)]
        self.post_done = [torch.cuda.Event() for _ in range(self.n_slots)]
        self.k = 0

    def enqueue(self, x, wait_for=None, consume=None):
        """x: device input of the plan; wait_for: optional event the forward has to wait for (e.g. the H2D copy of x)."""
        slot = self.k % self.n_slots
        with torch.cuda.stream(self.fwd_stream):
            if wait_for is not None:
                self.fwd_stream.wait_event(wait_for)
            if self.k >= self.n_slots:
                self.fwd_stream.wait_event(self.post_done[slot])
            cls, reg = self.plan.forward(x, use_graph=self.model.use_cuda_graph, slot=slot, frame_format=self.frame_format,
                                         resize_scale=self.resize_scale)
            self.fwd_done[slot].record(self.fwd_stream)
        with torch.cuda.stream(self.post_stream):
            self.post_stream.wait_event(self.fwd_done[slot])
            results = self.post.run(cls, reg, self.score_thr, self.iou_thr)
            if consume is not None:
                consume(results)
            self.post_done[slot].record(self.post_stream)
        self.k += 1
        return results


class StreamingDetector(object):

    def __init__(self, model, batch, height, width, score_thr, iou_thr, max_out=1024, device=None, depth=3, copy_streams=4,
                 input_pipeline=None, frame_format='bgr', source_size=None, resize_scale=None):
        """input_pipeline: the model's val pipeline, run on the uint8 frames inside the stem kernel -- None: simple_normalize on BGR;
        else BGR2RGB / a final Normalize of the declarative stand-ins (lfd/data_pipeline/augmentation.py), e.g. the TrafficLight
        val_pipeline.  A pipeline the kernels cannot run raises ValueError here: frames are never normalised other than asked.
        frame_format: 'bgr' -- host frames uint8 [N,H,W,3]; 'nv12' -- NV12 video frames uint8 [N,3H/2,W] (H and W even), half the bytes
        to copy, converted to BGR inside the stem kernel bit for bit as cv2.cvtColor(frame, cv2.COLOR_YUV2BGR_NV12) would, after which
        input_pipeline applies as it does to BGR frames; 'gray' -- uint8 [N,H,W], for a gray model (a 1-channel stem conv).  A gray model
        takes 'gray' or 'nv12', of which it reads the Y plane only (cv2.COLOR_YUV2GRAY_NV12), and raises ValueError for 'bgr'; a BGR model
        raises ValueError for 'gray'.  'yuy2' / 'uyvy' -- YUV 4:2:2 camera frames uint8 [N,H,W,2] (W even; a gray model reads their Y
        bytes, cv2.COLOR_YUV2GRAY_YUY2 / _UYVY) and 'bgra' / 'rgba' -- uint8 [N,H,W,4] (BGR models only, the alpha byte is never read):
        converted inside the stem kernels (or the resize) bit for bit as cv2.cvtColor(frame, cv2.COLOR_{YUY2,UYVY,BGRA,RGBA}2BGR) would.
        source_size=(h, w): the host frames are h x w (any size, in frame_format) and height x width stays the network's input size (the
        plan's capacity).  Each batch goes up at source size and is resized on the device, on the forward stream, exactly as
        cv2.resize(frame, (0, 0), fx=s, fy=s) would (NV12: cv2.resize of the converted frame); the network runs at the resized size, and the
        detections are in source-frame coordinates: the post-process takes the reference's meta of a resized image, int(w * s) x int(h * s)
        and resize_scale s.  resize_scale=None takes the largest s whose result fits: min(height / h, width / w); an explicit scale whose
        result does not fit raises ValueError."""
        from ._engine import image_channels, PACKED_FORMATS
        if frame_format not in ('bgr', 'nv12', 'gray') and frame_format not in PACKED_FORMATS:
            raise ValueError("frame_format must be 'bgr' or 'nv12' ('gray' for a gray model), got %r (packed camera frames: 'yuy2', 'uyvy', "
                             "'bgra', 'rgba')" % (frame_format,))
        if source_size is None and resize_scale is not None:
            raise ValueError('resize_scale needs source_size: the size of the frames it resizes')
        src_h, src_w = (height, width) if source_size is None else (int(source_size[0]), int(source_size[1]))
        if frame_format == 'nv12' and (src_h % 2 or src_w % 2):
            raise ValueError('NV12 frames have an even height and width, got %dx%d' % (src_h, src_w))
        if frame_format in ('yuy2', 'uyvy') and src_w % 2:
            raise ValueError('4:2:2 frames have an even width, got %dx%d' % (src_h, src_w))
        self.source_size, self.resize_scale = None, None
        meta, (dh, dw) = (width, height, 1.0), (height, width)
        if source_size is not None:
            s = min(height / src_h, width / src_w) if resize_scale is None else float(resize_scale)
            try:
                _, dh, dw = nat.resize_query(src_h, src_w, s)
            except nat.LfdError as e:
                raise ValueError(str(e))
            if dh > height or dw > width:
                raise ValueError('%dx%d frames at resize scale %r are %dx%d, beyond the network size %dx%d' % (src_h, src_w, s, dh, dw, height, width))
            self.source_size, self.resize_scale = (src_h, src_w), s
            meta = (int(src_w * s), int(src_h * s), s)       # the reference's resized_width / resized_height / resize_scale
        gray = image_channels(model) == 1
        if gray and frame_format in ('bgra', 'rgba'):
            raise ValueError("a gray model takes frame_format 'gray', 'nv12', 'yuy2' or 'uyvy'; %r frames are colour" % (frame_format,))
        if gray != (frame_format == 'gray') and frame_format not in ('nv12', 'yuy2', 'uyvy', 'bgra', 'rgba'):
            raise ValueError("a %s model takes frame_format '%s' or 'nv12', got %r" % ('gray' if gray else 'BGR', 'gray' if gray else 'bgr', frame_format))
        self.frame_format = frame_format
        from .data_pipeline.augmentation import input_transform_of
        self.input_transform = input_transform_of(input_pipeline, channels=1 if gray else 3)
        self.model = model
        self.depth = max(2, int(depth))     # batches in flight: copy of i+2 | forward of i+1 | post-process + read-back of i
        self.device = device if device is not None else next(model.parameters()).device
        self.N, self.H, self.W = batch, height, width
        self.score_thr, self.iou_thr = float(score_thr), float(iou_thr)
        self.max_out = min(int(max_out), int(model.max_detections_per_image))
        dev = self.device
        with torch.cuda.device(dev):
            # the batch goes up in `copy_streams` chunks on as many streams: several DMA transfers in flight fill the PCIe link better
            # than one 22 MB copy (measured in bench.py: e2e.h2d_gbps; 1 / 2 / 4 streams: 0.606 / 0.609 / 0.597 ms per step end to end.
            # The copy itself costs the forward ~8 %: 0.561 ms per step with the input copy left out, tests/debug_e2e_timeline.py)
            self.copy_streams = [torch.cuda.Stream(device=dev) for _ in range(max(1, min(int(copy_streams), batch)))]
            self.copy_stream = self.copy_streams[0]
        own, model.input_transform = getattr(model, 'input_transform', None), self.input_transform
        try:
            self.plan = model.inference_plan(batch, height, width, dev, exact=True)
        finally:
            model.input_transform = own
        if getattr(model, 'use_cuda_graph', True) and not self.plan.autotuned:
            self.plan.autotune()
        # the level geometry of the frames the network runs on: the capacity's, or that of the resized extent below it
        level_sizes = self.plan.level_sizes if (dh, dw) == (height, width) else self.plan.extent_table(dh, dw)[1]
        for i, hw in enumerate(level_sizes):
            model._head_indexes_to_feature_map_sizes[i] = hw
        self.post = model.post_plan(batch, level_sizes, dev)   # greedy NMS or Soft-NMS: model._nms_cfg as of now
        self.post.set_meta([meta[0]] * batch, [meta[1]] * batch, [meta[2]] * batch)
        device_format = frame_format if frame_format == 'nv12' or frame_format in PACKED_FORMATS else None
        self.pipe = ForwardPostPipeline(model, self.plan, self.post, self.score_thr, self.iou_thr, frame_format=device_format,
                                        resize_scale=self.resize_scale)
        if frame_format == 'nv12':
            frame_shape = (batch, src_h * 3 // 2, src_w)
        elif frame_format in PACKED_FORMATS:
            frame_shape = (batch, src_h, src_w, PACKED_FORMATS[frame_format][1])
        else:
            frame_shape = self.plan.u8_shape(src_h, src_w)
        self.slots = []
        for _ in range(self.depth):
            self.slots.append(dict(
                x=torch.empty(frame_shape, dtype=torch.uint8, device=dev),
                out_dets=torch.empty((batch, self.max_out, 5), dtype=torch.float32).pin_memory(),
                out_labels=torch.empty((batch, self.max_out), dtype=torch.int32).pin_memory(),
                out_count=torch.empty((batch + 1,), dtype=torch.int32).pin_memory(),
                h2d=torch.cuda.Event(), h2d_aux=[torch.cuda.Event() for _ in self.copy_streams[1:]], done=torch.cuda.Event(), busy=False))
        self.step = 0
        self.h2d_bytes = math.prod(frame_shape)
        self.d2h_bytes = batch * self.max_out * (5 * 4 + 4) + (batch + 1) * 4

    def submit(self, frames_u8):
        """frames_u8: pinned (or pageable) host uint8 [N,H,W,3] (frame_format 'nv12': [N,3H/2,W]; 'gray': [N,H,W]; 'yuy2' / 'uyvy':
        [N,H,W,2]; 'bgra' / 'rgba': [N,H,W,4]); H x W is source_size
        when given.  Enqueues copy + compute; returns the slot index."""
        s = self.slots[self.step % self.depth]
        if s['busy']:
            s['done'].synchronize()
        self.stage_input(self.step % self.depth, frames_u8)

        def read_back(results):          # runs with the post-process stream current
            dets, labels, _, count = results
            s['out_dets'].copy_(dets[:, :self.max_out], non_blocking=True)
            s['out_labels'].copy_(labels[:, :self.max_out], non_blocking=True)
            s['out_count'].copy_(count, non_blocking=True)
            s['done'].record(self.pipe.post_stream)

        self.pipe.enqueue(s['x'], wait_for=s['h2d'], consume=read_back)
        s['busy'] = True
        self.step += 1
        return (self.step - 1) % self.depth

    def stage_input(self, slot, frames_u8):
        """Host -> device copy of one batch into slot `slot`, split over the copy streams; s['h2d'] fires when all of it landed."""
        s = self.slots[slot]
        k = len(self.copy_streams)
        bounds = [(self.N * i) // k for i in range(k + 1)]
        for i in range(1, k):
            with torch.cuda.stream(self.copy_streams[i]):
                s['x'][bounds[i]:bounds[i + 1]].copy_(frames_u8[bounds[i]:bounds[i + 1]], non_blocking=True)
                s['h2d_aux'][i - 1].record(self.copy_streams[i])
        with torch.cuda.stream(self.copy_stream):
            s['x'][bounds[0]:bounds[1]].copy_(frames_u8[bounds[0]:bounds[1]], non_blocking=True)
            for ev in s['h2d_aux']:
                self.copy_stream.wait_event(ev)
            s['h2d'].record(self.copy_stream)

    def collect(self, slot):
        """Blocks until the slot's results are on the host.  -> (dets [N,max_out,5], labels [N,max_out], counts [N])."""
        s = self.slots[slot]
        s['done'].synchronize()
        s['busy'] = False
        if int(s['out_count'][self.N]) != 0:
            raise nat.LfdError('post-process capacity overflow; raise model.max_detections_per_image')
        return s['out_dets'], s['out_labels'], s['out_count'][:self.N]

    def infer(self, frames_u8):
        return self.collect(self.submit(frames_u8))
