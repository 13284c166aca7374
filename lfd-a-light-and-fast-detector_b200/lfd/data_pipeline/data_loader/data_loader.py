# -*- coding: utf-8 -*-
"""DataLoader with the reference's interface (lfd/data_pipeline/data_loader/data_loader.py) whose pixel work runs on the GPU.

For each batch the host makes the random draws, decodes, and copies only the source rectangle each crop reads into a pinned staging
slot; one host-to-device copy and one lfd_input_batch launch on a side stream then resize, crop, flip, order the channels and
normalise the whole batch.  The consumer's stream waits on an event recorded after the kernel.

Draw order is fixed and does not depend on num_workers: the dataset sampler's draws for the whole epoch first (as the reference's
__iter__ queues every batch before its workers start), then for each image in order the region sampler's draws followed by the
flip's random.random() < p.  With one worker the reference makes the same sampler draws in the same order.  albumentations' own
use of the random stream (Compose and each transform draw for their `p`) is not reproduced: only the flip draws.

Batches are (image_batch, annotation_batch, meta_batch) as in the reference: annotations are (float32 [G, 4] xywh, int64 [G]) per
image, meta the sample's non-reserved keys (None when there are none).  image_batch is a CUDA tensor: uint8 NHWC BGR when every crop
has the same size and the pipeline is simple_normalize without channel swap (the model's stem fuses that normalisation), else
float32 NCHW normalised and zero-padded at the bottom-right like the reference's _image_batch_postprocess.  A pipeline other than
None, a Compose of the stand-ins in lfd.data_pipeline.augmentation, or a function choosing one by the sample's keys runs on the host
exactly as the reference does, and the batch goes to the device as float32 NCHW.

input_channels=1 feeds a gray (1-channel) model: the input kernel converts BGR sources to gray as cv2.cvtColor(COLOR_BGR2GRAY) at
decode, then resizes, crops and flips the gray image, and image_batch is uint8 [n, H, W] or float32 [n, 1, H, W] under the same rule
as above.  The draws, annotations and metas are those of input_channels=3.  Only the device path makes gray batches.

Under torch.distributed every rank makes every draw but decodes, copies and resamples only its shard_range of the batch and yields a
RankLocalBatch, which Executor.train / val use without slicing again.
"""
import ctypes as C
import random
import time
from concurrent.futures import ThreadPoolExecutor

import numpy
import torch

from ..augmentation import input_transform_of, pipeline_device_spec
from ..dataset import reserved_keys
from ..sampler.region_sampler import apply_draw, resize_plan, RESIZE_AREA2, RESIZE_LINEAR

__all__ = ['DataLoader', 'RankLocalBatch']

try:
    from turbojpeg import TurboJPEG as _TurboJPEG
    _turbojpeg = _TurboJPEG()
except Exception:  # noqa: BLE001 -- not installed or libturbojpeg missing: cv2 decodes, as in the reference
    _turbojpeg = None


class RankLocalBatch(tuple):
    """A (image_batch, annotation_batch, meta_batch) that already holds only this rank's share of the global batch."""


def decode_image(sample):
    if 'image' in sample:
        return sample['image']
    if 'image_bytes' in sample:
        data = sample['image_bytes']
    elif 'image_path' in sample:
        with open(sample['image_path'], 'rb') as f:
            data = f.read()
    else:
        raise ValueError('sample does not have "image", "image_bytes" or "image_path"!')
    if _turbojpeg is not None:
        try:
            return _turbojpeg.decode(data)
        except Exception:  # noqa: BLE001 -- not a JPEG: cv2 below, as the reference falls back
            pass
    import cv2
    image = cv2.imdecode(numpy.frombuffer(data, dtype=numpy.uint8), cv2.IMREAD_UNCHANGED)
    if image is None:
        raise ValueError('image could not be decoded')
    return image


def _encoded_size(data):
    """(h, w) from a JPEG's SOF or a PNG's IHDR header, None for anything else."""
    if data[:8] == b'\x89PNG\r\n\x1a\n':
        return int.from_bytes(data[20:24], 'big'), int.from_bytes(data[16:20], 'big')
    if data[:2] != b'\xff\xd8':
        return None
    i = 2
    while i + 9 < len(data):
        if data[i] != 0xff:
            return None
        marker = data[i + 1]
        if marker == 0xff:
            i += 1
            continue
        length = int.from_bytes(data[i + 2:i + 4], 'big')
        if 0xc0 <= marker <= 0xcf and marker not in (0xc4, 0xc8, 0xcc):
            return int.from_bytes(data[i + 5:i + 7], 'big'), int.from_bytes(data[i + 7:i + 9], 'big')
        i += 2 + length
    return None


def image_size(sample):
    """(h, w) of the sample's image, from the header when it is encoded (the other ranks' images are never decoded)."""
    if 'image' in sample:
        return tuple(sample['image'].shape[:2])
    data = sample.get('image_bytes')
    if data is None and 'image_path' in sample:
        with open(sample['image_path'], 'rb') as f:
            data = f.read()
    hw = _encoded_size(data) if data is not None else None
    return hw if hw is not None else tuple(decode_image(sample).shape[:2])


def _taps(lo, hi, scale, n):
    """Source indices [first, last] that cv2's INTER_LINEAR reads for resized indices lo..hi (input.cu: src_coord)."""
    f = ((numpy.array([lo, hi], numpy.float64) + 0.5) * (1.0 / scale) - 0.5).astype(numpy.float32)
    i = numpy.floor(f).astype(numpy.int64)
    return int(min(max(i[0], 0), n - 1)), int(min(max(i[1] + 1, 0), n - 1))


def source_window(h, w, scale, crop):
    """(x, y, w, h) of the source rectangle the kernel reads for `crop` of the image resized by `scale`; 0 x 0 when it misses."""
    mode, dh, dw = resize_plan(h, w, scale)
    cx, cy, cw, ch = crop
    r0, r1, c0, c1 = max(0, cy), min(dh, cy + ch) - 1, max(0, cx), min(dw, cx + cw) - 1
    if r1 < r0 or c1 < c0:
        return 0, 0, 0, 0
    if mode == RESIZE_AREA2:
        (y0, y1), (x0, x1) = (2 * r0, min(h - 1, 2 * r1 + 1)), (2 * c0, min(w - 1, 2 * c1 + 1))
    elif mode == RESIZE_LINEAR:
        (y0, y1), (x0, x1) = _taps(r0, r1, scale, h), _taps(c0, c1, scale, w)
    else:
        y0, y1, x0, x1 = r0, r1, c0, c1
    return x0, y0, x1 - x0 + 1, y1 - y0 + 1


def flip_boxes(bboxes, width):
    return [(width - b[0] - b[2], b[1], b[2], b[3]) for b in bboxes]


def _annotation(sample):
    if 'bboxes' in sample:
        return numpy.array(sample['bboxes'], dtype=numpy.float32).reshape(-1, 4), numpy.array(sample['bbox_labels'], dtype=numpy.int64)
    return numpy.empty((0, 4), dtype=numpy.float32), numpy.empty((0,), dtype=numpy.int64)


def _meta(sample):
    keys = set(sample.keys()) - set(reserved_keys)
    return {k: sample[k] for k in keys} if keys else None


def _sample_temp(sample):
    """The reference's per-image copy: boxes, labels and meta keys, never the image itself."""
    tmp = {k: sample[k] for k in set(sample.keys()) - set(reserved_keys)}
    if 'bboxes' in sample:
        tmp['bboxes'], tmp['bbox_labels'] = sample['bboxes'], sample['bbox_labels']
    return tmp


_DESC_ALIGN = 256


class _Slot(object):
    """Pinned staging memory for one batch: descriptors, then every source window.  Reused only after its copy finished."""

    def __init__(self):
        self.buffer, self.event = None, None

    def acquire(self, nbytes):
        if self.event is not None:
            self.event.synchronize()
        if self.buffer is None or self.buffer.numel() < nbytes:
            self.buffer = torch.empty(max(nbytes, 1 << 20) * 5 // 4, dtype=torch.uint8, pin_memory=True)
        return self.buffer


class DataLoader(object):

    def __init__(self, dataset, dataset_sampler, region_sampler, augmentation_pipeline=None, num_workers=1, model_normalizes=False,
                 input_channels=3):
        """model_normalizes: the model's stem kernels run the pipeline's channel swap and normalisation (LFD.set_input_transform with
        this loader's `input_transform`; Executor.train does that): batches of equal-size crops are then raw uint8 BGR NHWC, a quarter of
        the bytes, for every pipeline the input kernel can run.  The flip stays in the input kernel.  A batch with crops of different
        sizes is float32 NCHW, normalised here, as without the argument (its zero padding is zero AFTER normalisation, which no byte
        expresses); the model takes float32 batches as they are.
        input_channels: 3 (BGR batches) or 1 (gray batches for a gray model: uint8 [n, H, W] or float32 [n, 1, H, W]).  With 1 the pipeline
        must be one the input kernel runs, without BGR2RGB and with a Normalize of one constant or three equal ones (ValueError otherwise);
        gray and BGR sources both become gray, BGR ones as cv2.cvtColor(COLOR_BGR2GRAY) before the resize."""
        if input_channels not in (1, 3):
            raise ValueError('input_channels must be 3 (BGR) or 1 (gray), got %r' % (input_channels,))
        self._dataset = dataset
        self._dataset_sampler = dataset_sampler
        self._loops = len(dataset_sampler)
        self._batch_size = dataset_sampler.get_batch_size()
        self._region_sampler = region_sampler
        self._augmentation_pipeline = augmentation_pipeline
        self._num_workers = max(1, int(num_workers))
        self._pool = ThreadPoolExecutor(self._num_workers)
        specs = {b: pipeline_device_spec(augmentation_pipeline, b) for b in (False, True)}
        native = hasattr(region_sampler, 'draw') and all(s is not None for s in specs.values())
        if native:   # one batch = one launch: both variants must agree on channel order and normalisation
            (_, sw0, m0, s0), (_, sw1, m1, s1) = specs[False], specs[True]
            native = sw0 == sw1 and numpy.array_equal(m0, m1) and numpy.array_equal(s0, s1)
        self._specs = specs if native else None
        if model_normalizes and not native:
            raise ValueError('model_normalizes needs a region sampler with draw() and a pipeline the input kernel can run (flip, BGR2RGB, a final Normalize)')
        if input_channels == 1:
            if not native:
                raise ValueError('input_channels=1 needs a region sampler with draw() and a pipeline the input kernel can run (flip, a final '
                                 'Normalize): gray batches are made on the device only')
            input_transform_of(augmentation_pipeline, allow_flip=True, channels=1)     # ValueError for BGR2RGB or unequal constants
        self.input_channels = input_channels
        # what the model has to do to this loader's uint8 batches; None: simple_normalize, the only pipeline that gives uint8 batches
        # without model_normalizes
        self.input_transform = input_transform_of(augmentation_pipeline, allow_flip=True, channels=input_channels) if model_normalizes else None
        self._slots = [_Slot(), _Slot()]
        self._stream = None
        self.last_stats = None   # host timings / bytes of the last native batch (tests/debug_input_timing.py)

    def __len__(self):
        return self._loops

    @property
    def batch_size(self):
        return self._batch_size

    @property
    def on_device(self):
        """True when batches are built by the input kernel, False when the pipeline runs on the host."""
        return self._specs is not None

    def __iter__(self):
        index_batches = list(self._dataset_sampler)
        if self._specs is None:
            for index_batch in index_batches:
                yield self._host_batch(index_batch)
            return
        pending = None
        for k, index_batch in enumerate(index_batches):
            job = self._launch(index_batch, self._slots[k % len(self._slots)])
            if pending is not None:
                yield self._hand_over(pending)
            pending = job
        if pending is not None:
            yield self._hand_over(pending)

    # ------------------------------------------------------------------ host path (the reference's worker, unchanged semantics)
    def _host_batch(self, index_batch):
        images, annotations, metas = [], [], []
        for sample_index in index_batch:
            sample = self._dataset[sample_index]
            tmp = _sample_temp(sample)
            tmp['image'] = decode_image(sample)
            tmp = self._region_sampler(tmp)
            if tmp['image'].ndim == 2:
                tmp['image'] = numpy.tile(tmp['image'], (3, 1, 1)).transpose([1, 2, 0])
            if self._augmentation_pipeline is not None:
                tmp = self._augmentation_pipeline(tmp)
            images.append(tmp['image'])
            annotations.append(_annotation(tmp))
            metas.append(_meta(tmp))
        batch = numpy.zeros((len(images), max(i.shape[0] for i in images), max(i.shape[1] for i in images), 3), dtype=numpy.float32)
        for i, image in enumerate(images):
            batch[i, :image.shape[0], :image.shape[1]] = image
        batch = torch.from_numpy(batch.transpose([0, 3, 1, 2]))
        return (batch.cuda(non_blocking=False) if torch.cuda.is_available() else batch), annotations, metas

    # ------------------------------------------------------------------ device path
    def plan(self, index_batch, rank=0, world_size=1):
        """Every draw for one batch, in the fixed order; decodes (in the worker threads) only the images of this rank's shard.
        -> (items, annotations, metas, (H, W), (swap_rb, mean, scale), (begin, end)): items[j] = (image, RegionDraw, flip) and the
        annotations and meta of the images begin..end-1 of the batch; H x W is the largest crop of the whole batch."""
        from ...execution.parallel import shard_range
        b, e = shard_range(len(index_batch), rank, world_size)
        samples = [self._dataset[i] for i in index_batch]
        futures = {j: self._pool.submit(decode_image, samples[j]) for j in range(b, e)}
        items, annotations, metas = [], [], []
        for j, sample in enumerate(samples):
            image = futures[j].result() if j in futures else None
            if image is not None and image.ndim == 3 and image.shape[2] not in (1, 3):
                raise ValueError('image with %d channels: the loader takes gray or BGR images' % image.shape[2])
            tmp = _sample_temp(sample)
            d = self._region_sampler.draw(tmp, image_shape=image.shape[:2] if image is not None else image_size(sample))
            apply_draw(tmp, d)
            flip_p = self._specs['bboxes' in tmp][0]
            flip = flip_p is not None and random.random() < flip_p
            if flip and 'bboxes' in tmp:
                tmp['bboxes'] = flip_boxes(tmp['bboxes'], d.crop[2])
            items.append((image, d, flip))
            annotations.append(_annotation(tmp))
            metas.append(_meta(tmp))
        H, W = max(it[1].crop[3] for it in items), max(it[1].crop[2] for it in items)
        _, swap, mean, scale = self._specs[False]
        return items[b:e], annotations[b:e], metas[b:e], (H, W), (swap, mean, scale), (b, e)

    def _launch(self, index_batch, slot):
        from ...execution.parallel import world
        from ... import _native as nat
        t0 = time.perf_counter()
        rank, world_size = world()
        items, annotations, metas, (H, W), (swap, mean, scale), _ = self.plan(index_batch, rank, world_size)
        t1 = time.perf_counter()
        n = len(items)
        descs = (nat.InputDesc * max(n, 1))()
        off = (C.sizeof(descs) + _DESC_ALIGN - 1) // _DESC_ALIGN * _DESC_ALIGN
        copies = []
        for j, (image, d, flip) in enumerate(items):
            h, w = image.shape[:2]
            ch = 1 if image.ndim == 2 or image.shape[2] == 1 else 3
            mode, dh, dw = resize_plan(h, w, d.scale)
            wx, wy, ww, wh = source_window(h, w, d.scale, d.crop)
            cx, cy, cw, chh = d.crop
            descs[j] = nat.InputDesc(off, 1.0 / d.scale, ww * ch, ch, wx, wy, ww, wh, w, h, dw, dh, mode, cx, cy, cw, chh, int(flip))
            copies.append((image, off, wx, wy, ww, wh, ch))
            off += (ww * wh * ch + 15) // 16 * 16
        buf = slot.acquire(off)
        host = buf.numpy()
        C.memmove(buf.data_ptr(), C.addressof(descs), C.sizeof(nat.InputDesc) * n)

        def copy_window(args):
            image, o, wx, wy, ww, wh, ch = args
            host[o:o + ww * wh * ch].reshape(wh, ww, ch)[...] = image[wy:wy + wh, wx:wx + ww].reshape(wh, ww, ch)

        list(self._pool.map(copy_window, copies))
        t2 = time.perf_counter()
        device = torch.device('cuda', torch.cuda.current_device())
        if self._stream is None:
            self._stream = torch.cuda.Stream(device)
        self._stream.wait_stream(torch.cuda.current_stream(device))
        u8 = all(d.crop[2] == W and d.crop[3] == H for _, d, _ in items) and (self.input_transform is not None or (
            not swap and numpy.array_equal(mean, numpy.full(3, 127.5, numpy.float32)) and
            numpy.array_equal(scale, numpy.full(3, numpy.float32(1.0) / numpy.float32(127.5), numpy.float32))))
        if u8:
            swap = False     # raw BGR bytes: with model_normalizes the swap happens in the stem kernel
        gray = self.input_channels == 1     # swap is False: the constructor refused BGR2RGB
        with torch.cuda.stream(self._stream):
            staged = torch.empty(off, dtype=torch.uint8, device=device)
            staged.copy_(buf[:off], non_blocking=True)
            if u8:
                out = torch.empty((n, H, W) if gray else (n, H, W, 3), dtype=torch.uint8, device=device)
                mode = nat.INPUT_OUT_U8_GRAY if gray else nat.INPUT_OUT_U8_NHWC
            else:
                out = torch.empty((n, 1, H, W) if gray else (n, 3, H, W), dtype=torch.float32, device=device)
                mode = nat.INPUT_OUT_F32_GRAY if gray else nat.INPUT_OUT_F32_NCHW
            m, s = (C.c_float * 3)(*mean.tolist()), (C.c_float * 3)(*scale.tolist())
            nat.check(nat.lib().lfd_input_batch(C.c_void_p(staged.data_ptr()), n, C.c_void_p(staged.data_ptr()), nat.ptr(out), mode,
                                                int(swap), H, W, m, s, C.c_void_p(self._stream.cuda_stream)))
            slot.event = torch.cuda.Event()
            slot.event.record(self._stream)
        self.last_stats = dict(draw_decode_ms=(t1 - t0) * 1e3, copy_ms=(t2 - t1) * 1e3, h2d_bytes=off, images=n)
        batch_cls = RankLocalBatch if world_size > 1 else tuple
        return out, annotations, metas, slot.event, batch_cls

    def _hand_over(self, job):
        out, annotations, metas, event, batch_cls = job
        stream = torch.cuda.current_stream(out.device)
        stream.wait_event(event)
        out.record_stream(stream)
        return batch_cls((out, annotations, metas))
