# -*- coding: utf-8 -*-
"""The training input kernel (lfd_input_batch) and the DataLoader built on it, against the numpy oracle (tests/input_oracle.py):
bit for bit across channels, scales (copy, INTER_AREA at s = 0.5, down- and upscaling), crops inside / over / outside the resized
image, flip, channel swap, crop sizes, both output modes and the three normalisations, mixed-size batches; then the loader under the
WIDERFACE, TT100K and TrafficLight pipelines, and Executor.train fed by the loader against the same steps fed the oracle's batch."""
import ctypes as C
import os
import random

import numpy as np
import pytest
import torch

import input_oracle as O
from helpers import synth_model
from lfd import _native as nat
from lfd.data_pipeline.augmentation import (BGR2RGB, Compose, HorizontalFlip, bbox_param, caffe_imagenet_normalize, pipeline_device_spec,
                                            simple_normalize, simple_widerface_train_pipeline, standard_normalize)
from lfd.data_pipeline.data_loader import DataLoader
from lfd.data_pipeline.data_loader.data_loader import source_window
from lfd.data_pipeline.sampler import RandomBBoxCropRegionSampler, RandomWithNegDatasetSampler, TypicalCOCOTrainingRegionSampler
from lfd.data_pipeline.sampler.region_sampler import apply_draw, resize_plan
from lfd.execution.executor import Executor

pytestmark = pytest.mark.gpu
NORMS = {'simple': simple_normalize, 'standard': standard_normalize, 'caffe': caffe_imagenet_normalize}


def _image(rng, h, w, ch):
    return rng.integers(0, 256, (h, w, 3) if ch == 3 else (h, w), dtype=np.uint8)


def run_kernel(items, out_mode, swap_rb=False, H=None, W=None, mean=(0, 0, 0), scale=(1, 1, 1)):
    """items as in input_oracle.build_batch; each image's window is the rectangle source_window() gives."""
    H = max(it[4] for it in items) if H is None else H
    W = max(it[5] for it in items) if W is None else W
    descs = (nat.InputDesc * len(items))()
    chunks, off = [], 0
    for j, (img, s, cx, cy, oh, ow, flip) in enumerate(items):
        h, w = img.shape[:2]
        ch = 1 if img.ndim == 2 else 3
        mode, dh, dw = resize_plan(h, w, s)
        wx, wy, ww, wh = source_window(h, w, s, (cx, cy, ow, oh))
        win = np.ascontiguousarray(img[wy:wy + wh, wx:wx + ww]).reshape(-1)
        descs[j] = nat.InputDesc(off, 1.0 / s, ww * ch, ch, wx, wy, ww, wh, w, h, dw, dh, mode, cx, cy, ow, oh, int(flip))
        chunks.append(win)
        chunks.append(np.zeros((-win.size) % 16 + 16, np.uint8))     # windows are not contiguous: a read past one would show
        off += win.size + (-win.size) % 16 + 16
    src = torch.from_numpy(np.concatenate(chunks) if chunks else np.zeros(16, np.uint8)).cuda()
    d = torch.frombuffer(bytearray(bytes(descs)), dtype=torch.uint8).cuda()
    out = torch.full((len(items), H, W, 3) if out_mode == O.OUT_U8_NHWC else (len(items), 3, H, W), 77,
                     dtype=torch.uint8 if out_mode == O.OUT_U8_NHWC else torch.float32, device='cuda')
    m, sc = (C.c_float * 3)(*[float(v) for v in mean]), (C.c_float * 3)(*[float(v) for v in scale])
    nat.check(nat.lib().lfd_input_batch(nat.ptr(d), len(items), nat.ptr(src), nat.ptr(out), out_mode, int(swap_rb), H, W, m, sc, nat.stream_ptr()))
    torch.cuda.synchronize()
    return out.cpu().numpy()


def _items(seed, n, crop, ch, scales, flip):
    rng = np.random.default_rng(seed)
    out = []
    for j in range(n):
        h, w = int(rng.integers(crop // 2, 2 * crop)) | 1, int(rng.integers(crop // 2, 2 * crop))
        s = scales[j % len(scales)]
        _, dh, dw = resize_plan(h, w, s)
        cx, cy = int(rng.integers(-crop // 2, max(1, dw - crop // 2))), int(rng.integers(-crop // 2, max(1, dh - crop // 2)))
        out.append((_image(rng, h, w, ch), s, cx, cy, crop, crop, flip if flip is not None else bool(j % 2)))
    return out


@pytest.mark.parametrize('crop', [480, 512, 640, 37])
@pytest.mark.parametrize('ch', [1, 3])
@pytest.mark.parametrize('swap', [False, True])
def test_kernel_u8_matches_oracle(crop, ch, swap):
    scales = [0.5, 1.0, 0.73, 1.37, 2.3, 0.5000001, 32 / 64]
    items = _items(crop * 10 + ch + swap, 7, crop, ch, scales, None)
    ref = O.build_batch(items, O.OUT_U8_NHWC, swap_rb=swap)
    got = run_kernel(items, O.OUT_U8_NHWC, swap_rb=swap)
    assert np.array_equal(got, ref)


@pytest.mark.parametrize('norm', list(NORMS))
@pytest.mark.parametrize('swap', [False, True])
def test_kernel_f32_matches_oracle_mixed_sizes(norm, swap):
    rng = np.random.default_rng(7)
    items = []
    for j, (oh, ow) in enumerate([(64, 96), (33, 17), (128, 128), (5, 200), (96, 64)]):
        h, w = int(rng.integers(20, 300)), int(rng.integers(20, 300))
        s = [0.5, 1.0, float(rng.uniform(0.5, 1.5)), 1.9, 0.61][j]
        _, dh, dw = resize_plan(h, w, s)
        cx, cy = [(0, 0), (-10, -7), (dw - 20, dh - 30), (dw + 5, 0), (-200, dh + 1)][j]       # inside, over every edge, fully outside
        items.append((_image(rng, h, w, 3 if j % 2 == 0 else 1), s, cx, cy, oh, ow, j in (1, 2)))
    mean, scale = NORMS[norm].constants()
    ref = O.build_batch(items, O.OUT_F32_NCHW, swap_rb=swap, mean=mean, scale=scale)
    got = run_kernel(items, O.OUT_F32_NCHW, swap_rb=swap, mean=mean, scale=scale)
    assert got.shape == ref.shape and np.array_equal(got.view(np.uint32), ref.view(np.uint32))


def test_kernel_odd_widths_and_random_scales():
    rng = np.random.default_rng(11)
    for k in range(6):
        items = [(_image(rng, int(rng.integers(3, 90)), int(rng.integers(3, 90)), int(rng.choice([1, 3]))), float(rng.uniform(0.5, 1.5)),
                  int(rng.integers(-8, 8)), int(rng.integers(-8, 8)), 23 + k, 29 + 2 * k, bool(rng.integers(2))) for _ in range(5)]
        assert np.array_equal(run_kernel(items, O.OUT_U8_NHWC), O.build_batch(items, O.OUT_U8_NHWC))


# ------------------------------------------------------------------------------------------------------------------ loader
class MemoryDataset(object):
    def __init__(self, seed, n=12, size=(120, 260), num_classes=3):
        rng = np.random.default_rng(seed)
        self.samples = {}
        for i in range(n):
            h, w = int(rng.integers(*size)), int(rng.integers(*size))
            s = {'image': _image(rng, h, w, 1 if i % 5 == 4 else 3), 'image_id': i}
            if i % 4 != 3:
                k = int(rng.integers(1, 5))
                bw, bh = rng.integers(8, 60, k), rng.integers(8, 60, k)
                s['bboxes'] = [[int(rng.integers(0, w - a)), int(rng.integers(0, h - b)), int(a), int(b)] for a, b in zip(bw, bh)]
                s['bbox_labels'] = [int(v) for v in rng.integers(0, num_classes, k)]
            self.samples[i] = s

    def __len__(self):
        return len(self.samples)

    def __getitem__(self, i):
        return self.samples[i]

    def get_indexes(self):
        return list(self.samples.keys())


def _oracle_batches(dataset, sampler, region_sampler, pipeline, out_mode=O.OUT_F32_NCHW):
    """The same draws as the loader, in its order, rendered by the oracle."""
    flip_p = {b: pipeline_device_spec(pipeline, b)[0] for b in (False, True)}
    _, swap, mean, scale = pipeline_device_spec(pipeline, False)
    out = []
    for index_batch in list(sampler):
        items, anns = [], []
        for i in index_batch:
            smp = dataset[i]
            tmp = {k: v for k, v in smp.items() if k != 'image'}
            d = region_sampler.draw(tmp, image_shape=smp['image'].shape[:2])
            apply_draw(tmp, d)
            p = flip_p['bboxes' in tmp]
            flip = p is not None and random.random() < p
            boxes = tmp.get('bboxes', [])
            if flip:
                boxes = [(d.crop[2] - b[0] - b[2], b[1], b[2], b[3]) for b in boxes]
            items.append((smp['image'], d.scale, d.crop[0], d.crop[1], d.crop[3], d.crop[2], flip))
            anns.append((np.array(boxes, np.float32).reshape(-1, 4), np.array(tmp.get('bbox_labels', []), np.int64)))
        out.append((O.build_batch(items, out_mode, swap_rb=swap, mean=mean, scale=scale), anns))
    return out


def _tl_pipeline():
    return Compose([BGR2RGB(), standard_normalize], bbox_params=bbox_param, p=1.)


def _tt_pipeline(sample):      # the shape of the shipped config files: a function choosing a Compose by the sample's keys
    with_boxes = Compose([simple_normalize], bbox_params=bbox_param, p=1.)
    without = Compose([simple_normalize], p=1.)
    return with_boxes(**sample) if 'bboxes' in sample else without(**sample)


@pytest.mark.parametrize('name', ['WIDERFACE', 'TT100K', 'TrafficLight', 'COCO'])
@pytest.mark.parametrize('workers', [1, 3])
def test_loader_matches_oracle(name, workers):
    pipeline = {'WIDERFACE': simple_widerface_train_pipeline, 'TT100K': _tt_pipeline, 'TrafficLight': _tl_pipeline(),
                'COCO': Compose([HorizontalFlip(p=0.5), caffe_imagenet_normalize], bbox_params=bbox_param)}[name]
    ds = MemoryDataset(3)
    region = (TypicalCOCOTrainingRegionSampler((96, 128), 200, 32) if name == 'COCO' else
              RandomBBoxCropRegionSampler(crop_size=96, resize_range=(0.5, 1.5), resize_prob=0.5))
    random.seed(5), np.random.seed(5)
    loader = DataLoader(ds, RandomWithNegDatasetSampler(ds, batch_size=4, neg_ratio=0.25), region, pipeline, num_workers=workers)
    assert loader.on_device
    got = [(x.float().cpu().numpy(), ann, meta) for x, ann, meta in loader]
    random.seed(5), np.random.seed(5)
    ref = _oracle_batches(ds, RandomWithNegDatasetSampler(ds, batch_size=4, neg_ratio=0.25), region, pipeline)
    assert len(got) == len(ref) == len(loader)
    for (x, ann, meta), (rx, rann) in zip(got, ref):
        if x.ndim == 4 and x.shape[-1] == 3 and name in ('WIDERFACE', 'TT100K'):        # uint8 NHWC: normalise like the fused stem does
            x = ((x.astype(np.float32) - np.float32(127.5)) * (np.float32(1.0) / np.float32(127.5))).transpose(0, 3, 1, 2)
        assert x.shape == rx.shape and np.array_equal(x, rx)
        for (b, l), (rb, rl) in zip(ann, rann):
            assert b.dtype == np.float32 and l.dtype == np.int64 and np.array_equal(b, rb) and np.array_equal(l, rl)
        assert all(m is not None and 'image_id' in m for m in meta)


def test_executor_fed_by_loader_matches_oracle_batches(tmp_path):
    ds = MemoryDataset(9, n=12, size=(140, 220), num_classes=1)
    region = RandomBBoxCropRegionSampler(crop_size=128, resize_range=(0.5, 1.5), resize_prob=0.5)

    def config(loader, work):
        model, _ = synth_model('WIDERFACE_XS', cls_bias=-2.0)
        opt = torch.optim.SGD(model.parameters(), lr=0.02, momentum=0.9, weight_decay=1e-4)
        return dict(work_dir=os.path.join(str(tmp_path), work), log_path=None, model=model, optimizer=opt,
                    lr_scheduler=torch.optim.lr_scheduler.MultiStepLR(opt, milestones=[5]), training_epochs=1, gpu_list=[0],
                    train_data_loader=loader, val_data_loader=None, evaluator=None, val_interval=0, save_interval=100, display_interval=1,
                    optimizer_grad_clip_cfg=dict(max_norm=10, norm_type=2), resume_path=None, weight_path=None)

    def recording(batches, cfg, fed, losses):
        for batch in batches:
            fed.append(batch[0].clone())
            yield batch
            losses.append(float(cfg['loss'].detach()))

    random.seed(1), np.random.seed(1)
    loader = DataLoader(ds, RandomWithNegDatasetSampler(ds, batch_size=4, neg_ratio=0.25), region, simple_widerface_train_pipeline)
    a, fed_a, loss_a = config(None, 'a'), [], []
    a['train_data_loader'] = recording(loader, a, fed_a, loss_a)
    Executor(a).train()
    random.seed(1), np.random.seed(1)
    ref = _oracle_batches(ds, RandomWithNegDatasetSampler(ds, batch_size=4, neg_ratio=0.25), region, simple_widerface_train_pipeline,
                          O.OUT_U8_NHWC)
    assert len(ref) >= 3 and len(fed_a) == len(ref)
    assert all(torch.equal(x.cpu(), torch.from_numpy(r)) for x, (r, _) in zip(fed_a, ref))      # every step saw the oracle's pixels
    b, fed_b, loss_b = config(None, 'b'), [], []
    b['train_data_loader'] = recording([(torch.from_numpy(x).cuda(), ann, [None] * len(ann)) for x, ann in ref], b, fed_b, loss_b)
    Executor(b).train()
    assert a['train_iter'] == b['train_iter'] == len(ref) == len(loss_a) == len(loss_b)
    assert loss_a[0] == loss_b[0], (loss_a, loss_b)          # same parameters, same pixels: the same first loss
    # later steps agree up to the order of the fp32 atomics of the weight-gradient staging, which the SGD steps amplify
    # (test_gpu_executor.py; observed 0.7 % on the third loss)
    assert all(abs(x - y) <= 3e-2 * abs(y) for x, y in zip(loss_a, loss_b)), (loss_a, loss_b)
    for (name, p), q in zip(a['model'].state_dict().items(), b['model'].state_dict().values()):
        assert p.dtype.is_floating_point or torch.equal(p, q), name


def test_u8_batch_through_the_forward_equals_fp32():
    """The loader's uint8 NHWC batch (simple_normalize fused into the stem) and the same batch normalised to fp32 NCHW by the kernel
    give the same forward."""
    rng = np.random.default_rng(2)
    items = [(_image(rng, 150, 170, 3), s, -5, 7, 128, 128, bool(j % 2)) for j, s in enumerate([0.5, 1.0, 0.8, 1.3])]
    mean, scale = simple_normalize.constants()
    x8 = torch.from_numpy(run_kernel(items, O.OUT_U8_NHWC)).cuda()
    x32 = torch.from_numpy(run_kernel(items, O.OUT_F32_NCHW, mean=mean, scale=scale)).cuda()
    model, _ = synth_model('WIDERFACE_XS', cls_bias=-2.0)
    model.cuda().eval()
    with torch.no_grad():
        c8, r8 = model(x8)
        c32, r32 = model(x32)
    assert torch.equal(c8, c32) and torch.equal(r8, r32), ((c8 - c32).abs().max().item(), (r8 - r32).abs().max().item())
