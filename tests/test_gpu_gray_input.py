# -*- coding: utf-8 -*-
"""The gray modes of the training input kernel (lfd_input_batch LFD_INPUT_OUT_U8_GRAY / F32_GRAY) and DataLoader(input_channels=1),
bit for bit against the host rule they implement:

    g = image if image.ndim == 2 else cv2.cvtColor(image, cv2.COLOR_BGR2GRAY)
    g = crop_from_image(cv2.resize(g, (0, 0), fx=s, fy=s), crop)      # the region sampler's draw, on the 1-channel image (zero outside)
    g = g[:, ::-1] if flip else g
    uint8 batch [n, H, W]: g;  fp32 batch [n, 1, H, W]: (float32(g) - mean) * scale, zero-padded at the bottom-right

then a gray model trained through Executor from the loader against the same steps fed the rule's batches."""
import copy
import ctypes as C
import os
import random

import numpy as np
import pytest
import torch

from gen_golden_input import synthetic_samples
from gray_models import gray_pair
from helpers import ListDataset
from lfd import _native as nat
from lfd.data_pipeline import sampler as S
from lfd.data_pipeline.augmentation import Compose, HorizontalFlip, Normalize, bbox_param, pipeline_device_spec, simple_widerface_train_pipeline
from lfd.data_pipeline.data_loader import DataLoader
from lfd.data_pipeline.data_loader.data_loader import source_window
from lfd.data_pipeline.sampler.region_sampler import apply_draw, resize_plan
from lfd.execution.executor import Executor

cv2 = pytest.importorskip('cv2')
pytestmark = pytest.mark.gpu

GOLDEN = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'input_samplers.pt'), weights_only=False)
LFD_ERR_INVALID = 1          # include/lfd_b200.h
SENTINEL_U8, SENTINEL_F32 = 0xA5, -12345.5
EXTRA = 1031                 # elements of the output buffer past the batch: they must stay the sentinel


def _crop(image, x, y, w, h):
    """crop_from_image(image, (x, y, w, h)) of a 2-D image, also for a crop that misses the image entirely (all zero)."""
    out = np.zeros((h, w), image.dtype)
    y0, y1, x0, x1 = max(0, -y), min(h, image.shape[0] - y), max(0, -x), min(w, image.shape[1] - x)
    if y1 > y0 and x1 > x0:
        out[y0:y1, x0:x1] = image[y0 + y:y1 + y, x0 + x:x1 + x]
    return out


def rule_crop(image, s, cx, cy, oh, ow, flip):
    """uint8 [oh, ow]: the host pipeline the gray modes implement, with cv2."""
    g = image if image.ndim == 2 else cv2.cvtColor(image, cv2.COLOR_BGR2GRAY)
    g = _crop(cv2.resize(g, (0, 0), fx=s, fy=s), cx, cy, ow, oh)
    return np.ascontiguousarray(g[:, ::-1] if flip else g)


def rule_batch(items, f32, H, W, mean=0.0, scale=1.0):
    """items: (image, s, cx, cy, oh, ow, flip) -> uint8 [n, H, W] or float32 [n, 1, H, W] (numpy float32 arithmetic), zero-padded."""
    out = np.zeros((len(items), 1, H, W) if f32 else (len(items), H, W), np.float32 if f32 else np.uint8)
    for i, it in enumerate(items):
        g = rule_crop(*it)
        if f32:
            out[i, 0, :g.shape[0], :g.shape[1]] = (g.astype(np.float32) - np.float32(mean)) * np.float32(scale)
        else:
            out[i, :g.shape[0], :g.shape[1]] = g
    return out


def _descs_and_src(items):
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
    src = torch.from_numpy(np.concatenate(chunks)).cuda()
    d = torch.frombuffer(bytearray(bytes(descs)), dtype=torch.uint8).cuda()
    return d, src


def run_gray(items, f32, H, W, mean=0.0, scale=1.0, swap_rb=0, constants=True):
    """-> (return code, the batch, the output buffer's elements past the batch).  The buffer is larger than the batch and pre-filled."""
    d, src = _descs_and_src(items)
    numel = len(items) * H * W
    buf = torch.full((numel + EXTRA,), SENTINEL_F32 if f32 else SENTINEL_U8, dtype=torch.float32 if f32 else torch.uint8, device='cuda')
    m, sc = (C.c_float * 3)(mean, 0.0, 0.0), (C.c_float * 3)(scale, 0.0, 0.0)
    rc = nat.lib().lfd_input_batch(nat.ptr(d), len(items), nat.ptr(src), nat.ptr(buf), nat.INPUT_OUT_F32_GRAY if f32 else nat.INPUT_OUT_U8_GRAY,
                                   int(swap_rb), H, W, m if constants else None, sc if constants else None, nat.stream_ptr())
    torch.cuda.synchronize()
    host = buf.cpu().numpy()
    batch = host[:numel].reshape((len(items), 1, H, W) if f32 else (len(items), H, W))
    return rc, batch, host[numel:]


def _same(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint32) if a.dtype == np.float32 else a,
                                                                         b.view(np.uint32) if b.dtype == np.float32 else b)


# ------------------------------------------------------------------------------------------------------------------ kernel
def test_every_bgr_triple_converts_like_cv2():
    """One 4096 x 4096 BGR image holding all 2^24 (B, G, R) triples, copied (s = 1) in the uint8 gray mode."""
    v = np.arange(1 << 24, dtype=np.uint32)
    img = np.stack([v & 0xff, v >> 8 & 0xff, v >> 16], axis=-1).astype(np.uint8).reshape(4096, 4096, 3)
    rc, got, tail = run_gray([(img, 1.0, 0, 0, 4096, 4096, False)], False, 4096, 4096)
    assert rc == 0
    want = cv2.cvtColor(img, cv2.COLOR_BGR2GRAY)
    assert np.array_equal(got[0], want), int((got[0] != want).sum())
    assert (tail == SENTINEL_U8).all()


def _items(seed, n, crop_h, crop_w, scales):
    """Gray and BGR sources alternating; crops inside, over every edge and fully outside the resized image; flips alternating."""
    rng = np.random.default_rng(seed)
    out = []
    for j in range(n):
        h, w = max(4, int(rng.integers(crop_h // 2, 2 * crop_h + 3)) | 1), max(4, int(rng.integers(crop_w // 2, 2 * crop_w + 3)))
        img = rng.integers(0, 256, (h, w) if j % 2 else (h, w, 3), dtype=np.uint8)
        s = scales[j % len(scales)]
        _, dh, dw = resize_plan(h, w, s)
        cx, cy = [(0, 0), (-5, -3), (dw - crop_w + 4, dh - crop_h + 2), (int(rng.integers(0, max(1, dw - crop_w))), int(rng.integers(0, max(1, dh - crop_h)))),
                  (dw + 3, -crop_h - 1), (-7, dh - 1)][j % 6]
        out.append((img, s, cx, cy, crop_h, crop_w, bool(j % 3 == 1)))
    return out


SCALES = [1.0, 0.5, 0.73, 1.37, 0.5000001, 2.3, 32 / 64]     # copy, AREA2, LINEAR down and up


@pytest.mark.parametrize('crop', [(64, 64), (37, 53), (40, 29), (5, 2), (128, 131)])
@pytest.mark.parametrize('f32', [False, True])
def test_kernel_matches_the_rule(crop, f32):
    """Mixed gray and BGR sources in one batch, every resize mode, crops off every edge, flips, widths with W % 4 != 0; the batch
    equals the rule bit for bit and the buffer past it is untouched."""
    oh, ow = crop
    items = _items(oh * 1000 + ow + f32, 12, oh, ow, SCALES)
    mean, scale = (Normalize(mean=(0.4,), std=(0.3,)).constants() if f32 else (np.zeros(1), np.ones(1)))
    rc, got, tail = run_gray(items, f32, oh, ow, float(mean[0]), float(scale[0]))
    assert rc == 0
    want = rule_batch(items, f32, oh, ow, mean[0], scale[0])
    assert _same(got, want)
    assert (tail == (SENTINEL_F32 if f32 else SENTINEL_U8)).all()


@pytest.mark.parametrize('f32', [False, True])
def test_kernel_pads_mixed_sizes(f32):
    """Crops of different sizes in one batch: each in the top-left corner, the rest 0 (in fp32, 0 after normalisation)."""
    rng = np.random.default_rng(3)
    items = []
    for j, (oh, ow) in enumerate([(64, 96), (33, 17), (70, 101), (5, 200), (96, 64)]):
        h, w = int(rng.integers(20, 300)), int(rng.integers(20, 300))
        s = [0.5, 1.0, float(rng.uniform(0.5, 1.5)), 1.9, 0.61][j]
        _, dh, dw = resize_plan(h, w, s)
        cx, cy = [(0, 0), (-10, -7), (dw - 20, dh - 30), (dw + 5, 0), (-200, dh + 1)][j]
        items.append((rng.integers(0, 256, (h, w, 3) if j % 2 == 0 else (h, w), dtype=np.uint8), s, cx, cy, oh, ow, j in (1, 2)))
    H, W = max(it[4] for it in items), max(it[5] for it in items) + 3
    mean, scale = Normalize(mean=(0.5,) * 3, std=(0.5,) * 3).constants()
    rc, got, tail = run_gray(items, f32, H, W, float(mean[0]), float(scale[0]))
    assert rc == 0
    assert _same(got, rule_batch(items, f32, H, W, mean[0], scale[0]))
    assert (tail == (SENTINEL_F32 if f32 else SENTINEL_U8)).all()


@pytest.mark.parametrize('case', ['swap_u8', 'swap_f32', 'no_constants'])
def test_invalid_calls_write_nothing(case):
    rng = np.random.default_rng(5)
    items = [(rng.integers(0, 256, (50, 60, 3), dtype=np.uint8), 0.8, 2, 3, 32, 36, False)]
    f32 = case != 'swap_u8'
    rc, got, tail = run_gray(items, f32, 32, 36, 127.5, 1.0 / 127.5, swap_rb=case.startswith('swap'), constants=case != 'no_constants')
    assert rc == LFD_ERR_INVALID, rc
    sentinel = SENTINEL_F32 if f32 else SENTINEL_U8
    assert (got == sentinel).all() and (tail == sentinel).all()


# ------------------------------------------------------------------------------------------------------------------ loader
def _replay(ds, sampler, region, pipeline):
    """The loader's draws, in its order -> per batch the rule's items and the flipped annotations."""
    flip_p = {b: pipeline_device_spec(pipeline, b)[0] for b in (False, True)}
    out = []
    for index_batch in list(sampler):
        items = []
        for i in index_batch:
            smp = ds[i]
            tmp = {k: v for k, v in smp.items() if k != 'image'}
            d = region.draw(tmp, image_shape=smp['image'].shape[:2])
            apply_draw(tmp, d)
            p = flip_p['bboxes' in tmp]
            items.append((smp['image'], d.scale, d.crop[0], d.crop[1], d.crop[3], d.crop[2], p is not None and random.random() < p))
        out.append(items)
    return out


PIPELINES = {
    'widerface-model-normalizes': (simple_widerface_train_pipeline, True),
    'equal-constants': (Compose([HorizontalFlip(p=0.5), Normalize(mean=(0.4,) * 3, std=(0.3,) * 3)], bbox_params=bbox_param), False),
}


@pytest.mark.parametrize('k', range(len(GOLDEN['region'])))
@pytest.mark.parametrize('pipe', list(PIPELINES))
def test_loader_gray_batches_follow_the_rule(k, pipe):
    """Over the golden region samplers and samples: input_channels=1 makes the draws, annotations and metas of input_channels=3, and
    its images are the rule's -- uint8 [n, H, W] for equal crops under model_normalizes, float32 [n, 1, H, W] otherwise."""
    g = GOLDEN['region'][k]
    pipeline, model_normalizes = PIPELINES[pipe]
    ds = ListDataset(synthetic_samples())
    region = getattr(S, g['cls'])(**g['kwargs'])
    runs = {}
    for channels in (3, 1):
        random.seed(g['seed']), np.random.seed(g['seed'])
        loader = DataLoader(ds, S.RandomDatasetSampler(ds, batch_size=5), region, pipeline, num_workers=2, model_normalizes=model_normalizes,
                            input_channels=channels)
        assert loader.on_device and loader.input_channels == channels
        runs[channels] = [(x.cpu().numpy(), copy.deepcopy(ann), copy.deepcopy(meta)) for x, ann, meta in loader]
    random.seed(g['seed']), np.random.seed(g['seed'])
    ref = _replay(ds, S.RandomDatasetSampler(ds, batch_size=5), region, pipeline)
    assert len(runs[1]) == len(runs[3]) == len(ref) > 0
    _, _, mean, scale = pipeline_device_spec(pipeline, False)
    for (x1, ann1, meta1), (x3, ann3, meta3), items in zip(runs[1], runs[3], ref):
        for (b1, l1), (b3, l3) in zip(ann1, ann3):
            assert b1.dtype == np.float32 and l1.dtype == np.int64 and np.array_equal(b1, b3) and np.array_equal(l1, l3)
        assert meta1 == meta3
        H, W = max(it[4] for it in items), max(it[5] for it in items)
        equal = all(it[4] == H and it[5] == W for it in items)
        u8 = equal and (model_normalizes or (np.array_equal(mean, np.full(3, 127.5, np.float32)) and
                                             np.array_equal(scale, np.full(3, np.float32(1.0) / np.float32(127.5), np.float32))))
        assert (x3.dtype == np.uint8) == u8 and (x3.shape[-1] == 3 if u8 else x3.shape[1] == 3)     # the 3-channel loader, as before
        assert _same(x1, rule_batch(items, not u8, H, W, mean[0], scale[0]))


# ------------------------------------------------------------------------------------------------------------------ end to end
def test_gray_model_trains_from_the_gray_loader(tmp_path):
    """Two Executor steps of a gray model fed by DataLoader(input_channels=1, model_normalizes=True) against the same two steps fed the
    rule's uint8 [n, H, W] batches: every batch the same bytes, the first loss the same bits, the parameters the same up to the order of
    the fp32 atomics of the weight-gradient staging (test_gpu_input_pipeline.py, test_gpu_executor.py)."""
    rng = np.random.default_rng(9)
    samples = []
    for i in range(8):
        h, w = int(rng.integers(140, 220)), int(rng.integers(140, 220))
        s = {'image': rng.integers(0, 256, (h, w) if i % 3 == 2 else (h, w, 3), dtype=np.uint8), 'image_id': i}
        k = int(rng.integers(1, 4))
        bw, bh = rng.integers(12, 60, k), rng.integers(12, 60, k)
        s['bboxes'] = [[int(rng.integers(0, w - a)), int(rng.integers(0, h - b)), int(a), int(b)] for a, b in zip(bw, bh)]
        s['bbox_labels'] = [0] * k
        samples.append(s)
    ds = ListDataset(samples)
    region = S.RandomBBoxCropRegionSampler(crop_size=128, resize_range=(0.5, 1.5), resize_prob=0.5)

    def config(work):
        model, _ = gray_pair('WIDERFACE_XS', cls_bias=-2.0)
        opt = torch.optim.SGD(model.parameters(), lr=0.02, momentum=0.9, weight_decay=1e-4)
        return dict(work_dir=os.path.join(str(tmp_path), work), log_path=None, model=model.train(), optimizer=opt,
                    lr_scheduler=torch.optim.lr_scheduler.MultiStepLR(opt, milestones=[5]), training_epochs=1, gpu_list=[0],
                    train_data_loader=None, val_data_loader=None, evaluator=None, val_interval=0, save_interval=100, display_interval=1,
                    optimizer_grad_clip_cfg=dict(max_norm=10, norm_type=2), resume_path=None, weight_path=None)

    def recording(batches, cfg, fed, losses):
        for batch in batches:
            fed.append((batch[0].clone(), batch[1]))
            yield batch
            losses.append(float(cfg['loss'].detach()))

    random.seed(1), np.random.seed(1)
    loader = DataLoader(ds, S.RandomDatasetSampler(ds, batch_size=4), region, simple_widerface_train_pipeline, model_normalizes=True,
                        input_channels=1)
    a, fed_a, loss_a = config('a'), [], []
    ex = Executor(a)
    ex._set_input_transform(loader)          # what Executor.train does with the loader itself; the recording wrapper hides it
    a['train_data_loader'] = recording(loader, a, fed_a, loss_a)
    ex.train()
    random.seed(1), np.random.seed(1)
    ref = _replay(ds, S.RandomDatasetSampler(ds, batch_size=4), region, simple_widerface_train_pipeline)
    assert len(ref) == len(fed_a) == 2
    for (x, _), items in zip(fed_a, ref):
        assert x.dtype == torch.uint8 and tuple(x.shape) == (4, 128, 128)
        assert _same(x.cpu().numpy(), rule_batch(items, False, 128, 128))
    b, fed_b, loss_b = config('b'), [], []
    exb = Executor(b)
    exb.config_dict['model'].set_input_transform(loader.input_transform)
    host = [(torch.from_numpy(rule_batch(items, False, 128, 128)).cuda(), ann, [None] * len(ann)) for items, (_, ann) in zip(ref, fed_a)]
    b['train_data_loader'] = recording(host, b, fed_b, loss_b)
    exb.train()
    assert a['train_iter'] == b['train_iter'] == 2 and len(loss_a) == len(loss_b) == 2
    assert loss_a[0] == loss_b[0], (loss_a, loss_b)
    assert abs(loss_a[1] - loss_b[1]) <= 3e-2 * abs(loss_b[1]), (loss_a, loss_b)
    worst = 0.0
    for (name, p), q in zip(a['model'].state_dict().items(), b['model'].state_dict().values()):
        if p.dtype.is_floating_point:
            worst = max(worst, float((p.float() - q.float()).abs().max() / p.float().abs().max().clamp(min=1e-6)))
        else:
            assert torch.equal(p, q), name
    assert worst < 2e-2, worst
