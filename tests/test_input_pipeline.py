# -*- coding: utf-8 -*-
"""Host side of the training input pipeline (lfd.data_pipeline), no GPU: region-sampler draws, dataset samplers and cropped pixels
against the reference's (tests/golden/input_samplers.pt, tests/gen_golden_input.py), the numpy oracle of the input kernel against
cv2.resize, packed-dataset pickles, per-rank sharding of the draws, and the host fallback for pipelines the kernel cannot run."""
import copy
import os
import pickle
import random

import numpy as np
import pytest
import torch

import input_oracle as O
from gen_golden_input import digest, synthetic_samples
from lfd.data_pipeline import Dataset, Sample, simple_normalize_pipeline
from lfd.data_pipeline import sampler as S
from lfd.data_pipeline.augmentation import Compose, HorizontalFlip, bbox_param, pipeline_device_spec, simple_normalize, simple_widerface_train_pipeline
from lfd.data_pipeline.data_loader import DataLoader, RankLocalBatch
from lfd.data_pipeline.data_loader.data_loader import _encoded_size, source_window
from lfd.data_pipeline.sampler.region_sampler import apply_draw
from lfd.execution.executor import Executor

GOLDEN = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'input_samplers.pt'), weights_only=False)
SAMPLES = synthetic_samples()     # the goldens keep digests of the images, not the images


def test_regenerated_samples_are_the_golden_ones():
    assert [digest(s['image']) for s in SAMPLES] == GOLDEN['source_digests']
    assert [{k: v for k, v in s.items() if k != 'image'} for s in SAMPLES] == GOLDEN['samples']


class ListDataset(object):
    def __init__(self, samples):
        self.samples = dict(enumerate(samples))

    def __len__(self):
        return len(self.samples)

    def __getitem__(self, i):
        return self.samples[i]

    def get_indexes(self):
        return list(self.samples.keys())


@pytest.mark.parametrize('k', range(len(GOLDEN['region'])))
def test_region_draws_and_pixels_match_reference(k):
    g = GOLDEN['region'][k]
    sampler = getattr(S, g['cls'])(**g['kwargs'])
    # draw() + the oracle's pixels
    random.seed(g['seed'])
    for i, (s, ref) in enumerate(zip(SAMPLES, g['results'])):
        tmp = {key: v for key, v in copy.deepcopy(s).items() if key != 'image'}
        d = sampler.draw(tmp, image_shape=s['image'].shape[:2])
        apply_draw(tmp, d)
        assert set(tmp) == set(ref) - {'image'}
        for key in tmp:
            assert tmp[key] == ref[key], key
        if g['cls'] == 'IdleRegionSampler':
            continue
        img = O.render(s['image'], d.scale, d.crop[0], d.crop[1], d.crop[3], d.crop[2], False)
        assert digest(img if len(ref['image'][0]) == 3 else img[:, :, 0]) == ref['image'], i      # a gray crop stays 2-D in the reference
    # __call__: the reference's host contract (cv2)
    pytest.importorskip('cv2')
    random.seed(g['seed'])
    for i, (s, ref) in enumerate(zip(SAMPLES, g['results'])):
        out = sampler(copy.deepcopy(s))
        assert set(out) == set(ref) and digest(out['image']) == ref['image'], i
        assert all(out[key] == ref[key] for key in out if key != 'image')


def test_region_goldens_cover_area_copy_gray_and_edges():
    scales = {round(r['resize_scale'], 6) for g in GOLDEN['region'] for r in g['results'] if 'resize_scale' in r}
    assert any(s['image'].ndim == 2 for s in SAMPLES)
    seen = set()
    for g in GOLDEN['region'][:4]:
        sampler = getattr(S, g['cls'])(**g['kwargs'])
        random.seed(g['seed'])
        for s in SAMPLES:
            d = sampler.draw(copy.deepcopy(s))
            mode, dh, dw = S.resize_plan(s['image'].shape[0], s['image'].shape[1], d.scale)
            seen.add(('mode', mode))
            cx, cy, cw, ch = d.crop
            seen.update({('left', cx < 0), ('top', cy < 0), ('right', cx + cw > dw), ('bottom', cy + ch > dh)})
    assert {('mode', 0), ('mode', 1), ('mode', 2)} <= seen, seen
    assert {('left', True), ('top', True), ('right', True), ('bottom', True)} <= seen, seen
    assert scales  # TypicalCOCO / Idle meta present


@pytest.mark.parametrize('k', range(len(GOLDEN['index_batches'])))
def test_dataset_samplers_match_reference(k):
    g = GOLDEN['index_batches'][k]
    random.seed(g['seed']), np.random.seed(g['seed'])
    sampler = getattr(S, g['cls'])(ListDataset(SAMPLES), **g['kwargs'])
    assert len(sampler) == len(g['epochs'][0])
    assert [list(sampler) for _ in range(2)] == g['epochs']


def test_oracle_matches_cv2_exactly():
    """The oracle restates cv2 4.x's fixed-point INTER_LINEAR and INTER_AREA (1/s == 2) on uint8: measured 0 differing pixels."""
    cv2 = pytest.importorskip('cv2')
    rng = np.random.default_rng(0)
    cases = [(float(rng.uniform(0.5, 1.5)), int(rng.integers(9, 300)), int(rng.integers(9, 300)), int(rng.choice([1, 3]))) for _ in range(30)]
    cases += [(0.5, 37, 51, 3), (0.5, 36, 50, 1), (0.5, 7, 5, 3), (1.0, 30, 40, 3), (2.7, 33, 47, 3), (1.0001, 11, 13, 3), (32 / 64, 71, 69, 1)]
    total = bad = 0
    for s, h, w, c in cases:
        img = rng.integers(0, 256, (h, w, c) if c == 3 else (h, w), dtype=np.uint8)
        ref = cv2.resize(img, (0, 0), fx=s, fy=s)
        ref = ref if ref.ndim == 3 else ref[:, :, None]
        _, dh, dw = O.resize_plan(h, w, s)
        got = O.resized(img, s, np.arange(dh), np.arange(dw))
        assert got.shape == ref.shape
        total += got.size
        bad += int((got != ref).sum())
    assert bad == 0, '%d of %d pixels differ' % (bad, total)


def test_source_window_holds_every_read():
    """The window the loader copies contains every source pixel the oracle reads (so the copy is all the kernel needs)."""
    rng = np.random.default_rng(1)
    for _ in range(200):
        h, w = int(rng.integers(2, 80)), int(rng.integers(2, 80))
        s = [0.5, 1.0, float(rng.uniform(0.3, 3.0))][int(rng.integers(3))]
        mode, dh, dw = O.resize_plan(h, w, s)
        crop = (int(rng.integers(-40, dw + 5)), int(rng.integers(-40, dh + 5)), int(rng.integers(1, 60)), int(rng.integers(1, 60)))
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        x, y, ww, wh = source_window(h, w, s, crop)
        masked = np.zeros_like(img)
        masked[y:y + wh, x:x + ww] = img[y:y + wh, x:x + ww]
        a = O.render(img, s, crop[0], crop[1], crop[3], crop[2], False)
        b = O.render(masked, s, crop[0], crop[1], crop[3], crop[2], False)
        assert np.array_equal(a, b)


def test_reference_pickle_loads_and_parser_packs(tmp_path):
    samples = {i: Sample(s) for i, s in enumerate(SAMPLES[:5])}
    path = os.path.join(str(tmp_path), 'packed.pkl')
    with open(path, 'wb') as f:
        pickle.dump([{'name': 'synthetic'}, samples], f, pickle.HIGHEST_PROTOCOL)
    ds = Dataset(load_path=path)
    assert len(ds) == 5 and ds.get_indexes() == list(range(5)) and ds.meta_info == {'name': 'synthetic'}
    assert np.array_equal(ds[3]['image'], samples[3]['image'])

    class Parser(object):
        def get_meta_info(self):
            return {'parser': 1}

        def generate_sample(self):
            yield from samples.values()

    out = os.path.join(str(tmp_path), 'sub', 'packed2.pkl')
    Dataset(parser=Parser(), save_path=out)
    again = Dataset(load_path=out)
    assert len(again) == 5 and again.meta_info == {'parser': 1}


def test_pipeline_specs():
    assert pipeline_device_spec(simple_widerface_train_pipeline, True)[:2] == (0.5, False)
    assert pipeline_device_spec(simple_normalize_pipeline, True) is None      # any other callable: host
    flip = Compose([HorizontalFlip(p=1.0), simple_normalize], bbox_params=bbox_param)
    out = flip({'image': np.arange(24, dtype=np.uint8).reshape(2, 4, 3), 'bboxes': [[1, 0, 2, 1]], 'bbox_labels': [0]})
    assert list(out['bboxes'][0]) == [1, 0, 2, 1] and out['image'].dtype == np.float32     # x' = W - x - w = 4 - 1 - 2


def _loader_samples():
    rng = np.random.default_rng(4)
    out = []
    for i in range(10):
        h, w = int(rng.integers(40, 90)), int(rng.integers(40, 90))
        s = {'image': rng.integers(0, 256, (h, w, 3) if i % 3 else (h, w), dtype=np.uint8), 'image_id': i}
        if i % 4:
            s['bboxes'], s['bbox_labels'] = [[int(rng.integers(0, w - 20)), int(rng.integers(0, h - 20)), 15, 18]], [i % 2]
        out.append(s)
    return out


def test_sharded_draws_are_slices_of_the_world_1_batch():
    ds = ListDataset(_loader_samples())
    region = S.RandomBBoxCropRegionSampler(crop_size=32, resize_range=(0.5, 1.5), resize_prob=0.5)
    loader = DataLoader(ds, S.RandomDatasetSampler(ds, batch_size=5), region, simple_widerface_train_pipeline)
    index_batch = [0, 3, 4, 7, 9]
    plans = []
    for rank, world in [(0, 1), (0, 2), (1, 2)]:
        random.seed(3)
        plans.append(loader.plan(index_batch, rank, world))
    full, r0, r1 = plans
    assert r0[5] == (0, 3) and r1[5] == (3, 5)
    for part, (b, e) in ((r0, (0, 3)), (r1, (3, 5))):
        assert part[3] == full[3]
        assert [(it[1], it[2]) for it in part[0]] == [(it[1], it[2]) for it in full[0][b:e]]
        assert all(np.array_equal(a[0], c[0]) and np.array_equal(a[1], c[1]) for a, c in zip(part[1], full[1][b:e]))
        assert part[2] == full[2][b:e]
    # Executor uses a rank-local batch as it is and slices a plain one
    local = RankLocalBatch((np.zeros((2, 3, 4, 4)), [1, 2], [None, None]))
    assert Executor._local(local)[1] == [1, 2]
    assert Executor._local((np.zeros((2, 3, 4, 4)), [1, 2], [None, None]))[1] == [1, 2]


def test_encoded_size_reads_headers():
    cv2 = pytest.importorskip('cv2')
    img = np.random.default_rng(0).integers(0, 256, (37, 53, 3), dtype=np.uint8)
    for ext in ('.jpg', '.png'):
        assert _encoded_size(cv2.imencode(ext, img)[1].tobytes()) == (37, 53)


def test_host_fallback_runs_the_reference_path():
    pytest.importorskip('cv2')
    ds = ListDataset(_loader_samples())
    region = S.RandomBBoxCropRegionSampler(crop_size=32, resize_range=(0.5, 1.5), resize_prob=0.5)
    random.seed(9)
    loader = DataLoader(ds, S.RandomDatasetSampler(ds, batch_size=4, shuffle=False), region, simple_normalize_pipeline, num_workers=2)
    assert not loader.on_device
    batches = list(loader)
    assert len(batches) == len(loader) == 3
    random.seed(9)
    for k, (x, ann, meta) in enumerate(batches):
        x = x.cpu().numpy()
        assert x.dtype == np.float32 and x.shape[1] == 3
        for j, i in enumerate(range(4 * k, min(4 * k + 4, 10))):
            s = ds[i]
            d = region.draw({key: v for key, v in s.items() if key != 'image'}, image_shape=s['image'].shape[:2])
            img = O.render(s['image'], d.scale, d.crop[0], d.crop[1], d.crop[3], d.crop[2], False)
            ref = ((img.astype(np.float32) - np.float32(127.5)) * np.float32(1.0 / 127.5)).transpose(2, 0, 1)
            assert np.array_equal(x[j], ref)
            assert meta[j] == {'image_id': i}
            assert ann[j][0].dtype == np.float32 and ann[j][1].dtype == np.int64
