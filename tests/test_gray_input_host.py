# -*- coding: utf-8 -*-
"""Host side of the gray training batches, no GPU: the gray output modes of lfd_input_batch in lfd/_native.py against the header,
and the ValueErrors of DataLoader(input_channels=...) and of Executor for a loader whose channel count is not the model's."""
import os
import re

import numpy as np
import pytest
import torch

from gray_models import gray_pair
from helpers import ListDataset, synth_model
from lfd import _native as nat
from lfd.data_pipeline import sampler as S
from lfd.data_pipeline import simple_normalize_pipeline
from lfd.data_pipeline.augmentation import (BGR2RGB, Compose, HorizontalFlip, Normalize, bbox_param, simple_widerface_train_pipeline,
                                            standard_normalize)
from lfd.data_pipeline.data_loader import DataLoader
from lfd.execution.executor import Executor

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'include', 'lfd_b200.h')


def test_output_mode_constants_match_the_header():
    with open(HEADER) as f:
        text = f.read()
    enum = re.search(r'enum\s*\{([^}]*LFD_INPUT_OUT_U8_NHWC[^}]*)\}', text).group(1)
    values = {k: int(v) for k, v in re.findall(r'LFD_INPUT_OUT_(\w+)\s*=\s*(\d+)', enum)}
    assert values == {'U8_NHWC': 0, 'F32_NCHW': 1, 'U8_GRAY': 2, 'F32_GRAY': 3}
    for name, v in values.items():
        assert getattr(nat, 'INPUT_OUT_' + name) == v, name


def _loader(pipeline=simple_widerface_train_pipeline, region=None, **kw):
    rng = np.random.default_rng(0)
    ds = ListDataset([{'image': rng.integers(0, 256, (60, 70, 3), dtype=np.uint8), 'bboxes': [[5, 6, 20, 22]], 'bbox_labels': [0], 'image_id': i}
                      for i in range(6)])
    return DataLoader(ds, S.RandomDatasetSampler(ds, batch_size=3), region or S.RandomBBoxCropRegionSampler(crop_size=32), pipeline, **kw)


def test_input_channels_defaults_to_three():
    assert _loader().input_channels == 3
    gray = _loader(input_channels=1, model_normalizes=True)
    assert gray.input_channels == 1 and gray.on_device
    assert gray.input_transform.swap_rb is False and len(set(gray.input_transform.mean)) == 1


@pytest.mark.parametrize('channels', [0, 2, 4, '1'])
def test_input_channels_other_than_1_or_3_is_refused(channels):
    with pytest.raises(ValueError, match='input_channels'):
        _loader(input_channels=channels)


@pytest.mark.parametrize('pipeline', [Compose([HorizontalFlip(p=0.5), BGR2RGB(), Normalize(mean=(0.5,) * 3, std=(0.5,) * 3)], bbox_params=bbox_param),
                                      Compose([standard_normalize], bbox_params=bbox_param)], ids=['BGR2RGB', 'unequal-constants'])
@pytest.mark.parametrize('model_normalizes', [False, True])
def test_gray_loader_refuses_what_one_channel_cannot_mean(pipeline, model_normalizes):
    _loader(pipeline, model_normalizes=model_normalizes)          # fine for BGR batches
    with pytest.raises(ValueError, match='gray'):
        _loader(pipeline, input_channels=1, model_normalizes=model_normalizes)


def test_gray_loader_takes_one_constant():
    loader = _loader(Compose([HorizontalFlip(p=0.5), Normalize(mean=(0.4,), std=(0.3,))], bbox_params=bbox_param), input_channels=1)
    assert loader.on_device and loader.input_transform is None


class _Region(object):
    """A region sampler without draw(): only the host path can run it."""

    def __call__(self, sample):
        return sample


@pytest.mark.parametrize('case', ['opaque-pipeline', 'host-region-sampler'])
def test_gray_loader_refuses_host_only_inputs(case):
    kw = dict(pipeline=simple_normalize_pipeline) if case == 'opaque-pipeline' else dict(region=_Region())
    assert not _loader(**kw).on_device                               # BGR batches: the host path runs it
    with pytest.raises(ValueError, match='input_channels=1'):
        _loader(input_channels=1, **kw)


def _config(tmp_path, model, train, val=None):
    opt = torch.optim.SGD(model.parameters(), lr=0.01)
    return dict(work_dir=str(tmp_path), log_path=None, model=model, optimizer=opt, lr_scheduler=torch.optim.lr_scheduler.MultiStepLR(opt, [5]),
                training_epochs=1, gpu_list=[0], train_data_loader=train, val_data_loader=val, evaluator=None, val_interval=0, save_interval=100,
                display_interval=1, optimizer_grad_clip_cfg=dict(max_norm=10, norm_type=2), resume_path=None, weight_path=None)


class _Refusing(object):
    """A loader that fails the test if a step ever asks it for a batch."""

    def __init__(self, input_channels):
        self.input_channels, self.input_transform = input_channels, None

    def __iter__(self):
        raise AssertionError('the executor reached a step')

    def __len__(self):
        return 1


@pytest.mark.parametrize('which', ['train', 'val'])
@pytest.mark.parametrize('model_channels', [1, 3])
def test_executor_refuses_a_loader_of_other_channels(tmp_path, which, model_channels):
    model = gray_pair('WIDERFACE_XS')[0] if model_channels == 1 else synth_model('WIDERFACE_XS')[0]
    other = 4 - model_channels
    train, val = (_Refusing(other), _Refusing(model_channels)) if which == 'train' else (_Refusing(model_channels), _Refusing(other))
    ex = Executor(_config(tmp_path, model, train, val))
    with pytest.raises(ValueError, match='%d-channel batches' % other):
        ex.train()                                    # before the first step, whichever of the two loaders is wrong
    if which == 'val':
        with pytest.raises(ValueError, match='%d-channel batches' % other):
            ex.val()
