# -*- coding: utf-8 -*-
"""Batch index samplers with the reference's random draws, in its order (lfd/data_pipeline/sampler/dataset_sampler.py):
one random.shuffle per epoch, then for RandomWithNegDatasetSampler one numpy.random.choice over the negatives per batch."""
import random

import numpy

__all__ = ['BaseDatasetSampler', 'RandomDatasetSampler', 'RandomWithNegDatasetSampler']


class BaseDatasetSampler(object):
    def __iter__(self):
        raise NotImplementedError

    def __len__(self):
        raise NotImplementedError

    def get_batch_size(self):
        raise NotImplementedError


def _num_batches(n, per_batch, ignore_last):
    return n // per_batch + (1 if not ignore_last and n % per_batch else 0)


class RandomDatasetSampler(BaseDatasetSampler):
    """Shuffles every index once per epoch and cuts the order into batches (the last one may be short unless ignore_last)."""

    def __init__(self, dataset, batch_size=1, shuffle=True, ignore_last=False):
        assert len(dataset) > 0
        self._indexes = dataset.get_indexes()
        self._batch_size = batch_size
        self._shuffle = shuffle
        assert batch_size <= len(self._indexes)
        self._loops = _num_batches(len(self._indexes), batch_size, ignore_last)

    def __iter__(self):
        if self._shuffle:
            random.shuffle(self._indexes)
        for i in range(self._loops):
            end = None if i == self._loops - 1 else (i + 1) * self._batch_size
            yield self._indexes[i * self._batch_size:end]

    def __len__(self):
        return self._loops

    def get_batch_size(self):
        return self._batch_size


class RandomWithNegDatasetSampler(BaseDatasetSampler):
    """Samples with 'bboxes' are positives, the others negatives.  Each batch holds batch_size - int(batch_size * neg_ratio)
    positives, in a per-epoch shuffled order, followed by int(batch_size * neg_ratio) negatives drawn with replacement."""

    def __init__(self, dataset, batch_size=1, neg_ratio=0.1, shuffle=True, ignore_last=False):
        assert len(dataset) > 0, 'dataset is empty!'
        assert batch_size <= len(dataset), 'the number of samples should larger than batch size!'
        assert 0. <= neg_ratio <= 1, 'neg ratio should be in [0,1]!'
        self._batch_size = batch_size
        indexes = dataset.get_indexes()
        self._pos_indexes = [i for i in indexes if 'bboxes' in dataset[i]]
        self._neg_indexes = [i for i in indexes if 'bboxes' not in dataset[i]]
        self._num_neg = int(batch_size * neg_ratio) if self._neg_indexes else 0
        self._num_pos = batch_size - self._num_neg
        self._loop = _num_batches(len(self._pos_indexes), self._num_pos, ignore_last)

    def __len__(self):
        return self._loop

    def get_batch_size(self):
        return self._batch_size

    def __iter__(self):
        random.shuffle(self._pos_indexes)
        for i in range(self._loop):
            end = None if i == self._loop - 1 else (i + 1) * self._num_pos
            yield self._pos_indexes[i * self._num_pos:end] + numpy.random.choice(self._neg_indexes, self._num_neg).tolist()
