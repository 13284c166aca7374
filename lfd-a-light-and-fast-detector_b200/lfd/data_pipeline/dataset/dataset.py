# -*- coding: utf-8 -*-
import os
import pickle

__all__ = ['Dataset']


class Dataset(object):
    """A packed dataset: a pickle of [meta_info, {index: Sample}], the format of the reference's packing scripts
    (lfd/data_pipeline/dataset/dataset.py).  Dataset(load_path=...) loads one; Dataset(parser, save_path) packs the samples of any
    parser object with get_meta_info() and generate_sample() and writes the pickle."""

    def __init__(self, parser=None, save_path=None, load_path=None):
        if load_path is not None:
            if not os.path.exists(load_path):
                raise FileNotFoundError('[%s] path does not exist!' % load_path)
            with open(load_path, 'rb') as f:
                self._meta_info, self._dataset = pickle.load(f)
        else:
            if save_path is None:
                raise ValueError('When parser is provided, the save_path must be set!')
            self._meta_info = parser.get_meta_info()
            self._dataset = {index: sample for index, sample in enumerate(parser.generate_sample())}
            if os.path.dirname(save_path):
                os.makedirs(os.path.dirname(save_path), exist_ok=True)
            with open(save_path, 'wb') as f:
                pickle.dump([self._meta_info, self._dataset], f, pickle.HIGHEST_PROTOCOL)

    def __getitem__(self, index):
        return self._dataset[index]

    def __len__(self):
        return len(self._dataset)

    def get_indexes(self):
        return list(self._dataset.keys())

    @property
    def meta_info(self):
        return self._meta_info
