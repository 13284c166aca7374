# -*- coding: utf-8 -*-
"""The reference's training input pipeline under its module paths: packed datasets (dataset.Dataset), batch index samplers and
region samplers (sampler), declarative augmentation pipelines (augmentation) and the DataLoader, whose resize / crop / flip /
normalisation runs in one CUDA kernel per batch (lfd_input_batch).  Dataset parsers and packing scripts are not included: files
packed by the reference load as they are."""
from .dataset import Sample, Dataset
from .augmentation import *
from .sampler import *
from .data_loader import DataLoader, RankLocalBatch
