# -*- coding: utf-8 -*-
from .sample import Sample, reserved_keys
from .dataset import Dataset
