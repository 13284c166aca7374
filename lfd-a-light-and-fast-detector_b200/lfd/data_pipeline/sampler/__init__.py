# -*- coding: utf-8 -*-
from .dataset_sampler import *
from .region_sampler import *
