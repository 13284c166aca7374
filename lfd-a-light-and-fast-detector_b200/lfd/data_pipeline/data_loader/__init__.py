# -*- coding: utf-8 -*-
from .data_loader import DataLoader, RankLocalBatch
