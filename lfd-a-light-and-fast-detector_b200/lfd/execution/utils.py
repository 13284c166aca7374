# -*- coding: utf-8 -*-
"""Checkpoint io, logging, seeding helpers with the reference's file format and call signatures
(lfd/execution/utils.py:19-122,198-321)."""
import logging as _logging
import os
import random
import sys
import time
import traceback
from collections import OrderedDict, defaultdict

import numpy
import torch
import torch.distributed as dist

__all__ = ['load_checkpoint', 'save_checkpoint', 'get_root_logger', 'set_cudnn_backend', 'set_random_seed', 'AverageMeter',
           'customize_exception_hook']


def _rank():
    return dist.get_rank() if dist.is_available() and dist.is_initialized() else 0


def load_checkpoint(model, load_path, map_location='cpu', strict=False, logger=None):
    """Reads {'meta', 'state_dict', ['optimizer_state_dict'], ['lr_scheduler_state_dict']}; strips a 'module.' prefix."""
    if not os.path.isfile(load_path):
        raise IOError('{} is not a checkpoint file'.format(load_path))
    checkpoint = torch.load(load_path, map_location=map_location, weights_only=False)
    if not (isinstance(checkpoint, dict) and 'state_dict' in checkpoint):
        raise RuntimeError('No state_dict found in checkpoint file {}'.format(load_path))
    state_dict = checkpoint['state_dict']
    if list(state_dict.keys())[0].startswith('module.'):
        state_dict = {k[7:]: v for k, v in state_dict.items()}
    missing, unexpected = model.load_state_dict(state_dict, strict=strict)
    if hasattr(model, 'invalidate_plans'):
        model.invalidate_plans()
    if _rank() == 0:
        say = logger.info if logger is not None else print
        if missing:
            say('[state dict loading warning] missing keys: {}'.format(','.join(missing)))
        if unexpected:
            say('[state dict loading warning] unexpected keys: {}'.format(','.join(unexpected)))
    return checkpoint


def save_checkpoint(model, save_path, optimizer=None, lr_scheduler=None, meta=None):
    if meta is None:
        meta = {}
    elif not isinstance(meta, dict):
        raise TypeError('meta must be a dict or None, but got {}'.format(type(meta)))
    meta.update(time=time.asctime())
    d = os.path.dirname(save_path)
    if d and not os.path.exists(d):
        os.makedirs(d)
    net = model.module if hasattr(model, 'module') else model
    checkpoint = {'meta': meta, 'state_dict': OrderedDict((k, v.cpu()) for k, v in net.state_dict().items())}
    if optimizer is not None:
        checkpoint['optimizer_state_dict'] = optimizer.state_dict()
    if lr_scheduler is not None:
        checkpoint['lr_scheduler_state_dict'] = lr_scheduler.state_dict()
    torch.save(checkpoint, save_path)


def get_root_logger(log_path=None, log_level=_logging.INFO):
    logger = _logging.getLogger('lfd')
    if logger.handlers:
        return logger
    fmt = _logging.Formatter('%(asctime)s - %(levelname)s - %(message)s')
    handlers = [_logging.StreamHandler(sys.stdout)]
    if log_path is not None and _rank() == 0:
        handlers.append(_logging.FileHandler(log_path, 'w'))
    for h in handlers:
        h.setFormatter(fmt)
        logger.addHandler(h)
    logger.setLevel(log_level if _rank() == 0 else _logging.ERROR)
    return logger


def set_random_seed(seed, deterministic=False):
    random.seed(seed)
    numpy.random.seed(seed)
    torch.manual_seed(seed)
    if torch.cuda.is_available():
        torch.cuda.manual_seed_all(seed)


def set_cudnn_backend(benchmark=True, deterministic=False):
    """Kept for config-script compatibility; the H100 path does not go through cuDNN."""
    torch.backends.cudnn.benchmark = bool(benchmark)
    torch.backends.cudnn.deterministic = bool(deterministic)


def customize_exception_hook(log_path):
    def hook(exc_type, exc_value, exc_tb):
        text = ''.join(traceback.format_exception(exc_type, exc_value, exc_tb))
        with open(log_path, 'a') as f:
            f.write(text)
        sys.__excepthook__(exc_type, exc_value, exc_tb)
    return hook


class AverageMeter(object):
    """Running averages per name (the reference's version uses the removed numpy.float, utils.py:312-313)."""

    def __init__(self):
        self.reset()

    def reset(self):
        self._sum = defaultdict(float)
        self._count = defaultdict(float)
        self._pending = []

    def update(self, name, value, n=1):
        self._sum[name] += float(value) * n
        self._count[name] += n

    def update_all(self, values, n=1):
        """values: a mapping name -> number that may still be on its way from the device (lfd.model.lfd.LossValues): it is only read
        when an average is asked for, so that logging never stalls the training loop."""
        self._pending.append((values, n))

    def _fold(self):
        pending, self._pending = self._pending, []
        for values, n in pending:
            for name, value in values.items():
                self.update(name, value, n)

    def average(self, name):
        self._fold()
        return self._sum[name] / max(self._count[name], 1e-12)

    def averages(self):
        self._fold()
        return OrderedDict((k, self.average(k)) for k in self._sum)
