# -*- coding: utf-8 -*-
"""Executor -- the train / val loop of the reference (lfd/execution/executor.py:13-259) with the same `config_dict`
contract and hook bus, re-hosted on one process per GPU: the model is placed on this rank's device (no DataParallel
wrap), each rank runs its shard of every batch through the native forward, the loss is the native `get_loss`, and
gradients are combined by `parallel.allreduce_gradients` (one flat NCCL bucket) before clipping and the optimizer step.
"""
import logging
import os
from collections import OrderedDict

import torch

from .hooks import CheckpointHook, EvaluationHook, LoggerHook, LrSchedulerHook, OptimizerHook, SpeedHook, get_priority
from .parallel import broadcast_module_state, shard_batch, world
from ..data_pipeline.data_loader import RankLocalBatch
from .utils import AverageMeter, get_root_logger, load_checkpoint, save_checkpoint

_RESUME_BLACKLIST = ('timestamp', 'work_dir', 'log_path', 'training_epochs', 'gpu_list', 'display_interval', 'save_interval',
                     'val_interval', 'weight_path', 'resume_path', 'batch_size', 'num_train_workers', 'num_val_workers',
                     'train_dataset_path', 'optimizer_grad_clip_cfg')


class Executor(object):

    def __init__(self, config_dict):
        self.config_dict = cfg = config_dict
        if not os.path.exists(cfg['work_dir']):
            os.makedirs(cfg['work_dir'], exist_ok=True)
        cfg['logger'] = get_root_logger(cfg.get('log_path'), log_level=logging.INFO)
        cfg.update(epoch=0, train_iter=0, inner_train_iter=0, inner_val_iter=0,
                   train_average_meter=AverageMeter(), val_average_meter=AverageMeter())
        if cfg.get('resume_path') is not None:
            self.resume_weight()
        elif cfg.get('weight_path') is not None:
            self.load()
        rank, _ = world()
        gpu_list = cfg.get('gpu_list') or [0]
        self.device = torch.device('cuda', gpu_list[rank % len(gpu_list)]) if torch.cuda.is_available() else torch.device('cpu')
        cfg['model'] = cfg['model'].to(self.device)
        # every replica starts from rank 0's parameters AND buffers (freshly initialised, loaded or resumed): with seed=None or
        # diverged RNG state the ranks would otherwise train different models (the reference's DataParallel re-broadcasts
        # module 0 every iteration, executor.py:39)
        broadcast_module_state(cfg['model'])
        # the reference's torch.optim.SGD + clip_grad_norm_ (optimizer_hook.py:21-36) run as the fused native optimizer over
        # the model's flat parameter buffer; param_groups stay shared with the original optimizer (lr schedulers keep working)
        if self.device.type == 'cuda' and type(cfg.get('optimizer')) is torch.optim.SGD and hasattr(cfg['model'], 'train_plan_for'):
            from .optim import FusedSGD
            cfg['optimizer'] = FusedSGD.from_torch(cfg['optimizer'], cfg['model'])
        if cfg.get('resume_path') is not None:
            self.resume_optimizer()
            self.resume_lr_scheduler()
        self._hooks = []
        self._register_all_hooks()

    # ------------------------------------------------------------------ hooks
    def _register_hook(self, hook, priority='NORMAL'):
        hook.priority = get_priority(priority)
        for i in range(len(self._hooks) - 1, -1, -1):
            if hook.priority >= self._hooks[i].priority:
                self._hooks.insert(i + 1, hook)
                return
        self._hooks.insert(0, hook)

    def _register_all_hooks(self):
        """Same hooks, priorities and registration order as the reference (executor.py:67-99): equal priorities run in
        registration order, i.e. lr scheduler -> optimizer -> evaluation, then speed, logger, checkpoint."""
        cfg = self.config_dict
        self._register_hook(CheckpointHook(), 'LOWEST')
        self._register_hook(LoggerHook(), 'VERY_LOW')
        self._register_hook(LrSchedulerHook(**cfg['warmup_setting']) if 'warmup_setting' in cfg else LrSchedulerHook(), 'NORMAL')
        self._register_hook(OptimizerHook(cfg.get('optimizer_grad_clip_cfg'), cfg['training_epochs']), 'NORMAL')
        self._register_hook(SpeedHook(), 'LOW')
        self._register_hook(EvaluationHook(), 'NORMAL')

    def _call_hooks(self, fn_name):
        for hook in self._hooks:
            getattr(hook, fn_name)(self)

    # ------------------------------------------------------------------ checkpoints
    def _generate_meta(self):
        types = [str, int, float, list, dict, bool, type(None), OrderedDict]
        return {k: v for k, v in self.config_dict.items() if type(v) in types}

    def save(self):
        """Rank 0 writes the checkpoint.  BatchNorm running statistics are per replica (no SyncBN, like the reference's
        DataParallel, where only replica 0's buffers persist): rank 0's are the ones saved."""
        cfg = self.config_dict
        save_checkpoint(cfg['model'], os.path.join(cfg['work_dir'], 'epoch_' + str(cfg['epoch']) + '.pth'),
                        optimizer=cfg['optimizer'], lr_scheduler=cfg['lr_scheduler'], meta=self._generate_meta())

    def load(self):
        cfg = self.config_dict
        cfg['logger'].info('Load weights from checkpoint:{}'.format(cfg['weight_path']))
        load_checkpoint(cfg['model'], load_path=cfg['weight_path'], strict=True, logger=cfg['logger'])

    def resume_weight(self):
        cfg = self.config_dict
        cfg['logger'].info('Resume training from checkpoint:{}'.format(cfg['resume_path']))
        checkpoint = load_checkpoint(cfg['model'], load_path=cfg['resume_path'], strict=True, logger=cfg['logger'])
        cfg['checkpoint'] = checkpoint
        for k in _RESUME_BLACKLIST:
            checkpoint['meta'].pop(k, None)
        cfg.update(checkpoint['meta'])

    def resume_optimizer(self):
        if 'optimizer_state_dict' in self.config_dict['checkpoint']:
            self.config_dict['optimizer'].load_state_dict(self.config_dict['checkpoint']['optimizer_state_dict'])

    def resume_lr_scheduler(self):
        if 'lr_scheduler_state_dict' in self.config_dict['checkpoint']:
            self.config_dict['lr_scheduler'].load_state_dict(self.config_dict['checkpoint']['lr_scheduler_state_dict'])

    def get_current_lr(self):
        return self.config_dict['optimizer'].param_groups[0]['lr']

    # ------------------------------------------------------------------ loops
    def _to_device(self, image_batch):
        t = torch.from_numpy(image_batch) if not torch.is_tensor(image_batch) else image_batch
        return t.to(self.device, non_blocking=True)

    @staticmethod
    def _local(data_batch):
        """This rank's share of a batch: a RankLocalBatch already is one (the loader built only this rank's images)."""
        return tuple(data_batch) if isinstance(data_batch, RankLocalBatch) else shard_batch(data_batch)

    def _check_input_channels(self, loader):
        """A DataLoader's batches have its input_channels (3: BGR, 1: gray); the model must read that many (ValueError otherwise)."""
        model = self.config_dict['model']
        channels = getattr(loader, 'input_channels', None)
        if channels is None or not hasattr(model, '_backbone'):
            return
        from .._engine import image_channels
        if channels != image_channels(model):
            raise ValueError('the data loader makes %d-channel batches (input_channels=%d) but the model reads %d-channel images'
                             % (channels, channels, image_channels(model)))

    def _set_input_transform(self, loader):
        """A loader that leaves channel order and normalisation to the model (DataLoader(model_normalizes=True)) says which: its uint8
        batches mean nothing without it.  A DataLoader without the argument resets the model to the default its uint8 batches assume.
        Its channel count must be the model's (ValueError before the first step)."""
        self._check_input_channels(loader)
        if hasattr(loader, 'input_transform') and hasattr(self.config_dict['model'], 'set_input_transform'):
            self.config_dict['model'].set_input_transform(loader.input_transform)

    def train(self):
        cfg = self.config_dict
        cfg['mode'] = 'train'
        cfg['model'].train()
        self._check_input_channels(cfg.get('val_data_loader'))     # the val loader too, so a mismatch stops the run before it trains
        self._set_input_transform(cfg['train_data_loader'])
        self._call_hooks('before_train_epoch')
        for i, data_batch in enumerate(cfg['train_data_loader']):
            cfg.update(inner_train_iter=i)
            self._call_hooks('before_train_iter')
            image_batch, annotation_batch, meta_batch = self._local(data_batch)
            cfg.update(batch_size=len(annotation_batch))
            if len(annotation_batch) == 0:
                # the last batch had fewer images than ranks: this rank has nothing to compute but must still take part in the
                # collectives of the step (positive counters, loss values, gradients), with zeros
                loss_dict = cfg['model'].empty_shard_loss()
            else:
                predict_outputs = cfg['model'](self._to_device(image_batch))
                loss_dict = cfg['model'].get_loss(predict_outputs, annotation_batch, meta_batch)
            cfg.update(loss=loss_dict['loss'])
            cfg['train_average_meter'].update_all(loss_dict['loss_values'], cfg['batch_size'])     # read when the logger asks
            cfg['train_iter'] += 1
            self._call_hooks('after_train_iter')
        cfg['epoch'] += 1
        self._call_hooks('after_train_epoch')

    def val(self):
        cfg = self.config_dict
        cfg['mode'] = 'val'
        cfg['model'].eval()
        self._set_input_transform(cfg['val_data_loader'])
        self._call_hooks('before_val_epoch')
        for i, data_batch in enumerate(cfg['val_data_loader']):
            cfg.update(inner_val_iter=i)
            self._call_hooks('before_val_iter')
            image_batch, annotation_batch, meta_batch = self._local(data_batch)
            cfg.update(batch_size=len(annotation_batch))
            with torch.no_grad():
                predict_outputs = cfg['model'](self._to_device(image_batch))
                loss_dict = cfg['model'].get_loss(predict_outputs, annotation_batch, meta_batch)
                predict_results = cfg['model'].get_results(predict_outputs, meta_batch)
            cfg['val_average_meter'].update_all(loss_dict['loss_values'], cfg['batch_size'])
            cfg.update(eval_results=(predict_results, meta_batch))
            self._call_hooks('after_val_iter')
        self._call_hooks('after_val_epoch')

    def run(self):
        cfg = self.config_dict
        self._call_hooks('before_run')
        while cfg['epoch'] < cfg['training_epochs']:
            self.train()
            if cfg.get('evaluator') is not None and cfg.get('val_interval', 0) > 0 and cfg['epoch'] % cfg['val_interval'] == 0:
                self.val()
        self._call_hooks('after_run')
