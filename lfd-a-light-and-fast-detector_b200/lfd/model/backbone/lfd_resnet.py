# -*- coding: utf-8 -*-
"""LFDResNet -- same constructor, attributes and state_dict keys as the reference
(lfd/model/backbone/lfd_resnet.py:218-509), but the modules here are parameter containers:
the arithmetic runs in liblfd_b200.so through the layer plan built by lfd/_engine.py.
"""
import os

import torch
import torch.nn as nn

__all__ = ['FastBlock', 'FasterBlock', 'FastestBlock', 'LFDResNet']


def make_norm(norm_cfg, channels):
    """mmdet-style dict(type='BatchNorm2d'|'GroupNorm', ...) -> module (reference: get_operator_from_cfg)."""
    cfg = dict(norm_cfg)
    kind = cfg.pop('type')
    if kind == 'BatchNorm2d':
        return nn.BatchNorm2d(num_features=channels, **cfg)
    if kind == 'GroupNorm':
        return nn.GroupNorm(num_channels=channels, **cfg)
    raise ValueError('norm type must be BatchNorm2d or GroupNorm, got %r' % (kind,))


def make_activation(activation_cfg):
    cfg = dict(activation_cfg)
    kind = cfg.pop('type')
    if kind != 'ReLU':
        raise NotImplementedError('only ReLU is fused into the H100 kernels (got %r)' % (kind,))
    return nn.ReLU(**cfg)


def init_conv_norm(module):
    """lfd_resnet.py:342-352."""
    for m in module.modules():
        if isinstance(m, nn.Conv2d):
            nn.init.kaiming_normal_(m.weight, mode='fan_out', nonlinearity='relu')
            if m.bias is not None:
                nn.init.constant_(m.bias, 0)
        elif isinstance(m, (nn.BatchNorm2d, nn.GroupNorm)):
            if m.weight is not None:
                nn.init.constant_(m.weight, 1)
            if m.bias is not None:
                nn.init.constant_(m.bias, 0)


class _Block(nn.Module):
    """Residual block container.  `LAYERS` = ((kernel, takes_block_stride, width_divisor), ...);
    the last conv is followed by the residual add and the final activation."""
    LAYERS = ()

    def __init__(self, num_input_channels, num_block_channels, stride=1, downsample=None,
                 activation_cfg=dict(type='ReLU', inplace=True), norm_cfg=None):
        super(_Block, self).__init__()
        if downsample is not None:
            assert stride == 2
        if norm_cfg is not None:
            assert norm_cfg['type'] in ['BatchNorm2d', 'GroupNorm']
        self._num_input_channel = num_input_channels
        self._num_block_channel = num_block_channels
        self._stride = stride
        self._activation_cfg = activation_cfg
        self._norm_cfg = norm_cfg
        self._downsample = downsample
        cin = num_input_channels
        for i, (k, strided, div) in enumerate(self.LAYERS, 1):
            cout = num_block_channels // div
            setattr(self, '_conv%d' % i, nn.Conv2d(cin, cout, kernel_size=k, stride=stride if strided else 1,
                                                   padding=k // 2, bias=norm_cfg is None))
            if norm_cfg is not None:
                setattr(self, '_norm%d' % i, make_norm(norm_cfg, cout))
            if i == 1:
                self._activation = make_activation(activation_cfg)
            cin = cout

    def conv_norm_pairs(self):
        return [(getattr(self, '_conv%d' % i), getattr(self, '_norm%d' % i, None)) for i in range(1, len(self.LAYERS) + 1)]

    def forward(self, x):
        raise RuntimeError('block modules are parameter containers; run the model through lfd.model.LFD')


class FastBlock(_Block):      # 3x3(s) -> 1x1 -> 3x3          (reference :21-93)
    LAYERS = ((3, True, 1), (1, False, 1), (3, False, 1))


class FasterBlock(_Block):    # 3x3(s) -> 3x3                 (reference :96-154)
    LAYERS = ((3, True, 1), (3, False, 1))


class FastestBlock(_Block):   # 3x3(s, C/2) -> 3x3            (reference :157-215)
    LAYERS = ((3, True, 2), (3, False, 1))


class LFDResNet(nn.Module):
    mode_to_body_architectures = {'fast': [4, 2, 2, 1, 1], 'faster': [2, 1, 1, 1, 1], 'fastest': [2, 1, 1, 1, 1]}
    mode_to_body_channels = {'fast': [64, 64, 128, 256, 512], 'faster': [64, 64, 128, 128, 256], 'fastest': [32, 32, 64, 64, 128]}
    # stem conv list per mode: (kernel, stride, output = stem_channels // div)
    STEMS = {'fast': ((3, 2, 1), (1, 1, 1)),
             'faster': ((3, 2, 1), (1, 1, 1), (3, 2, 1), (1, 1, 1)),
             'fastest': ((3, 2, 2), (3, 2, 1))}
    BLOCKS = {'fast': FastBlock, 'faster': FasterBlock, 'fastest': FastestBlock}

    def __init__(self, block_mode='fast', stem_mode='fast', body_mode='fast', input_channels=3, stem_channels=64,
                 body_architecture=None, body_channels=None, out_indices=((0, 3), (1, 1), (2, 1), (3, 0), (4, 0)),
                 frozen_stages=-1, activation_cfg=dict(type='ReLU', inplace=True), norm_cfg=dict(type='BatchNorm2d'),
                 init_with_weight_file=None, norm_eval=False):
        super(LFDResNet, self).__init__()
        assert block_mode in ['fast', 'faster', 'fastest']
        assert stem_mode in ['fast', 'faster', 'fastest']
        assert body_mode in ['fast', 'faster', 'fastest', None]
        if body_mode is None:
            assert body_architecture is not None and body_channels is not None
            self._body_architecture, self._body_channels = list(body_architecture), list(body_channels)
        else:
            self._body_architecture = list(self.mode_to_body_architectures[body_mode])
            self._body_channels = list(self.mode_to_body_channels[body_mode] if body_channels is None else body_channels)
        assert len(self._body_architecture) == len(self._body_channels)
        self._block_mode, self._stem_mode = block_mode, stem_mode
        self._input_channels, self._stem_channels = input_channels, stem_channels
        self._out_indices = sorted(out_indices, key=lambda x: (x[0], x[1]))
        for (s, b) in self._out_indices:
            assert 0 <= s < len(self._body_architecture) and 0 <= b < self._body_architecture[s]
        max_stage = max(s for (s, _) in self._out_indices)
        self._body_architecture = self._body_architecture[:max_stage + 1]
        self._body_channels = self._body_channels[:max_stage + 1]
        assert frozen_stages <= max_stage + 1
        self._frozen_stages = frozen_stages
        self._activation_cfg, self._norm_cfg = activation_cfg, norm_cfg
        self._init_with_weight_file, self._norm_eval = init_with_weight_file, norm_eval

        self._make_stem()
        self._make_stages()
        init_conv_norm(self)
        if init_with_weight_file is not None:
            assert isinstance(init_with_weight_file, str), 'weight file must be the string path of the file!'
            self._init_with_pretrained_weights()

        stem_stride = 2 if stem_mode == 'fast' else 4
        self._num_output_channels_list = [self._body_channels[s] for (s, _) in self._out_indices]
        self._num_output_strides_list = [stem_stride * 2 ** (s + 1) for (s, _) in self._out_indices]

    @property
    def num_output_channels_list(self):
        return self._num_output_channels_list

    @property
    def num_output_strides_list(self):
        return self._num_output_strides_list

    def _make_stem(self):
        layers, cin = [], self._input_channels
        for (k, s, div) in self.STEMS[self._stem_mode]:
            cout = self._stem_channels // div
            layers.append(nn.Conv2d(cin, cout, kernel_size=k, stride=s, padding=k // 2, bias=self._norm_cfg is None))
            if self._norm_cfg is not None:
                layers.append(make_norm(self._norm_cfg, cout))
            layers.append(make_activation(self._activation_cfg))
            cin = cout
        self._stem = nn.Sequential(*layers)

    def _make_stages(self):
        block = self.BLOCKS[self._block_mode]
        for i, num_blocks in enumerate(self._body_architecture):
            ch = self._body_channels[i]
            cin = self._stem_channels if i == 0 else self._body_channels[i - 1]
            stage = nn.ModuleList()
            for j in range(num_blocks):
                if j == 0:
                    ds = [nn.Conv2d(cin, ch, kernel_size=1, stride=2, padding=0, bias=self._norm_cfg is None)]
                    if self._norm_cfg is not None:
                        ds.append(make_norm(self._norm_cfg, ch))
                    stage.append(block(cin, ch, stride=2, downsample=nn.Sequential(*ds),
                                       activation_cfg=self._activation_cfg, norm_cfg=self._norm_cfg))
                else:
                    stage.append(block(ch, ch, stride=1, downsample=None,
                                       activation_cfg=self._activation_cfg, norm_cfg=self._norm_cfg))
            setattr(self, 'stage%d' % i, stage)

    def _init_with_pretrained_weights(self):
        """Backbone-only checkpoint load, key renaming as lfd_resnet.py:314-340."""
        assert os.path.isfile(self._init_with_weight_file), \
            'pretrained weight file [{}] does not exist!'.format(self._init_with_weight_file)
        weights = torch.load(self._init_with_weight_file, map_location='cpu')
        new_state = dict()
        for k, v in weights['state_dict'].items():
            parts = k.split('.')
            if 'backbone' in parts[0]:
                parts = parts[1:]
            new_state['.'.join(parts)] = v
        missing, unexpected = self.load_state_dict(new_state, strict=False)
        if missing:
            print('[WARNING: ResNet pretrained weights load] missing keys:\n' + '\t'.join(missing))
        if unexpected:
            print('[WARNING: ResNet pretrained weights load] unexpected keys:\n' + '\t'.join(unexpected))

    def _freeze_stages(self):
        if self._frozen_stages > 0:
            self._stem.eval()
            for p in self._stem.parameters():
                p.requires_grad = False
        for i in range(0, self._frozen_stages):
            for m in getattr(self, 'stage%d' % i):
                m.eval()
                for p in m.parameters():
                    p.requires_grad = False

    def train(self, mode=True):
        super(LFDResNet, self).train(mode)
        self._freeze_stages()
        if mode and self._norm_eval:
            for m in self.modules():
                if isinstance(m, nn.BatchNorm2d):
                    m.eval()

    # --- layer walk used by the plan builder -----------------------------------------------------
    def stem_layers(self):
        """[(conv, norm, relu)] in execution order."""
        mods, out = list(self._stem), []
        i = 0
        while i < len(mods):
            conv = mods[i]
            norm = mods[i + 1] if self._norm_cfg is not None else None
            out.append((conv, norm, True))
            i += 3 if self._norm_cfg is not None else 2
        return out

    def stages(self):
        return [getattr(self, 'stage%d' % i) for i in range(len(self._body_architecture))]

    def forward(self, x):
        raise RuntimeError('LFDResNet is a parameter container in lfd_b200; run it through lfd.model.LFD '
                           '(the whole forward is one native layer plan, there is no per-module PyTorch path)')
