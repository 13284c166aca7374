# -*- coding: utf-8 -*-
"""TrafficLight LFD-S (TrafficLight_train/TL_LFD_S.py:78-150 of the reference): the shipped config whose stem and stage 0 are 48
channels wide.  It runs for inference only, so it is kept out of oracle.CONFIGS, which lists the trainable configs; the tests of the
48-channel path build it from here."""
from oracle import lfd_oracle as orc

# stem 'fast' 48, body [4, 2, 1, 1, 1] x [48, 64, 64, 128, 128], taps ((0, 3), (1, 1), (2, 0), (3, 0), (4, 0)), one class,
# detection_scales, QualityFocalLoss (a sigmoid head), merged shared head without norm layers, 'dist' assignment
TL_S = orc._cfg('fast', 48, [4, 2, 1, 1, 1], [48, 64, 64, 128, 128], ((0, 3), (1, 1), (2, 0), (3, 0), (4, 0)), 1,
                ((0, 16), (16, 32), (32, 64), (64, 128), (128, 256)), 'QualityFocalLoss', True, 'dist', head_norm=False)
FORWARD_CASE = (2, 168, 232, -1.0)       # N, H, W, cls_bias of tests/golden/forward_TL_S.pt


def build_model(cfg=TL_S):
    """The product's LFD with the classes and arguments of TL_LFD_S.py (helpers.build_model maps every loss except FocalLoss to
    CrossEntropyLoss, which would give the head a background column).  cfg: TL_S, or the same network at other widths."""
    from lfd.model.backbone import LFDResNet
    from lfd.model.neck import SimpleNeck
    from lfd.model.head import LFDHead
    from lfd.model.losses import QualityFocalLoss, IoULoss
    from lfd.model import LFD
    bb, hd, lc = cfg['backbone'], cfg['head'], cfg['lfd']
    cls_loss = QualityFocalLoss(use_sigmoid=True, beta=2.0, reduction='mean', loss_weight=2.0)
    reg_loss = IoULoss(eps=1e-6, reduction='mean', loss_weight=1.0)
    backbone = LFDResNet(block_mode=bb['block_mode'], stem_mode=bb['stem_mode'], body_mode=None, input_channels=3,
                         stem_channels=bb['stem_channels'], body_architecture=bb['body_architecture'], body_channels=bb['body_channels'],
                         out_indices=bb['out_indices'], frozen_stages=-1, activation_cfg=dict(type='ReLU', inplace=True),
                         norm_cfg=dict(type='BatchNorm2d'), init_with_weight_file=None, norm_eval=False)
    neck = SimpleNeck(num_neck_channels=128, num_input_channels_list=backbone.num_output_channels_list,
                      num_input_strides_list=backbone.num_output_strides_list, norm_cfg=dict(type='BatchNorm2d'),
                      activation_cfg=dict(type='ReLU', inplace=True))
    head = LFDHead(num_classes=hd['num_classes'], num_heads=len(neck.num_output_strides_list), num_input_channels=128,
                   num_head_channels=128, num_conv_layers=2, activation_cfg=dict(type='ReLU', inplace=True), norm_cfg=None,
                   share_head_flag=True, merge_path_flag=True, classification_loss_type=type(cls_loss).__name__,
                   regression_loss_type=type(reg_loss).__name__)
    return LFD(backbone=backbone, neck=neck, head=head, num_classes=lc['num_classes'], regression_ranges=lc['regression_ranges'],
               gray_range_factors=lc['gray_range_factors'], range_assign_mode=lc['range_assign_mode'],
               point_strides=neck.num_output_strides_list, classification_loss_func=cls_loss, regression_loss_func=reg_loss,
               distance_to_bbox_mode=lc['distance_to_bbox_mode'])


def synth_model(cls_bias=-1.0, seed=666):
    import synth
    model = build_model()
    sd = synth.synth_state_dict(model.state_dict(), seed=seed, cls_bias=cls_bias)
    model.load_state_dict(sd, strict=True)
    model.eval()
    return model, sd
