# -*- coding: utf-8 -*-
"""FocalLoss -- API of lfd/model/losses/focal_loss.py:12-92; the element-wise forward / backward run in
liblfd_b200.so (lfd_sigmoid_focal_loss_{forward,backward}), the sm_90a replacement of the reference's
sigmoid_focal_loss_ext (which needs THC and no longer builds).  CUDA only, like the reference."""
import torch
import torch.nn as nn
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from ... import _native as nat
from .utils import weight_reduce_loss

__all__ = ['FocalLoss']


class SigmoidFocalLossFunction(Function):

    @staticmethod
    def forward(ctx, input, target, gamma=2.0, alpha=0.25):
        if not input.is_cuda:
            raise RuntimeError('sigmoid focal loss is CUDA only (no CPU fallback)')
        x = input.detach().float().contiguous()
        t = target.detach().to(torch.int64).contiguous()
        ctx.save_for_backward(x, t)
        ctx.gamma, ctx.alpha = float(gamma), float(alpha)
        loss = torch.empty_like(x)
        with torch.cuda.device(x.device):
            nat.check(nat.lib().lfd_sigmoid_focal_loss_forward(nat.ptr(x), nat.ptr(t), x.shape[0], x.shape[1], ctx.gamma, ctx.alpha,
                                                               nat.ptr(loss), nat.stream_ptr()))
        return loss

    @staticmethod
    @once_differentiable
    def backward(ctx, d_loss):
        x, t = ctx.saved_tensors
        d_loss = d_loss.float().contiguous()
        d_input = torch.empty_like(x)
        with torch.cuda.device(x.device):
            nat.check(nat.lib().lfd_sigmoid_focal_loss_backward(nat.ptr(x), nat.ptr(t), nat.ptr(d_loss), x.shape[0], x.shape[1],
                                                                ctx.gamma, ctx.alpha, nat.ptr(d_input), nat.stream_ptr()))
        return d_input, None, None, None


def sigmoid_focal_loss(pred, target, weight=None, gamma=2.0, alpha=0.25, reduction='mean', avg_factor=None):
    loss = SigmoidFocalLossFunction.apply(pred, target, gamma, alpha)
    if weight is not None:
        weight = weight.view(-1, 1)
    return weight_reduce_loss(loss, weight, reduction, avg_factor)


class FocalLoss(nn.Module):

    def __init__(self, use_sigmoid=True, gamma=2.0, alpha=0.25, reduction='mean', loss_weight=1.0):
        super(FocalLoss, self).__init__()
        assert use_sigmoid is True, 'Only sigmoid focal loss supported now.'
        self.use_sigmoid, self.gamma, self.alpha = use_sigmoid, gamma, alpha
        self.reduction, self.loss_weight = reduction, loss_weight

    def forward(self, pred, target, weight=None, avg_factor=None, reduction_override=None):
        assert reduction_override in (None, 'none', 'mean', 'sum')
        reduction = reduction_override if reduction_override else self.reduction
        return self.loss_weight * sigmoid_focal_loss(pred, target, weight, gamma=self.gamma, alpha=self.alpha,
                                                     reduction=reduction, avg_factor=avg_factor)
