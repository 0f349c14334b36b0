"""Fused BatchNorm2d (+ residual add) (+ ReLU) for channels-last activations.

``FusedBatchNormAct2d`` is a drop-in ``nn.BatchNorm2d`` (same parameters, buffers and state-dict
keys) whose forward is ``act(bn(x) [+ residual])`` in ONE pass over the activations
(csrc/bn_act.cu): 8 tensor passes per layer and iteration instead of ~13 for
``BatchNorm2d -> (+) -> ReLU`` as separate cuDNN / ATen kernels.  On inputs the kernels do not
cover (CPU, NCHW, widths that are not a power-of-two number of 128-bit vectors, views that are not
16-byte aligned, bf16 affine parameters, eval-mode backward) it falls back to the equivalent PyTorch composite, so a model
using it runs everywhere.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import native


class _BNActFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, residual, weight, bias, running_mean, running_var, momentum, eps, relu):
        C = native()
        y, mean, invstd, scale, shift = C.bn_act_forward(x, residual, weight, bias, running_mean, running_var, True,
                                                         momentum, eps, relu)
        has_res = residual is not None
        ctx.relu, ctx.has_res = relu, has_res
        ctx.save_for_backward(x, y if (has_res and relu) else None, mean, invstd, scale, shift)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, y, mean, invstd, scale, shift = ctx.saved_tensors
        dx, dz, dgamma, dbeta = native().bn_act_backward(dy, x, y, mean, invstd, scale, shift, ctx.relu, ctx.has_res)
        return (dx, dz if ctx.has_res else None,
                dgamma if ctx.needs_input_grad[2] else None, dbeta if ctx.needs_input_grad[3] else None,
                None, None, None, None, None)


def _composite(x, residual, weight, bias, running_mean, running_var, training, momentum, eps, relu):
    y = F.batch_norm(x, running_mean, running_var, weight, bias, training, momentum, eps)
    if residual is not None:
        y = y + residual
    return F.relu(y) if relu else y


def bn_act(x: torch.Tensor, weight, bias, running_mean, running_var, training: bool, momentum: float, eps: float,
           relu: bool = True, residual: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Functional form.  Uses the fused kernels when they apply, else the PyTorch composite."""
    C = native()
    ok = (C is not None and x.is_cuda and momentum is not None and C.bn_act_supported(x, residual)
          and (weight is None or weight.dtype == torch.float32) and (bias is None or bias.dtype == torch.float32)
          and (residual is None or (residual.dtype == x.dtype and residual.shape == x.shape
                                    and residual.is_contiguous(memory_format=torch.channels_last))))
    if ok and training:
        if x.numel() == x.size(1):                    # what F.batch_norm raises: one value per channel has no variance
            raise ValueError("Expected more than 1 value per channel when training, got input size {}".format(x.size()))
        return _BNActFunction.apply(x, residual, weight, bias, running_mean, running_var, float(momentum), float(eps), relu)
    if ok and not torch.is_grad_enabled() and running_mean is not None:
        return C.bn_act_forward(x, residual, weight, bias, running_mean, running_var, False, float(momentum), float(eps),
                                relu)[0]
    if x.is_cuda and x.data_ptr() % 16:
        x = x.clone()                                  # cuDNN's batch norm loads 16-byte vectors too
    return _composite(x, residual, weight, bias, running_mean, running_var, training, momentum, eps, relu)


class FusedBatchNormAct2d(nn.BatchNorm2d):
    """``nn.BatchNorm2d`` followed by an optional residual add and an optional ReLU."""

    def __init__(self, num_features, eps=1e-5, momentum=0.1, affine=True, track_running_stats=True, relu=True,
                 device=None, dtype=None):
        super().__init__(num_features, eps, momentum, affine, track_running_stats, device=device, dtype=dtype)
        self.relu = relu

    def forward(self, x: torch.Tensor, residual: Optional[torch.Tensor] = None) -> torch.Tensor:
        self._check_input_dim(x)
        training = self.training or (self.running_mean is None and self.running_var is None)
        momentum = self.momentum
        if self.training and self.track_running_stats and self.num_batches_tracked is not None:
            self.num_batches_tracked.add_(1)
            if momentum is None:                       # cumulative moving average
                momentum = 1.0 / float(self.num_batches_tracked)
        rm = self.running_mean if (not self.training or self.track_running_stats) else None
        rv = self.running_var if (not self.training or self.track_running_stats) else None
        return bn_act(x, self.weight, self.bias, rm, rv, training, momentum if momentum is not None else 0.0, self.eps,
                      relu=self.relu, residual=residual)

    def extra_repr(self):
        return super().extra_repr() + ", relu=%s" % self.relu
