"""Fused bias + GELU around a bias-free GEMM (csrc/ln_fused.cu: bias_gelu_*).

``linear_gelu(x, w, b)`` = ``gelu(F.linear(x, w, b))`` computed as a bias-free GEMM followed by ONE
elementwise kernel ``gelu(z + b)``; its backward is ONE kernel that produces ``dz = dh * gelu'(z + b)``
and the bias gradient (column sums of ``dz``) in the same pass.  PyTorch eager — what the reference's
BERT runs (transformers' BertIntermediate, dear/bert_benchmark.py:60-75) — needs GELU-backward plus a
separate [tokens, 4*hidden] -> [4*hidden] reduction for the bias gradient.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from . import native


class _BiasGelu(torch.autograd.Function):
    @staticmethod
    def forward(ctx, z, bias):
        ctx.save_for_backward(z, bias)
        return native().bias_gelu_forward(z, bias)

    @staticmethod
    def backward(ctx, dh):
        z, bias = ctx.saved_tensors
        if not dh.is_contiguous() or dh.data_ptr() % 16:
            dh = dh.clone(memory_format=torch.contiguous_format)
        dz, dbias = native().bias_gelu_backward(dh, z, bias)
        return dz, (dbias if ctx.needs_input_grad[1] else None)


def bias_gelu(z: torch.Tensor, bias: torch.Tensor) -> torch.Tensor:
    """``gelu(z + bias)`` (erf form) with the bias gradient fused into the backward."""
    C = native()
    if (C is not None and z.is_cuda and hasattr(C, "bias_gelu_supported") and C.bias_gelu_supported(z, bias)
            and bias.dtype == z.dtype and bias.is_contiguous()):
        return _BiasGelu.apply(z, bias)
    return F.gelu(z + bias)


def linear_gelu(x: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor) -> torch.Tensor:
    """``gelu(F.linear(x, weight, bias))``."""
    if bias is None:
        return F.gelu(F.linear(x, weight))
    return bias_gelu(F.linear(x, weight), bias)
