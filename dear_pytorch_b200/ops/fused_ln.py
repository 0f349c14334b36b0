"""Fused dropout + residual add + LayerNorm (csrc/ln_fused.cu).

``dropout_add_layer_norm(a, residual, weight, bias, p, training, eps)`` computes
``layer_norm(residual + dropout(a, p))`` — the tail of both halves of a post-LN transformer layer
(the reference's BERT: transformers' BertSelfOutput / BertOutput, dear/bert_benchmark.py:60-75) —
in one kernel forward and one (+ a tiny column reduction) backward instead of three and four-five
ATen kernels.  ``FusedDropoutAddLayerNorm`` is a drop-in ``nn.LayerNorm`` (same parameters and
state-dict keys) with a ``forward(a, residual)``.

The kernels cover 16-byte aligned CUDA tensors in fp32 / bf16 with a hidden size up to 1024 that is a
multiple of one 128-bit vector; anything else takes the PyTorch composite, which is also the numerics reference.
"""
from __future__ import annotations

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import native


class _DropAddLN(torch.autograd.Function):
    @staticmethod
    def forward(ctx, a, residual, weight, bias, p, training, eps, branch_bias):
        y, s, mean, rstd, mask = native().ln_forward(a, residual, weight, bias, p, training, eps, branch_bias)
        ctx.save_for_backward(s, mean, rstd, weight, mask)
        ctx.p = p
        ctx.has_branch_bias = branch_bias is not None
        return y

    @staticmethod
    def backward(ctx, dy):
        s, mean, rstd, weight, mask = ctx.saved_tensors
        if not dy.is_contiguous() or dy.data_ptr() % 16:
            dy = dy.clone(memory_format=torch.contiguous_format)
        want_dbias = ctx.has_branch_bias and ctx.needs_input_grad[7]
        d_res, d_a, dgamma, dbeta, dbias = native().ln_backward(dy, s, mean, rstd, weight, mask, ctx.p, want_dbias)
        return (d_a if ctx.needs_input_grad[0] else None, d_res if ctx.needs_input_grad[1] else None,
                dgamma if ctx.needs_input_grad[2] else None, dbeta if ctx.needs_input_grad[3] else None,
                None, None, None, dbias if want_dbias else None)


def _composite(a, residual, weight, bias, p, training, eps, branch_bias=None):
    if branch_bias is not None:
        a = a + branch_bias
    return F.layer_norm(residual + F.dropout(a, p, training), (a.shape[-1],), weight, bias, eps)


def fused_ln_applicable(a: torch.Tensor, residual: torch.Tensor, weight, bias, branch_bias=None) -> bool:
    C = native()
    return (C is not None and a.is_cuda and weight is not None and bias is not None and hasattr(C, "ln_supported")
            and C.ln_supported(a, residual, weight, bias, branch_bias) and a.shape == residual.shape and a.dtype == residual.dtype == weight.dtype == bias.dtype
            and a.is_contiguous() and residual.is_contiguous())


def dropout_add_layer_norm(a, residual, weight, bias, p: float = 0.0, training: bool = False, eps: float = 1e-5,
                           branch_bias=None):
    """``layer_norm(residual + dropout(a [+ branch_bias], p))`` over the last dimension.

    ``branch_bias`` is the bias of the linear layer that produced ``a`` when its GEMM ran bias-free
    (``a = F.linear(x, W)``): the kernel adds it on the fly and its gradient — the column sums of
    ``d a`` — falls out of the backward kernel, which already reduces over rows for the LayerNorm
    parameters, instead of costing a separate reduction kernel."""
    if a.is_cuda and not a.is_contiguous():
        a = a.contiguous()
    if residual.is_cuda and not residual.is_contiguous():
        residual = residual.contiguous()
    if fused_ln_applicable(a, residual, weight, bias, branch_bias) and (
            branch_bias is None or (branch_bias.dtype == a.dtype and branch_bias.is_contiguous())):
        return _DropAddLN.apply(a, residual, weight, bias, float(p), bool(training), float(eps), branch_bias)
    return _composite(a, residual, weight, bias, p, training, eps, branch_bias)


class FusedDropoutAddLayerNorm(nn.LayerNorm):
    """``nn.LayerNorm(hidden)`` whose forward takes the branch output and the residual stream."""

    def __init__(self, hidden: int, eps: float = 1e-5, p: float = 0.0, device=None, dtype=None):
        super().__init__(hidden, eps=eps, elementwise_affine=True, device=device, dtype=dtype)
        self.p = float(p)

    def forward(self, a: torch.Tensor, residual: torch.Tensor, branch_bias=None) -> torch.Tensor:   # type: ignore[override]
        return dropout_add_layer_norm(a, residual, self.weight, self.bias, self.p, self.training, self.eps, branch_bias)

    def extra_repr(self) -> str:
        return super().extra_repr() + ", p=%g" % self.p
