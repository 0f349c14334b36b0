"""Transformer feed-forward block on the hand-written wgmma GEMMs of ``csrc/tc_ffn_hw.cu`` (opt-in: ``--tc-ffn 1``).

``fused_ffn(x, w1, b1, w2, b2)`` = ``linear(gelu(linear(x, w1, b1)), w2, b2)`` with

* forward: ONE kernel for ``x W1^T + b1`` and its GELU (the epilogue writes the activation and the
  pre-activation the backward needs), then the down projection;
* backward: the dgrad GEMM of the down projection applies ``gelu'(z)`` in its epilogue, so the
  [tokens, 4*hidden] gradient is written once instead of written, re-read and rewritten.

PyTorch eager (what the reference's BERT runs: transformers' BertIntermediate/BertOutput,
dear/bert_benchmark.py:60-75) launches GEMM, GELU, GEMM forward and GEMM, GELU-backward, GEMM...
backward.  Weight/bias gradients stay on cuBLAS (plain GEMMs and column sums).

On CUDA + bf16 the extension is mandatory (``require_tc`` raises if it is not built); any other
device/dtype takes the plain PyTorch formula, which is also the numerics reference of the tests.
"""
from __future__ import annotations

import importlib
import os

import torch
import torch.nn.functional as F

_TC = None
_tc_error = None


def tc_native():
    global _TC, _tc_error
    if _TC is None and _tc_error is None:
        try:
            _TC = importlib.import_module("dear_pytorch_b200._tc")
        except Exception as exc:        # pragma: no cover - depends on the build
            _tc_error = exc
    return _TC


def require_tc():
    mod = tc_native()
    if mod is None:
        raise RuntimeError("dear_pytorch_b200._tc (wgmma GEMMs) is not built: %r -- run "
                           "`python setup.py build_ext --inplace`" % (_tc_error,))
    return mod


def tc_launches() -> int:
    mod = tc_native()
    return int(mod.launches()) if mod is not None else 0



def _eligible(x: torch.Tensor, *ws: torch.Tensor) -> bool:
    if not (x.is_cuda and x.dtype == torch.bfloat16):
        return False
    return all(w.dtype == torch.bfloat16 and w.shape[-1] % 8 == 0 and w.shape[0] % 8 == 0 for w in ws if w.dim() == 2)


class _FusedFFN(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w1, b1, w2, b2):
        tc = require_tc()
        x2 = x.reshape(-1, x.shape[-1])
        if not x2.is_contiguous():
            x2 = x2.contiguous()
        h, z = tc.ffn_up_hw(x2, w1, b1)                  # GEMM + bias + GELU; activation and pre-activation in one pass
        y = torch.addmm(b2, h, w2.t())                   # plain GEMM: cuBLAS
        ctx.save_for_backward(x2, w1, w2, h, z)
        ctx.x_shape = x.shape
        return y.view(*x.shape[:-1], w2.shape[0])

    @staticmethod
    def backward(ctx, dy):
        tc = require_tc()
        x2, w1, w2, h, z = ctx.saved_tensors
        dy2 = dy.reshape(-1, dy.shape[-1])
        if not dy2.is_contiguous():
            dy2 = dy2.contiguous()
        # (dy W2) * gelu'(z) in one kernel; W2 [hidden, inter] is read as it is stored (MN-major B operand)
        dz = tc.ffn_dgelu_hw_nt(dy2, w2, z)
        dw2 = dy2.t().mm(h) if ctx.needs_input_grad[3] else None
        db2 = dy2.sum(0) if ctx.needs_input_grad[4] else None
        dw1 = dz.t().mm(x2) if ctx.needs_input_grad[1] else None
        db1 = dz.sum(0) if ctx.needs_input_grad[2] else None
        dx = dz.mm(w1).view(ctx.x_shape) if ctx.needs_input_grad[0] else None
        return dx, dw1, db1, dw2, db2


def fused_ffn(x, w1, b1, w2, b2):
    """``linear(gelu(linear(x, w1, b1)), w2, b2)``; wgmma kernels on CUDA bf16."""
    if _eligible(x, w1, w2):
        return _FusedFFN.apply(x, w1, b1, w2, b2)
    return F.linear(F.gelu(F.linear(x, w1, b1)), w2, b2)
