#!/usr/bin/env python
"""Micro-benchmark of the BERT-layer hot ops of this repo against their PyTorch-eager equivalents
(cuBLASLt GEMMs + ATen elementwise kernels) at the benchmark's shapes (BERT-large, batch 32 x seq 64
= 2048 tokens, hidden 1024, intermediate 4096, bf16).

Every candidate is captured (x REPS) in a CUDA graph and replayed, so the numbers are device time
per call without CPU launch overhead; timing is CUDA events around the replays after a warm-up.

    python tools/bert_ops_bench.py [--tokens 2048] [--hidden 1024] [--inter 4096] [--json out.json]
"""
import argparse
import json
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from dear_pytorch_b200.ops.fused_ln import dropout_add_layer_norm       # noqa: E402
from dear_pytorch_b200.ops.tc_gemm import fused_ffn, require_tc         # noqa: E402

REPS = 10


def graph_time(fn, iters=20):
    """us per call of fn() replayed from a CUDA graph (inf and a message if the candidate raises)."""
    try:
        return _graph_time(fn, iters)
    except Exception as exc:          # a kernel configuration that cannot run this shape: report, keep going
        print("candidate failed: %s" % str(exc).splitlines()[0][:200], flush=True)
        return float("inf")


def _graph_time(fn, iters):
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            fn()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(REPS):
            fn()
    for _ in range(3):
        g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / (iters * REPS)


def _gemm_section(r, tc, x, w1, b1, w2, b2, h, z, dy):
    """The FFN's two fusable GEMMs: library path (cuBLAS + elementwise kernels) vs the hand-written wgmma kernels
    (csrc/tc_ffn_hw.cu) with 1 / 2 / 4 CTAs per cluster sharing the B tile through TMA multicast."""
    # 1. up projection + bias + GELU (forward)
    r["up_gelu_eager"] = graph_time(lambda: F.gelu(F.linear(x, w1, b1)))
    r["up_gemm_only_cublas"] = graph_time(lambda: F.linear(x, w1, b1))
    for cl in (1, 2, 4):
        tc.set_ffn_hw_cluster(cl)
        r["up_gelu_wgmma_handwritten_cl%d" % cl] = graph_time(lambda: tc.ffn_up_hw(x, w1, b1))
    tc.set_ffn_hw_cluster(-1)
    r["up_gelu_wgmma_handwritten"] = graph_time(lambda: tc.ffn_up_hw(x, w1, b1))
    # 2. down projection (forward): plain GEMM, cuBLAS in both paths
    r["down_eager"] = graph_time(lambda: F.linear(h, w2, b2))
    # 3. dgrad of the down projection + GELU backward
    def eager_dgelu():
        dh = dy.mm(w2)
        return torch.ops.aten.gelu_backward(dh, z)
    r["dgrad_dgelu_eager"] = graph_time(eager_dgelu)
    r["dgrad_gemm_only_cublas"] = graph_time(lambda: dy.mm(w2))
    for cl in (1, 2, 4):
        tc.set_ffn_hw_cluster(cl)
        r["dgrad_dgelu_wgmma_handwritten_cl%d" % cl] = graph_time(lambda: tc.ffn_dgelu_hw_nt(dy, w2, z))
    tc.set_ffn_hw_cluster(-1)
    r["dgrad_dgelu_wgmma_handwritten"] = graph_time(lambda: tc.ffn_dgelu_hw_nt(dy, w2, z))
    w2t = w2.t().contiguous()
    r["dgrad_dgelu_wgmma_handwritten_kmajor_needs_transpose"] = graph_time(lambda: tc.ffn_dgelu_hw(dy, w2t, z))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", type=int, default=2048)
    ap.add_argument("--hidden", type=int, default=1024)
    ap.add_argument("--inter", type=int, default=4096)
    ap.add_argument("--json", default=None)
    ap.add_argument("--sections", default="gemm,ffn,ln,lg,attn",
                    help="comma list: gemm (wgmma variants vs cuBLAS), ffn (whole block), ln, lg (linear+gelu), attn")
    a = ap.parse_args()
    sections = set(a.sections.split(","))
    dev = torch.device("cuda:0")
    tc = require_tc()
    M, H, I = a.tokens, a.hidden, a.inter
    bf = torch.bfloat16
    torch.manual_seed(0)
    x = torch.randn(M, H, device=dev).to(bf)
    w1 = (torch.randn(I, H, device=dev) * H ** -0.5).to(bf)
    b1 = torch.randn(I, device=dev).to(bf)
    w2 = (torch.randn(H, I, device=dev) * I ** -0.5).to(bf)
    b2 = torch.randn(H, device=dev).to(bf)
    z = torch.randn(M, I, device=dev).to(bf)
    h = F.gelu(z)
    dy = torch.randn(M, H, device=dev).to(bf)
    gamma = torch.ones(H, device=dev, dtype=bf)
    beta = torch.zeros(H, device=dev, dtype=bf)
    flops_up = 2.0 * M * H * I
    out = {"shape": {"tokens": M, "hidden": H, "inter": I}, "us": {}}
    r = out["us"]

    if "gemm" in sections:
        _gemm_section(r, tc, x, w1, b1, w2, b2, h, z, dy)
    # 4. whole feed-forward block, forward + backward
    xs = x.clone().requires_grad_(True)
    ps = [t.clone().requires_grad_(True) for t in (w1, b1, w2, b2)]

    def ffn_eager():
        y = F.linear(F.gelu(F.linear(xs, ps[0], ps[1])), ps[2], ps[3])
        return torch.autograd.grad(y, [xs] + ps, dy)

    def ffn_fused():
        y = fused_ffn(xs, ps[0], ps[1], ps[2], ps[3])
        return torch.autograd.grad(y, [xs] + ps, dy)
    if "ffn" in sections:
        r["ffn_fwd_bwd_eager"] = graph_time(ffn_eager)
        r["ffn_fwd_bwd_wgmma_handwritten"] = graph_time(ffn_fused)

    # 5. dropout + add + LayerNorm, forward + backward
    av = x.clone().requires_grad_(True)
    rv = dy.clone().requires_grad_(True)
    gv, bv = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)

    def ln_eager():
        y = F.layer_norm(rv + F.dropout(av, 0.1, True), (H,), gv, bv, 1e-12)
        return torch.autograd.grad(y, [av, rv, gv, bv], dy)

    def ln_fused():
        y = dropout_add_layer_norm(av, rv, gv, bv, 0.1, True, 1e-12)
        return torch.autograd.grad(y, [av, rv, gv, bv], dy)
    if "ln" in sections:
        r["drop_add_ln_fwd_bwd_eager"] = graph_time(ln_eager)
        r["drop_add_ln_fwd_bwd_fused"] = graph_time(ln_fused)
        r["drop_add_ln_fwd_eager"] = graph_time(
            lambda: F.layer_norm(rv.detach() + F.dropout(av.detach(), 0.1, True), (H,), gamma, beta, 1e-12))
        r["drop_add_ln_fwd_fused"] = graph_time(
            lambda: dropout_add_layer_norm(av.detach(), rv.detach(), gamma, beta, 0.1, True, 1e-12))
        bbv = b2.clone().requires_grad_(True)

        def ln_bias_eager():       # the bias lives in the GEMM epilogue in eager mode; its gradient is a separate reduction
            y = F.layer_norm(rv + F.dropout(av + bbv, 0.1, True), (H,), gv, bv, 1e-12)
            return torch.autograd.grad(y, [av, rv, gv, bv, bbv], dy)

        def ln_bias_fused():
            y = dropout_add_layer_norm(av, rv, gv, bv, 0.1, True, 1e-12, branch_bias=bbv)
            return torch.autograd.grad(y, [av, rv, gv, bv, bbv], dy)
        r["bias_drop_add_ln_fwd_bwd_eager"] = graph_time(ln_bias_eager)
        r["bias_drop_add_ln_fwd_bwd_fused"] = graph_time(ln_bias_fused)

    # 6. bias + GELU around a bias-free GEMM, forward + backward (bias gradient included)
    from dear_pytorch_b200.ops.bias_gelu import linear_gelu
    w1g, b1g = w1.clone().requires_grad_(True), b1.clone().requires_grad_(True)
    dh = torch.randn(M, I, device=dev).to(bf)

    def lg_eager():
        return torch.autograd.grad(F.gelu(F.linear(xs, w1g, b1g)), [xs, w1g, b1g], dh)

    def lg_fused():
        return torch.autograd.grad(linear_gelu(xs, w1g, b1g), [xs, w1g, b1g], dh)
    if "lg" in sections:
        r["linear_gelu_fwd_bwd_eager"] = graph_time(lg_eager)
        r["linear_gelu_fwd_bwd_fused"] = graph_time(lg_fused)

    # 7. attention at the benchmark's shape (batch 32, 16 heads, seq 64, head dim 64), forward + backward
    from torch.nn.attention import SDPBackend, sdpa_kernel
    Bq, S, nh, hd = max(1, M // 64), 64, H // 64, 64
    qkv = torch.randn(Bq, S, 3, nh, hd, device=dev).to(bf).requires_grad_(True)
    abias = torch.zeros(Bq, 1, 1, S, device=dev, dtype=bf)
    do = torch.randn(Bq, nh, S, hd, device=dev).to(bf)

    def attn(backend, mask=True, index=False):
        def f():
            if index:
                t = qkv.permute(2, 0, 3, 1, 4)
                q, k, v = t[0], t[1], t[2]
            else:
                q, k, v = (t.transpose(1, 2) for t in qkv.unbind(2))
            if backend is None:
                o = F.scaled_dot_product_attention(q, k, v, attn_mask=abias if mask else None, dropout_p=0.1)
            else:
                with sdpa_kernel(backend):
                    o = F.scaled_dot_product_attention(q, k, v, attn_mask=abias if mask else None, dropout_p=0.1)
            return torch.autograd.grad(o, qkv, do)
        return f
    if "attn" in sections:
        r["attn_fwd_bwd_default_indexing"] = graph_time(attn(None, index=True))
        r["attn_fwd_bwd_default_unbind"] = graph_time(attn(None))
        r["attn_fwd_bwd_cudnn"] = graph_time(attn(SDPBackend.CUDNN_ATTENTION))
        r["attn_fwd_bwd_efficient"] = graph_time(attn(SDPBackend.EFFICIENT_ATTENTION))
        r["attn_fwd_bwd_flash_nomask"] = graph_time(attn(SDPBackend.FLASH_ATTENTION, mask=False))
        r["attn_fwd_bwd_math"] = graph_time(attn(SDPBackend.MATH))

    for k in list(r):
        r[k] = round(r[k], 2)
    if "gemm" in sections:
        out["tflops"] = {"up_gelu_wgmma_handwritten": round(flops_up / r["up_gelu_wgmma_handwritten"] / 1e6, 1),
                         "up_gemm_only_cublas": round(flops_up / r["up_gemm_only_cublas"] / 1e6, 1),
                         "dgrad_dgelu_wgmma_handwritten": round(flops_up / r["dgrad_dgelu_wgmma_handwritten"] / 1e6, 1),
                         "dgrad_gemm_only_cublas": round(flops_up / r["dgrad_gemm_only_cublas"] / 1e6, 1)}
    print(json.dumps(out, indent=1))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
