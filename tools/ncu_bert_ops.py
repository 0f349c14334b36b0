#!/usr/bin/env python
"""Launch the BERT-layer kernels of this repo a few times at the benchmark's shapes, for an ncu capture:

    ncu --set full --clock-control none --import-source on -k regex:'ffn_hw_kernel|ln_fwd_kernel|ln_bwd_kernel|bias_gelu_bwd' \
        --launch-skip 10 --launch-count 5 -o gpurun_out/prof_bert_ops python tools/ncu_bert_ops.py

Per iteration, in order: hand-written wgmma GEMM+bias+GELU, dgrad GEMM x GELU' (MN-major weight), fused dropout+add+LN
forward, its backward, bias+GELU backward (5 kernels matching the regex above)."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dear_pytorch_b200.ops import require_native            # noqa: E402
from dear_pytorch_b200.ops.tc_gemm import require_tc        # noqa: E402


def main():
    dev = torch.device("cuda:0")
    C, tc = require_native(), require_tc()
    M, H, I = 2048, 1024, 4096
    bf = torch.bfloat16
    x = torch.randn(M, H, device=dev).to(bf)
    w1 = (torch.randn(I, H, device=dev) / 32).to(bf)
    b1 = torch.randn(I, device=dev).to(bf)
    w2 = (torch.randn(H, I, device=dev) / 64).to(bf)
    z = torch.randn(M, I, device=dev).to(bf)
    dy = torch.randn(M, H, device=dev).to(bf)
    dh = torch.randn(M, I, device=dev).to(bf)
    g, b = torch.ones(H, device=dev, dtype=bf), torch.zeros(H, device=dev, dtype=bf)
    for _ in range(3):
        tc.ffn_up_hw(x, w1, b1)
        tc.ffn_dgelu_hw_nt(dy, w2, z)
        y, s, mean, rstd, mask = C.ln_forward(x, dy, g, b, 0.1, True, 1e-12, g)
        C.ln_backward(dy, s, mean, rstd, g, mask, 0.1, True)
        C.bias_gelu_backward(dh, z, b1)
    torch.cuda.synchronize()
    print("ok")


if __name__ == "__main__":
    main()
