"""Hand-written wgmma GEMMs with fused epilogues (csrc/tc_ffn_hw.cu) against plain PyTorch fp32 references."""
import pytest
import torch
import torch.nn.functional as F

from dear_pytorch_b200.ops.tc_gemm import fused_ffn, require_tc, tc_launches


def test_cpu_fallback_is_the_plain_formula():
    torch.manual_seed(0)
    x = torch.randn(5, 7, 16, requires_grad=True)
    w1, b1, w2, b2 = torch.randn(32, 16), torch.randn(32), torch.randn(16, 32), torch.randn(16)
    torch.testing.assert_close(fused_ffn(x, w1, b1, w2, b2), F.linear(F.gelu(F.linear(x, w1, b1)), w2, b2))


def test_fast_gelu_math_matches_erf():
    """The epilogue's Abramowitz-Stegun normal tail (csrc/tc_ffn_hw.cu: gelu_fast / dgelu_fast) against erf, in fp32 on the host."""
    import math
    x = torch.linspace(-9.0, 9.0, 20001, dtype=torch.float64)
    ax = x.abs()
    t = 1.0 / (1.0 + 0.3275911 * 0.7071067811865476 * ax)
    poly = ((((1.061405429 * t - 1.453152027) * t + 1.421413741) * t - 0.284496736) * t + 0.254829592) * t
    e = torch.exp(-0.5 * x * x)
    q = 0.5 * poly * e
    cdf = torch.where(x < 0, q, 1.0 - q)
    ref = 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0)))
    assert (cdf - ref).abs().max().item() < 1e-7
    assert (x * cdf - x * ref).abs().max().item() < 5e-7
    dref = ref + x * torch.exp(-0.5 * x * x) / math.sqrt(2 * math.pi)
    assert ((cdf + x * 0.3989422804014327 * e) - dref).abs().max().item() < 2e-7


def _rand(shape, dev, scale=1.0):
    return (scale * torch.randn(shape, device=dev)).to(torch.bfloat16)


@pytest.mark.gpu
@pytest.mark.parametrize("M,K,N", [(128, 64, 256), (2048, 1024, 4096), (300, 72, 264), (1, 8, 8)])
def test_handwritten_ffn_up(M, K, N):
    tc = require_tc()
    dev = torch.device("cuda:0")
    torch.manual_seed(1)
    x, w, b = _rand((M, K), dev), _rand((N, K), dev, K ** -0.5), _rand((N,), dev)
    h, z = tc.ffn_up_hw(x, w, b)
    torch.cuda.synchronize()
    z_ref = x.float() @ w.float().t() + b.float()
    torch.testing.assert_close(z.float(), z_ref, rtol=1e-2, atol=1e-2)
    torch.testing.assert_close(h.float(), F.gelu(z_ref), rtol=1e-2, atol=1e-2)


@pytest.mark.gpu
@pytest.mark.parametrize("M,K,N", [(128, 64, 256), (2048, 1024, 4096), (300, 72, 264), (5, 8, 16)])
def test_handwritten_ffn_dgelu(M, K, N):
    tc = require_tc()
    dev = torch.device("cuda:0")
    torch.manual_seed(2)
    dy, w, z = _rand((M, K), dev), _rand((K, N), dev, K ** -0.5), _rand((M, N), dev)
    dz = tc.ffn_dgelu_hw(dy, w.t().contiguous(), z)         # the kernel takes the transposed weight [N, K]
    torch.cuda.synchronize()
    z32 = z.float().requires_grad_(True)
    F.gelu(z32).backward(dy.float() @ w.float())
    torch.testing.assert_close(dz.float(), z32.grad, rtol=1.5e-2, atol=1.5e-2)


@pytest.mark.gpu
@pytest.mark.parametrize("M,K,N", [(128, 64, 256), (2048, 1024, 4096), (300, 72, 264), (5, 8, 16)])
def test_handwritten_ffn_dgelu_mn_major_weight(M, K, N):
    """Same op with the weight [K, N] as nn.Linear stores it: the B operand is MN-major (TMA boxes of 64 contiguous n,
    wgmma descriptor with LBO/SBO of the MN-major canonical layout, transposed B) — no transposed copy."""
    tc = require_tc()
    dev = torch.device("cuda:0")
    torch.manual_seed(2)
    dy, w, z = _rand((M, K), dev), _rand((K, N), dev, K ** -0.5), _rand((M, N), dev)
    dz = tc.ffn_dgelu_hw_nt(dy, w, z)
    torch.cuda.synchronize()
    z32 = z.float().requires_grad_(True)
    F.gelu(z32).backward(dy.float() @ w.float())
    torch.testing.assert_close(dz.float(), z32.grad, rtol=1.5e-2, atol=1.5e-2)


@pytest.mark.gpu
@pytest.mark.parametrize("cl", [1, 2, 4])
@pytest.mark.parametrize("M,K,N", [(2048, 1024, 4096), (512, 192, 512), (1024, 64, 264)])
def test_handwritten_kernels_with_multicast_clusters(M, K, N, cl):
    """CL CTAs per cluster share the B tile: each loads 1/CL of it and multicasts (cp.async.bulk.tensor ...
    .multicast::cluster), every consumer warp releases a stage in every CTA (remote mbarrier arrive)."""
    tc = require_tc()
    dev = torch.device("cuda:0")
    torch.manual_seed(4)
    tc.set_ffn_hw_cluster(cl)
    try:
        x, w, b = _rand((M, K), dev), _rand((N, K), dev, K ** -0.5), _rand((N,), dev)
        h, z = tc.ffn_up_hw(x, w, b)
        z_ref = x.float() @ w.float().t() + b.float()
        torch.testing.assert_close(z.float(), z_ref, rtol=1e-2, atol=1e-2)
        torch.testing.assert_close(h.float(), F.gelu(z_ref), rtol=1e-2, atol=1e-2)
        dy, w2, zz = _rand((M, K), dev), _rand((K, N), dev, K ** -0.5), _rand((M, N), dev)
        dz = tc.ffn_dgelu_hw_nt(dy, w2, zz)
        torch.cuda.synchronize()
        z32 = zz.float().requires_grad_(True)
        F.gelu(z32).backward(dy.float() @ w2.float())
        torch.testing.assert_close(dz.float(), z32.grad, rtol=1.5e-2, atol=1.5e-2)
    finally:
        tc.set_ffn_hw_cluster(-1)


@pytest.mark.gpu
def test_fused_ffn_autograd_matches_eager_bf16():
    dev = torch.device("cuda:0")
    torch.manual_seed(3)
    H, I, M = 256, 1024, 520
    x = _rand((4, M // 4, H), dev).requires_grad_(True)
    w1, b1 = _rand((I, H), dev, H ** -0.5).requires_grad_(True), _rand((I,), dev, 0.1).requires_grad_(True)
    w2, b2 = _rand((H, I), dev, I ** -0.5).requires_grad_(True), _rand((H,), dev, 0.1).requires_grad_(True)
    dy = _rand((4, M // 4, H), dev)
    for _ in range(1):
        y = fused_ffn(x, w1, b1, w2, b2)
        grads = torch.autograd.grad(y, (x, w1, b1, w2, b2), dy)
        ps = [t.detach().float().requires_grad_(True) for t in (x, w1, b1, w2, b2)]
        y_ref = F.linear(F.gelu(F.linear(ps[0], ps[1], ps[2])), ps[3], ps[4])
        ref = torch.autograd.grad(y_ref, ps, dy.float())
        torch.testing.assert_close(y.float(), y_ref, rtol=2e-2, atol=2e-2)
        for g, r in zip(grads, ref):
            scale = r.abs().max().item()
            torch.testing.assert_close(g.float(), r, rtol=3e-2, atol=3e-2 * max(scale, 1.0))


@pytest.mark.gpu
def test_tc_ffn_inside_cuda_graph():
    dev = torch.device("cuda:0")
    tc = require_tc()
    x, w, b = _rand((512, 256), dev), _rand((1024, 256), dev, 1 / 16), _rand((1024,), dev)
    tc.ffn_up_hw(x, w, b)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        h, z = tc.ffn_up_hw(x, w, b)
    x.copy_(_rand((512, 256), dev))
    g.replay(); torch.cuda.synchronize()
    torch.testing.assert_close(z.float(), x.float() @ w.float().t() + b.float(), rtol=1e-2, atol=1e-2)
