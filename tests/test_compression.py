import torch

from dear_pytorch_b200.parallel.compression import compressors, SignCompressor


def test_registry_matches_reference():
    # the reference's registry (wfbp/compression.py:258-267) plus the gTop-k selectors its optimizer keys on by name
    # (wfbp/dopt.py:725) but never registers
    assert set(k for k in compressors if k) == {"none", "topk", "eftopk", "gaussian", "signum", "efsignum", "gtopk", "gtopkef"}


def test_topk_residual_bookkeeping():
    c = compressors["topk"]()
    g = torch.tensor([0.1, -5.0, 0.3, 4.0, -0.2, 0.05, 3.0, -0.01])
    t, idx, vals = c.compress(g.clone(), "w", ratio=0.375)
    assert sorted(idx.tolist()) == [1, 3, 6]
    res = c.residuals["w"]
    assert torch.equal(res[idx], torch.zeros(3))
    dense = torch.zeros_like(g)
    dense[idx] = vals
    torch.testing.assert_close(dense + res, g)                 # nothing is lost
    c.add_residuals(torch.tensor([0]), "w")                    # only the first selected value was globally kept
    kept = idx[0]
    assert res[kept] == 0 and all(res[i] == g[i] for i in idx[1:].tolist())


def test_eftopk_feeds_error_back():
    c = compressors["eftopk"]()
    g1 = torch.tensor([1.0, 0.4, 0.3, 0.2])
    c.compress(g1.clone(), "w", ratio=0.25)
    g2 = torch.tensor([0.0, 0.4, 0.0, 0.0])
    _, idx, vals = c.compress(g2.clone(), "w", ratio=0.25)
    assert idx.tolist() == [1] and abs(float(vals) - 0.8) < 1e-6


def test_gaussian_selects_about_k():
    torch.manual_seed(0)
    c = compressors["gaussian"]()
    g = torch.randn(20000)
    _, idx, vals = c.compress(g.clone(), "w", ratio=0.01)
    # every rank must contribute exactly k entries to the all-gather: short selections are padded with (0, 0.0)
    assert idx.numel() == 200 and vals.numel() == 200
    real = vals[vals != 0]
    assert 0 < real.numel() <= 200
    assert float(real.abs().min()) > float(g.abs().median())


def test_sign_pack_roundtrip_and_majority():
    torch.manual_seed(1)
    x = torch.randn(3, 37)
    words, sign = SignCompressor.packing(x)
    assert words.dtype == torch.int32 and words.numel() == (x.numel() + 31) // 32
    back = SignCompressor.unpacking(words, x.shape)
    assert torch.equal(back, torch.where(x >= 0, 1.0, -1.0))
    votes = [SignCompressor.packing(torch.randn(64) + m)[0] for m in (2.0, 2.0, -2.0)]
    maj = SignCompressor.unpacking(SignCompressor.majority_vote(votes), (64,))
    assert maj.mean() > 0.5


def test_efsign_residual():
    c = compressors["efsignum"]()
    g = torch.tensor([0.2, -3.0, 0.5])
    c.compress(g.clone(), "w")
    torch.testing.assert_close(c.residuals["w"], g - torch.sign(g))


def test_alpha_beta_fit_of_a_kernel_sweep(tmp_path):
    import json
    from dear_pytorch_b200.utils.perf_model import fit_alpha_beta, fused_kernel_model
    rows = [{"bucket_mb": mb, "t_us": 20.0 + 1.5 * mb} for mb in (1, 4, 24, 64)]
    a, b = fit_alpha_beta(rows, "t_us")
    assert abs(a - 20e-6) < 1e-9 and abs(b * 2 ** 20 - 1.5e-6) < 1e-12
    sweep = tmp_path / "sweep.json"
    sweep.write_text(json.dumps({"rows": [dict(world=8, bucket_mb=r["bucket_mb"], rs_us=r["t_us"]) for r in rows]}))
    m = fused_kernel_model(str(sweep))
    assert m["world"] == 8 and m["source"] == "sweep.json" and "allgather_update" not in m
    assert abs(m["reduce_scatter"][0] - 20e-6) < 1e-9 and abs(m["reduce_scatter"][1] * 2 ** 20 - 1.5e-6) < 1e-12
