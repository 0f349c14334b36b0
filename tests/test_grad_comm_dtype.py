"""``grad_comm_dtype``: fp32 gradients sent to the reduce-scatter as bf16 or fp16.

Semantics: the reduced shard of an fp32 bucket is  (sum over ranks, in rank order, of float32(g_q.to(D))) * s  with the
sum in fp32 and s = 1/P (times 1/scale with a loss scaler).  Everything after the shard is unchanged.  The reference is
single-process: each rank's gradient on its micro-batch, rounded with ``.to(D)``, summed in rank order, scaled, then
``torch.optim``.

The CPU part runs the host emulation of the kernels (and gloo where noted); the GPU part runs the kernels with ranks
sharing one GPU through CUDA IPC."""
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from _mp import run_ranks
from test_dear_equivalence import data
from test_fused_grad_clip import _WithSpare, _make_opt, _poison_hook

ENV = {"DEAR_SPIN_TIMEOUT_S": "15"}
WIRES = {"bf16": torch.bfloat16, "fp16": torch.float16}
DT_CODE = {"bf16": "DT_BF16", "fp16": "DT_F16"}


# ---------------------------------------------------------------------------------------------- bucket level
# segments of one fp32 bucket (element start, numel, kind); starts are multiples of 64 elements like the planner's
SEGS = [(0, 12345, "src"),            # odd count: a one-element tail
        (12352, 40001, "src"),        # crosses a 64 KiB tile of the 16-bit bucket, tail in the second tile
        (52416, 1000, "zero"),        # no gradient on this rank: zero-filled
        (53440, 3001, "staged")]      # copied into the bucket view by torch (copy_ rounds), packed in place
SPECIALS = {  # rank 0, segment 0: rounding ties, NaN, overflow and underflow of the 16-bit formats
    "bf16": [1.00390625, 1.01171875, -1.00390625, float("nan"), 7e4, -7e4, 3.4e38, 1e-30],
    "fp16": [1.00048828125, 1.00146484375, -1.00048828125, float("nan"), 7e4, -7e4, 65519.0, 65520.0, 1e-8, 3e-5]}


def _padded(world):
    q = world * 32                     # shard alignment of an fp32 bucket (128 bytes)
    end = SEGS[-1][0] + SEGS[-1][1]
    return (end + q - 1) // q * q


def _rank_grad(rank, wire, mode):
    """fp32 gradient of the whole bucket on this rank (zeros outside the segments and in the zero-filled one)."""
    g = torch.Generator().manual_seed(100 + rank)
    full = torch.zeros(_padded(8))
    for start, n, kind in SEGS:
        if kind != "zero":
            full[start:start + n] = torch.randn(n, generator=g) * 3
    if rank == 0 and mode == "specials":
        sp = torch.tensor(SPECIALS[wire])
        full[:len(sp)] = sp
        full[SEGS[0][1] - 1] = sp[0]                                     # the tail element is a tie too
    if rank == 0 and mode == "amp":
        full[5] = 7e4                                                    # finite in fp32 and bf16, inf in fp16
    return full


def formula(world, wire, mode, rounded=True):
    """Every rank's reduced shard, and the shard of the uncompressed sum."""
    n = _padded(world)
    acc = torch.zeros(n)
    for q in range(world):                                               # rank order, fp32
        g = _rank_grad(q, wire, mode)[:n]
        if mode == "specials" and q > 0:
            g[:len(SPECIALS[wire])] = 0.0
            g[SEGS[0][1] - 1] = 0.0
        acc = acc + (g.to(WIRES[wire]).float() if rounded else g)
    out = acc * (torch.tensor(1.0) / world)
    return list(out.view(world, -1))


def _bucket_worker(rank, world, wire, mode):
    import dear_pytorch_b200 as dear
    from dear_pytorch_b200 import ops
    C = ops.native()
    dev = dear.device()
    n = _padded(world)
    bs = C.BucketSet(dear.communicator(), [n], C.DT_F32, True, getattr(C, DT_CODE[wire]))
    shard = torch.zeros(n // world, device=dev)
    bs.set_shards(0, shard)
    gbuf = bs.grad_buffer(0)
    assert gbuf.dtype == WIRES[wire] and gbuf.numel() == n
    full = _rank_grad(rank, wire, mode)[:n]
    if mode == "specials" and rank > 0:
        full[:len(SPECIALS[wire])] = 0.0
        full[SEGS[0][1] - 1] = 0.0
    full = full.to(dev)
    keep, src, off, nbytes, flags = [], [], [], [], []
    for start, cnt, kind in SEGS:
        off.append(start * 2)
        nbytes.append(cnt * 2)
        if kind == "src":
            t = full[start:start + cnt].clone()
            keep.append(t)
            src.append(t.data_ptr()); flags.append(0)
        elif kind == "zero":
            gbuf[start:start + cnt].fill_(5.0)                          # stale contents the pack must clear
            src.append(0); flags.append(1)
        else:
            gbuf[start:start + cnt].copy_(full[start:start + cnt])      # torch rounds
            src.append(0); flags.append(0)
    state = None
    if mode == "amp":
        state = torch.zeros(9, dtype=torch.int32, device=dev)
        state.view(torch.float32)[2] = 1.0
        bs.set_amp(state)
    if mode == "clip":
        state = torch.zeros(C.clip_state_floats(1), dtype=torch.float32, device=dev)
        state[0] = 1.0
        state.view(torch.int32)[3] = 1
        bs.set_clip(state, [0])
    bs.set_pack(0, src, off, nbytes, flags)
    bs.reduce_scatter(0, True)
    bs.synchronize()
    extra = None
    if mode == "amp":
        extra = int(state[0])
    elif mode == "clip":
        extra = float(state[4])
    return shard.cpu(), extra, bs.rs_plan(0)


def _same_bits(a, b):
    """Bit for bit, except that every NaN matches every NaN (the payload of a rounded NaN is not part of .to())."""
    na, nb = torch.isnan(a), torch.isnan(b)
    assert torch.equal(na, nb)
    assert torch.equal(a[~na].view(torch.int32), b[~nb].view(torch.int32))


def _check_bucket(outs, world, wire, mode):
    ref = formula(world, wire, mode)
    plain = formula(world, wire, mode, rounded=False)
    for r, (shard, extra, plan) in enumerate(outs):
        _same_bits(shard, ref[r])
        assert not torch.equal(shard, plain[r])                          # the option is not ignored
        assert plan.startswith("oneshot") and plan.endswith(":wire=" + wire)
        if mode == "amp":                                                # 7e4 overflows fp16 only, in rank 0's shard
            assert extra == (1 if wire == "fp16" and r == 0 else 0)
        if mode == "clip":
            ss = float((ref[r].double() ** 2).sum())
            assert abs(extra - ss) <= 1e-4 * ss                          # fp32 sums of ~3e4 squares
    if mode == "specials" and world == 2:
        sp = outs[0][0][:len(SPECIALS[wire])] * 2                        # rank 0's own rounded values (exact at P = 2)
        if wire == "fp16":
            assert torch.isinf(sp[4]) and torch.isinf(sp[5]) and sp[6] == 65504.0 and torch.isinf(sp[7])
        else:
            assert torch.isfinite(sp[4]) and torch.isinf(sp[6])
        assert float(sp[0]) == 1.0 and torch.isnan(sp[3])                # a tie rounds to even; NaN stays NaN


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("wire", ["bf16", "fp16"])
@pytest.mark.parametrize("mode", ["specials", "amp", "clip"])
def test_reduced_shard_is_the_formula_bit_for_bit(world, wire, mode):
    _check_bucket(run_ranks(_bucket_worker, world=world, backend="emu", args=(wire, mode)), world, wire, mode)


def _plan_worker(rank, world):
    import dear_pytorch_b200 as dear
    from dear_pytorch_b200 import ops
    C = ops.native()
    plans = [C.BucketSet(dear.communicator(), [1 << 16], C.DT_F32, True, gd).rs_plan(0) for gd in (None, C.DT_BF16)]
    with pytest.raises(RuntimeError):
        C.BucketSet(dear.communicator(), [1 << 16], C.DT_BF16, True, C.DT_F16)      # only fp32 sets convert
    return plans


def test_converting_bucket_falls_back_to_oneshot_under_pipe():
    for plain, conv in run_ranks(_plan_worker, world=2, backend="emu", extra_env={"DEAR_RS_ALGO": "pipe"}):
        assert plain.startswith("pipe") and ":wire=" not in plain
        assert conv.startswith("oneshot") and conv.endswith(":wire=bf16")


# ---------------------------------------------------------------------------------------------- training
def reference(kind, steps, n, world, wire, passes=1, clip=None, model_fn=_WithSpare, make_opt=_make_opt):
    """Per-rank gradients rounded to the wire dtype, summed in rank order in fp32, times 1/P, then torch.optim."""
    m = model_fn(); m.eval()
    opt = make_opt(kind, m)
    per = n // world
    norms = []
    for t in range(steps):
        acc = {}
        for r in range(world):
            m.zero_grad()
            for k in range(passes):
                x, y = data(t * passes + k, n)
                F.cross_entropy(m(x[r * per:(r + 1) * per]), y[r * per:(r + 1) * per]).backward()
            for p in m.parameters():
                if p.grad is not None:
                    g = p.grad.to(WIRES[wire]).float() if wire else p.grad
                    acc[p] = acc.get(p, torch.zeros_like(p, dtype=torch.float32)) + g
        for p in m.parameters():
            p.grad = (acc[p] * (torch.tensor(1.0) / world)).to(p.dtype) if p in acc else None
        if clip is not None:
            norms.append(float(torch.nn.utils.clip_grad_norm_(m.parameters(), clip)))
        opt.step()
    return [p.detach().clone() for p in m.parameters()], norms


def train_worker(rank, world, kind, wire, steps, n, passes=1, clip=None, rebucket_at=None, mode="eager",
                 ckpt_at=None, ckpt_path=None, model_fn=_WithSpare, make_opt=_make_opt):
    import dear_pytorch_b200 as dear
    dev = dear.device()
    wdt = WIRES.get(wire)

    def build():
        m = model_fn().to(dev); m.eval()
        o = dear.DistributedOptimizer(make_opt(kind, m), m, threshold=0.001, norm_clip=clip, grad_comm_dtype=wdt,
                                      backward_passes_per_step=passes, verbose=False)
        return m, o

    m, opt = build()
    assert opt.engine.grad_comm_dtype == wdt
    direct = len(opt.engine._direct_params)
    step = dear.TrainStep(m, opt, F.cross_entropy, overlap_update=mode == "rotated") if mode != "eager" else None
    per = n // world
    norms = []
    for t in range(steps):
        if rebucket_at == t:
            opt.engine.rebucket(("threshold", 0.05))
        if ckpt_at == t:
            dear.save_checkpoint(ckpt_path, m, opt)
            opt.engine.close()
            m, opt = build()
            dear.load_checkpoint(ckpt_path, m, opt)
        if step is not None:
            x, y = data(t, n)
            step(x[rank * per:(rank + 1) * per].to(dev), y[rank * per:(rank + 1) * per].to(dev))
            continue
        for k in range(passes):
            x, y = data(t * passes + k, n)
            F.cross_entropy(m(x[rank * per:(rank + 1) * per].to(dev)), y[rank * per:(rank + 1) * per].to(dev)).backward()
        opt.step()
        if clip is not None:
            norms.append(float(opt.engine.last_grad_norm))
    opt.synchronize()
    if dear.communicator() is not None:
        dear.communicator().check_status()
    return [p.detach().float().cpu().clone() for p in m.parameters()], norms, direct


def _kw_worker(rank, world, kw):
    return train_worker(rank, world, **kw)


# atol: parameters that differ from the reference by ~1e-9 (summation order, torch.optim's formulas) give gradients that
# now and then round to the neighbouring 16-bit value on one side only; Adam (lr 0.01) turns such a one-ulp difference
# into up to a few 1e-5 of one parameter.  The bucket-level tests above pin the rounding down bit for bit.
def _check(outs, ref, rtol=2e-5, atol=5e-5, spare=True):
    ref_params, ref_norms = ref
    for params, norms, _ in outs:
        for a, b in zip(params, ref_params):
            torch.testing.assert_close(a, b, rtol=rtol, atol=atol)
        if ref_norms:
            torch.testing.assert_close(torch.tensor(norms), torch.tensor(ref_norms), rtol=1e-5, atol=1e-6)
        if spare:                                  # the Linear that never runs stays bit-exact
            fresh = _WithSpare().spare
            assert torch.equal(params[-2], fresh.weight.detach()) and torch.equal(params[-1], fresh.bias.detach())


STEPS, N = 5, 6


@pytest.mark.parametrize("backend,world", [("emu", 2), ("emu", 3), ("gloo", 2)])
@pytest.mark.parametrize("wire", ["bf16", "fp16"])
@pytest.mark.parametrize("kind", ["sgd", "sgd-nesterov", "adam", "adamw"])
def test_training_matches_the_rounded_reference(backend, world, wire, kind):
    ref = reference(kind, STEPS, N, world, wire)
    plain = reference(kind, STEPS, N, world, None)
    assert not all(torch.equal(a, b) for a, b in zip(ref[0], plain[0]))      # the rounding matters at this size
    _check(run_ranks(_kw_worker, world=world, backend=backend,
                     args=(dict(kind=kind, wire=wire, steps=STEPS, n=N),)), ref)


class _Mlp(nn.Module):
    """Linear layers only: every weight gradient is a GEMM that direct wgrad could write into the bucket."""

    def __init__(self):
        super().__init__()
        torch.manual_seed(0)
        self.net = nn.Sequential(nn.Flatten(), nn.Linear(192, 64), nn.ReLU(), nn.Linear(64, 64), nn.ReLU(),
                                 nn.Linear(64, 10))

    def forward(self, x):
        return self.net(x)


def _mlp_opt(kind, m):
    return torch.optim.SGD(m.parameters(), lr=0.05, momentum=0.9)


@pytest.mark.parametrize("wire", [None, "bf16"])
def test_direct_wgrad_is_off_for_converting_buckets(wire):
    ref = reference("sgd", 4, 4, 2, wire, model_fn=_Mlp, make_opt=_mlp_opt)
    outs = run_ranks(_kw_worker, world=2, backend="emu",
                     args=(dict(kind="sgd", wire=wire, steps=4, n=4, model_fn=_Mlp, make_opt=_mlp_opt),))
    _check(outs, ref, spare=False)
    for _, _, direct in outs:
        assert (direct > 0) == (wire is None)


def test_gradient_accumulation():
    ref = reference("adamw", 4, 4, 2, "bf16", passes=2)
    _check(run_ranks(_kw_worker, world=2, backend="emu",
                     args=(dict(kind="adamw", wire="bf16", steps=4, n=4, passes=2),)), ref)


def test_rebucket_mid_run():
    ref = reference("sgd", STEPS, N, 2, "fp16")
    _check(run_ranks(_kw_worker, world=2, backend="emu",
                     args=(dict(kind="sgd", wire="fp16", steps=STEPS, n=N, rebucket_at=2),)), ref)


def test_checkpoint_round_trip(tmp_path):
    ref = reference("adam", STEPS, N, 2, "bf16")
    _check(run_ranks(_kw_worker, world=2, backend="emu",
                     args=(dict(kind="adam", wire="bf16", steps=STEPS, n=N, ckpt_at=3,
                                ckpt_path=str(tmp_path / "ck.pt")),)), ref)


def test_norm_clip_is_the_norm_of_the_compressed_average():
    ref = reference("sgd", STEPS, N, 2, "bf16", clip=0.5)
    assert max(ref[1]) > 0.5
    _check(run_ranks(_kw_worker, world=2, backend="emu",
                     args=(dict(kind="sgd", wire="bf16", steps=STEPS, n=N, clip=0.5),)), ref)


@pytest.mark.parametrize("mode", ["natural", "rotated"])
def test_train_step(mode):
    ref = reference("sgd", STEPS, N, 2, "fp16")
    _check(run_ranks(_kw_worker, world=2, backend="emu",
                     args=(dict(kind="sgd", wire="fp16", steps=STEPS, n=N, mode=mode),)), ref)


class _MixedBf16(nn.Module):
    def __init__(self):
        super().__init__()
        torch.manual_seed(0)
        self.a = nn.Linear(192, 16).to(torch.bfloat16)
        self.b = nn.Linear(16, 10)

    def forward(self, x):
        return self.b(self.a(x.flatten(1).to(torch.bfloat16)).float())


def _mixed_opt(kind, m):
    return torch.optim.SGD(m.parameters(), lr=0.1, momentum=0.9)


def test_bf16_set_is_unaffected_in_a_mixed_model():
    """One step: the bf16 parameters are bitwise those of a run without the option, the fp32 ones follow the formula."""
    kw = dict(kind="sgd", steps=1, n=4, model_fn=_MixedBf16, make_opt=_mixed_opt)
    on = run_ranks(_kw_worker, world=2, backend="emu", args=(dict(kw, wire="bf16"),))
    off = run_ranks(_kw_worker, world=2, backend="emu", args=(dict(kw, wire=None),))
    for (pon, _, _), (poff, _, _) in zip(on, off):
        assert torch.equal(pon[0], poff[0]) and torch.equal(pon[1], poff[1])      # bf16 layer
        assert not torch.equal(pon[2], poff[2])                                    # fp32 layer: rounded gradients
    ref = reference("sgd", 1, 4, 2, "bf16", model_fn=_MixedBf16, make_opt=_mixed_opt)
    for params, _, _ in on:
        torch.testing.assert_close(params[2], ref[0][2], rtol=2e-5, atol=2e-6)


def test_world_one_is_a_no_op():
    kw = dict(kind="adamw", steps=4, n=4)
    on = run_ranks(_kw_worker, world=1, backend="emu", args=(dict(kw, wire="fp16"),))
    off = run_ranks(_kw_worker, world=1, backend="emu", args=(dict(kw, wire=None),))
    assert all(torch.equal(a, b) for a, b in zip(on[0][0], off[0][0]))


# ---- fp16 with a dynamic loss scaler: an overflow in the cast skips the step on every rank ----------------------------
def _scaler_worker(rank, world, wire, steps, n, poison_step):
    import dear_pytorch_b200 as dear
    dev = dear.device()
    m = _WithSpare().to(dev); m.eval()
    opt = dear.DistributedOptimizer(_make_opt("sgd", m), m, threshold=0.001, grad_comm_dtype=WIRES[wire], verbose=False)
    scaler = dear.GradScaler(opt, init_scale=2.0 ** 10, growth_interval=1000)
    st = {"t": 0, "rank": rank}
    m.net[0].weight.register_hook(_poison_hook(st, {poison_step: 1e5}, rank=world - 1))   # finite, > fp16's max
    per = n // world
    for t in range(steps):
        st["t"] = t
        x, y = data(t, n)
        scaler.scale(F.cross_entropy(m(x[rank * per:(rank + 1) * per].to(dev)),
                                     y[rank * per:(rank + 1) * per].to(dev))).backward()
        scaler.step(opt)
        scaler.update()
    opt.synchronize()
    return scaler.get_scale(), opt.engine.read_scaler()["applied"], [p.detach().cpu().clone() for p in m.parameters()]


@pytest.mark.parametrize("wire", ["bf16", "fp16"])
def test_fp16_overflow_in_the_cast_skips_the_step(wire):
    outs = run_ranks(_scaler_worker, world=2, backend="emu", args=(wire, 3, 4, 1))
    for scale, applied, params in outs:
        if wire == "fp16":
            assert scale == 2.0 ** 9 and applied == 2
        else:
            assert scale == 2.0 ** 10 and applied == 3
        assert all(torch.equal(a, b) for a, b in zip(params, outs[0][2]))


# ---- errors -----------------------------------------------------------------------------------------------------------
def _err_worker(rank, world):
    import dear_pytorch_b200 as dear
    m = _WithSpare()
    with pytest.raises(ValueError):
        dear.DistributedOptimizer(_make_opt("sgd", m), m, grad_comm_dtype=torch.int8, verbose=False)
    m = _WithSpare()
    try:
        dear.DistributedOptimizer(_make_opt("sgd", m), m, grad_comm_dtype=torch.bfloat16 if rank == 1 else None,
                                  verbose=False)
    except RuntimeError as e:
        return str(e)
    return None


def test_errors():
    for msg in run_ranks(_err_worker, world=2, backend="emu"):
        assert msg is not None and "grad_comm_dtype" in msg


# ---------------------------------------------------------------------------------------------- GPU (fused kernels)
def _gpu_worlds():
    n = torch.cuda.device_count()
    return [w for w in (2, 3, 4) if n in (1, w) or n % w == 0]


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3, 4])
@pytest.mark.parametrize("wire", ["bf16", "fp16"])
@pytest.mark.parametrize("mode", ["specials", "amp", "clip"])
def test_gpu_reduced_shard_is_the_formula_and_the_emulation(world, wire, mode):
    """W-specialised pulls at 2 and 4 ranks, the generic one at 3; the plain, AMP and CLIP instantiations."""
    if world not in _gpu_worlds():
        pytest.skip("needs %d ranks" % world)
    gpu = run_ranks(_bucket_worker, world=world, backend="b200", args=(wire, mode), extra_env=ENV, timeout=300)
    emu = run_ranks(_bucket_worker, world=world, backend="emu", args=(wire, mode))
    _check_bucket(gpu, world, wire, mode)
    for (sg, _, _), (se, _, _) in zip(gpu, emu):
        _same_bits(sg, se)


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("kind", ["sgd", "adamw"])
def test_gpu_training_matches_the_emulation(world, kind):
    if world not in _gpu_worlds():
        pytest.skip("needs %d ranks" % world)
    kw = dict(kind=kind, wire="bf16", steps=4, n=8)
    gpu = run_ranks(_kw_worker, world=world, backend="b200", args=(kw,), extra_env=ENV, timeout=300)
    emu = run_ranks(_kw_worker, world=world, backend="emu", args=(kw,))
    for (pg, _, _), (pe, _, _) in zip(gpu, emu):
        for a, b in zip(pg, pe):
            torch.testing.assert_close(a, b, rtol=2e-4, atol=1e-4)     # one-ulp rounding flips, as in _check


def _graph_worker(rank, world, mode, steps, n):
    import dear_pytorch_b200 as dear
    dev = dear.device()
    per = n // world
    res = []
    for use_graph in (False, True):
        m = _WithSpare().to(dev); m.eval()
        opt = dear.DistributedOptimizer(torch.optim.AdamW(m.parameters(), lr=0.01), m, threshold=0.001, norm_clip=0.5,
                                        grad_comm_dtype=torch.float16, verbose=False)
        scaler = dear.GradScaler(opt, init_scale=2.0 ** 10, growth_interval=3)
        step = dear.TrainStep(m, opt, F.cross_entropy, use_graph=use_graph, overlap_update=mode == "rotated",
                              scaler=scaler, graph_warmup=2)
        for t in range(steps):
            x, y = data(t, n)
            step(x[rank * per:(rank + 1) * per].to(dev), y[rank * per:(rank + 1) * per].to(dev))
        opt.synchronize()
        res.append(([p.detach().float().cpu().clone() for p in m.parameters()], float(opt.engine.last_grad_norm),
                    step._graph is not None))
        opt.engine.close()
    dear.communicator().check_status()
    return res


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["natural", "rotated"])
def test_gpu_cuda_graph_is_bitwise_equal_to_eager(mode):
    if 2 not in _gpu_worlds():
        pytest.skip("needs 2 ranks")
    outs = run_ranks(_graph_worker, world=2, backend="b200", args=(mode, 8, 8), extra_env=ENV, timeout=300)
    for (pe, ne, _), (pg, ng, captured) in outs:
        assert captured
        assert ne == ng
        assert all(torch.equal(a, b) for a, b in zip(pe, pg))


def _nvls_worker(rank, world, wire):
    import dear_pytorch_b200 as dear
    from dear_pytorch_b200 import ops
    C = ops.native()
    bs = C.BucketSet(dear.communicator(), [_padded(world)], C.DT_F32, True, getattr(C, DT_CODE[wire]))
    if not bs.has_multicast():
        return None
    return _bucket_worker(rank, world, wire, "specials")


@pytest.mark.gpu
@pytest.mark.parametrize("wire", ["bf16", "fp16"])
def test_gpu_nvls_converting_bucket(wire):
    """multimem.ld_reduce over a converting bucket: needs an NVLS multicast object across at least 2 GPUs."""
    if torch.cuda.device_count() < 2:
        pytest.skip("NVLS multicast needs at least 2 GPUs")
    world = min(torch.cuda.device_count(), 4)
    outs = run_ranks(_nvls_worker, world=world, backend="b200", args=(wire,),
                     extra_env=dict(ENV, DEAR_RS_ALGO="nvls"), timeout=300)
    if outs[0] is None:
        pytest.skip("no multicast object on this system")
    _check_bucket(outs, world, wire, "specials")
