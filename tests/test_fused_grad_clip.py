"""Global-norm clipping inside the fused kernels: Kernel A sums the squares of each bucket's reduced shard, the step's
first update kernel agrees on the norm with every rank, and every update kernel multiplies the coefficient into the
gradient.  Every case compares with single-process ``torch.optim`` + ``torch.nn.utils.clip_grad_norm_``.

The CPU part runs the host emulation of the kernels (same protocol, same arithmetic); the GPU part runs the kernels with
1, 2 or 4 ranks sharing the GPU through CUDA IPC."""
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from _mp import run_ranks
from test_dear_equivalence import data, make_model

ENV = {"DEAR_SPIN_TIMEOUT_S": "15"}
NAN = float("nan")


class _WithSpare(nn.Module):
    """The equivalence model plus a Linear that never takes part in the forward (its gradient is always None)."""

    def __init__(self):
        super().__init__()
        self.net = make_model()
        self.spare = nn.Linear(4, 4)

    def forward(self, x):
        return self.net(x)


def _make_opt(kind, model):
    ps = [p for n, p in model.named_parameters() if not n.startswith("spare")]
    groups = [{"params": ps[0::2]}, {"params": ps[1::2] + list(model.spare.parameters()), "lr": 0.02}]
    if kind == "sgd":
        return torch.optim.SGD(groups, lr=0.05, momentum=0.9, weight_decay=1e-3)
    if kind == "sgd-nesterov":
        return torch.optim.SGD(groups, lr=0.05, momentum=0.9, nesterov=True, weight_decay=1e-2)
    if kind == "adam":
        return torch.optim.Adam(groups, lr=0.01, weight_decay=1e-3)
    return torch.optim.AdamW(groups, lr=0.01)


def _poison_hook(state, poison, rank=None):
    def hook(g):
        v = poison.get(state["t"])
        if v is None or (rank is not None and state.get("rank") != rank):
            return g
        g = g.clone()
        g.view(-1)[0] = v
        return g
    return hook


def reference(kind, clips, steps, n, passes=1, poison=None):
    """``clips[t]``: max_norm of step t."""
    m = _WithSpare(); m.eval()
    opt = _make_opt(kind, m)
    st = {"t": 0}
    if poison:
        m.net[0].weight.register_hook(_poison_hook(st, poison))
    norms = []
    for t in range(steps):
        st["t"] = t
        opt.zero_grad()
        for k in range(passes):
            x, y = data(t * passes + k, n)
            F.cross_entropy(m(x), y).backward()
        norms.append(float(torch.nn.utils.clip_grad_norm_(m.parameters(), clips[t])))
        opt.step()
    return [p.detach().clone() for p in m.parameters()], norms


def clip_worker(rank, world, kind, clips, steps, n, passes=1, poison=None, rebucket_at=None, mode="eager",
                threshold=0.001):
    import dear_pytorch_b200 as dear
    dev = dear.device()
    m = _WithSpare().to(dev); m.eval()
    opt = dear.DistributedOptimizer(_make_opt(kind, m), m, threshold=threshold, norm_clip=clips[0],
                                    backward_passes_per_step=passes, verbose=False)
    dear.broadcast_parameters(m.state_dict(), 0)
    st = {"t": 0, "rank": rank}
    if poison:
        m.net[0].weight.register_hook(_poison_hook(st, poison, rank=world - 1))
    step = dear.TrainStep(m, opt, F.cross_entropy, overlap_update=mode == "rotated") if mode != "eager" else None
    per = n // world
    norms = []
    for t in range(steps):
        st["t"] = t
        if rebucket_at == t:
            opt.engine.rebucket(("threshold", 0.05))
        if opt.engine.norm_clip != clips[t]:
            opt.engine.norm_clip = clips[t]
        if step is not None:
            x, y = data(t, n)
            step(x[rank * per:(rank + 1) * per].to(dev), y[rank * per:(rank + 1) * per].to(dev))
            continue
        opt.zero_grad()
        for k in range(passes):
            x, y = data(t * passes + k, n)
            F.cross_entropy(m(x[rank * per:(rank + 1) * per].to(dev)), y[rank * per:(rank + 1) * per].to(dev)).backward()
        opt.step()
        norms.append(float(opt.engine.last_grad_norm))
    opt.synchronize()
    if dear.communicator() is not None:
        dear.communicator().check_status()
    return [p.detach().float().cpu().clone() for p in m.parameters()], norms


def _kw_worker(rank, world, kw):
    return clip_worker(rank, world, **kw)


def _check(outs, ref, rtol=2e-5, atol=2e-6, norm_rtol=1e-5):
    ref_params, ref_norms = ref
    for params, norms in outs:
        for a, b in zip(params, ref_params):
            torch.testing.assert_close(a, b, rtol=rtol, atol=atol, equal_nan=True)
        if norms:
            torch.testing.assert_close(torch.tensor(norms), torch.tensor(ref_norms), rtol=norm_rtol, atol=1e-6,
                                       equal_nan=True)
    first = outs[0][1]
    for _, norms in outs[1:]:
        assert torch.equal(torch.tensor(norms).view(torch.int32), torch.tensor(first).view(torch.int32))   # bit for bit


STEPS, N = 5, 6


# ------------------------------------------------------------------------------------------------ CPU (host emulation)
@pytest.mark.parametrize("world", [1, 2, 3])
@pytest.mark.parametrize("kind", ["sgd", "sgd-nesterov", "adam", "adamw"])
@pytest.mark.parametrize("clip", [0.5, 100.0])
def test_clipping_matches_clip_grad_norm(world, kind, clip):
    ref = reference(kind, [clip] * STEPS, STEPS, N)
    assert (max(ref[1]) > clip) == (clip < 1.0)              # 0.5 really clips, 100 never does
    _check(run_ranks(_kw_worker, world=world, backend="emu", args=(dict(kind=kind, clips=[clip] * STEPS, steps=STEPS, n=N),)),
           ref)


@pytest.mark.parametrize("mode", ["natural", "rotated"])
def test_train_step_matches_the_eager_loop(mode):
    ref = reference("sgd", [0.5] * STEPS, STEPS, N)
    _check(run_ranks(_kw_worker, world=2, backend="emu", args=(dict(kind="sgd", clips=[0.5] * STEPS, steps=STEPS, n=N,
                                                                   mode=mode),)), ref)


def test_gradient_accumulation():
    ref = reference("adamw", [0.5] * 4, 4, 4, passes=2)
    _check(run_ranks(_kw_worker, world=2, backend="emu", args=(dict(kind="adamw", clips=[0.5] * 4, steps=4, n=4, passes=2),)),
           ref)


@pytest.mark.parametrize("kind", ["sgd", "adam"])
def test_rebucket_mid_run(kind):
    ref = reference(kind, [0.5] * STEPS, STEPS, N)
    _check(run_ranks(_kw_worker, world=2, backend="emu", args=(dict(kind=kind, clips=[0.5] * STEPS, steps=STEPS, n=N,
                                                                   rebucket_at=2),)), ref)


def test_changing_norm_clip_between_steps_takes_effect():
    clips = [0.5, 0.5, 0.05, 100.0, 0.2]
    ref = reference("sgd", clips, len(clips), N)
    _check(run_ranks(_kw_worker, world=2, backend="emu", args=(dict(kind="sgd", clips=clips, steps=len(clips), n=N),)), ref)


@pytest.mark.parametrize("kind", ["sgd", "adam"])
def test_non_finite_gradient_without_a_scaler_matches_torch(kind):
    ref = reference(kind, [0.5] * 4, 4, N, poison={2: NAN})
    spare_w = ref[0][-2]
    assert torch.isnan(ref[0][0]).all() and not torch.isnan(spare_w).any()    # NaN everywhere but the unused Linear
    outs = run_ranks(_kw_worker, world=2, backend="emu", args=(dict(kind=kind, clips=[0.5] * 4, steps=4, n=N,
                                                                    poison={2: NAN}),))
    _check(outs, ref)
    for params, _ in outs:
        assert torch.equal(params[-2], _WithSpare().spare.weight.detach())         # untouched, not just close


def test_norms_are_bit_identical_across_ranks_and_runs():
    kw = dict(kind="adamw", clips=[0.5] * 4, steps=4, n=N)
    a = run_ranks(_kw_worker, world=3, backend="emu", args=(kw,))
    b = run_ranks(_kw_worker, world=3, backend="emu", args=(kw,))
    for (pa, na), (pb, nb) in zip(a, b):
        assert na == a[0][1] and nb == na
        assert all(torch.equal(x, y) for x, y in zip(pa, pb))


# ---- mixed dtypes: an fp16 and an fp32 bucket set share one coefficient ------------------------------------------------
class _Mixed(nn.Module):
    def __init__(self):
        super().__init__()
        torch.manual_seed(0)
        self.a = nn.Linear(8, 16).half()
        self.b = nn.Linear(16, 4)

    def forward(self, x):
        return self.b(self.a(x.half()).float())


def _mixed_batch(t, n):
    g = torch.Generator().manual_seed(7 + t)
    return torch.randn(n, 8, generator=g), torch.randint(0, 4, (n,), generator=g)


def _mixed_worker(rank, world, clip, steps, n):
    """One plain-SGD step at a time; returns, per step, the parameters before and after and the reported norm."""
    import dear_pytorch_b200 as dear
    dev = dear.device()
    m = _Mixed().to(dev)
    opt = dear.DistributedOptimizer(torch.optim.SGD(m.parameters(), lr=0.1), m, threshold=0.0001, norm_clip=clip,
                                    verbose=False)
    per = n // world
    out = []
    for t in range(steps):
        x, y = _mixed_batch(t, n)
        before = [p.detach().float().cpu().clone() for p in m.parameters()]
        opt.zero_grad()
        F.cross_entropy(m(x[rank * per:(rank + 1) * per].to(dev)), y[rank * per:(rank + 1) * per].to(dev)).backward()
        opt.step()
        norm = float(opt.engine.last_grad_norm)
        opt.synchronize()
        out.append((before, [p.detach().float().cpu().clone() for p in m.parameters()], norm))
    nsets = len(opt.engine.backend.sets)
    return out, nsets


def _check_mixed(outs, clip, n, world, tol=2e-3):
    for steps, nsets in outs:
        assert nsets == 2
        for t, (before, after, norm) in enumerate(steps):
            # the reference gradient of the parameters the rank held before the step, summed over the rank slices
            m = _Mixed()
            with torch.no_grad():
                for p, v in zip(m.parameters(), before):
                    p.copy_(v)
            x, y = _mixed_batch(t, n)
            per = n // world
            grads = [torch.zeros_like(v, dtype=torch.float64) for v in before]
            for r in range(world):
                m.zero_grad()
                F.cross_entropy(m(x[r * per:(r + 1) * per]), y[r * per:(r + 1) * per]).backward()
                for gsum, p in zip(grads, m.parameters()):
                    gsum += p.grad.double() / world
            total = torch.sqrt(sum((g * g).sum() for g in grads))
            coef = min(1.0, clip / (float(total) + 1e-6))
            assert coef < 0.5                                           # the clip bites: one coefficient matters
            assert abs(norm - float(total)) <= tol * float(total)
            for a, b, g in zip(after, before, grads):
                torch.testing.assert_close(a.double(), b.double() - 0.1 * coef * g, rtol=tol, atol=tol)


@pytest.mark.parametrize("world", [1, 2])
def test_fp16_and_fp32_sets_share_one_coefficient(world):
    outs = run_ranks(_mixed_worker, world=world, backend="emu", args=(0.05, 3, 4))
    _check_mixed(outs, 0.05, 4, world)


# ------------------------------------------------------------------------------------------------ GPU (fused kernels)
def _gpu_worlds():
    n = torch.cuda.device_count()
    return [w for w in (1, 2, 4) if n in (1, w) or n % w == 0]


def _gpu_env(algo):
    return dict(ENV, DEAR_RS_ALGO=algo)


@pytest.mark.gpu
@pytest.mark.parametrize("algo", ["oneshot", "pipe"])
@pytest.mark.parametrize("world", [1, 2, 4])
@pytest.mark.parametrize("kind", ["sgd", "adamw"])
def test_gpu_fp32_buckets_match_clip_grad_norm(algo, world, kind):
    if world not in _gpu_worlds():
        pytest.skip("needs %d ranks" % world)
    ref = reference(kind, [0.5] * 4, 4, 8)
    outs = run_ranks(_kw_worker, world=world, backend="b200", args=(dict(kind=kind, clips=[0.5] * 4, steps=4, n=8),),
                     extra_env=_gpu_env(algo), timeout=300)
    _check(outs, ref, rtol=2e-4, atol=2e-5, norm_rtol=1e-4)


def _bf16_worker(rank, world, clip, steps, n):
    import dear_pytorch_b200 as dear
    dev = dear.device()
    m = make_model().to(dev).to(torch.bfloat16); m.eval()
    opt = dear.DistributedOptimizer(torch.optim.SGD(m.parameters(), lr=0.05, momentum=0.9), m, threshold=0.001,
                                    norm_clip=clip, verbose=False)
    per = n // world
    norms = []
    for t in range(steps):
        x, y = data(t, n)
        opt.zero_grad()
        F.cross_entropy(m(x[rank * per:(rank + 1) * per].to(dev, torch.bfloat16)).float(),
                        y[rank * per:(rank + 1) * per].to(dev)).backward()
        opt.step()
        norms.append(float(opt.engine.last_grad_norm))
    opt.synchronize()
    dear.communicator().check_status()
    return [p.detach().float().cpu() for p in m.parameters()], norms


@pytest.mark.gpu
@pytest.mark.parametrize("algo", ["oneshot", "pipe"])
@pytest.mark.parametrize("world", [1, 2])
def test_gpu_bf16_buckets_with_masters_match_the_emulation(algo, world):
    """bf16 parameters with fp32 masters: the kernels against their host emulation (same protocol and arithmetic; the
    sums of squares are added in a different order, so the norms agree to rounding)."""
    if world not in _gpu_worlds():
        pytest.skip("needs %d ranks" % world)
    emu = run_ranks(_bf16_worker, world=world, backend="emu", args=(0.2, 3, 8))
    gpu = run_ranks(_bf16_worker, world=world, backend="b200", args=(0.2, 3, 8), extra_env=_gpu_env(algo), timeout=300)
    for (pg, ng), (pe, ne) in zip(gpu, emu):
        torch.testing.assert_close(torch.tensor(ng), torch.tensor(ne), rtol=1e-3, atol=1e-5)
        assert max(ne) > 0.2                             # the clip bites
        for a, b in zip(pg, pe):
            torch.testing.assert_close(a, b, rtol=2e-2, atol=2e-2)
    assert all(n == gpu[0][1] for _, n in gpu)


def _graph_worker(rank, world, mode, scaler_on, steps, n):
    """Eager loop and TrainStep(use_graph=True) on the same model / data; returns both parameter sets."""
    import dear_pytorch_b200 as dear
    dev = dear.device()
    per = n // world
    res = []
    for use_graph in (False, True):
        m = make_model().to(dev); m.eval()
        opt = dear.DistributedOptimizer(torch.optim.AdamW(m.parameters(), lr=0.01), m, threshold=0.001, norm_clip=0.5,
                                        verbose=False)
        scaler = dear.GradScaler(opt, init_scale=2.0 ** 10, growth_interval=3) if scaler_on else None
        step = dear.TrainStep(m, opt, F.cross_entropy, use_graph=use_graph, overlap_update=mode == "rotated",
                              scaler=scaler, graph_warmup=2)
        for t in range(steps):
            if t == steps - 2:
                opt.engine.norm_clip = 0.3                # a change between replays takes effect
            x, y = data(t, n)
            step(x[rank * per:(rank + 1) * per].to(dev), y[rank * per:(rank + 1) * per].to(dev))
        opt.synchronize()
        norm = float(opt.engine.last_grad_norm)
        res.append(([p.detach().float().cpu().clone() for p in m.parameters()], norm, step._graph is not None))
        opt.engine.close()
    dear.communicator().check_status()
    return res


@pytest.mark.gpu
@pytest.mark.parametrize("scaler_on", [False, True])
@pytest.mark.parametrize("mode", ["natural", "rotated"])
def test_gpu_cuda_graph_is_bitwise_equal_to_eager(mode, scaler_on):
    world = 2 if 2 in _gpu_worlds() else 1
    outs = run_ranks(_graph_worker, world=world, backend="b200", args=(mode, scaler_on, 8, 8), extra_env=ENV, timeout=300)
    for (pe, ne, _), (pg, ng, captured) in outs:
        assert captured
        assert ne == ng
        assert all(torch.equal(a, b) for a, b in zip(pe, pg))


def _slot_worker(rank, world, sizes, absent, algo_pipe):
    """BucketSet level: each bucket's slot == the float64 sum of squares of its reduced shard."""
    import dear_pytorch_b200 as dear
    from dear_pytorch_b200 import ops
    C = ops.native()
    dev = dear.device()
    comm = dear.communicator()
    bs = C.BucketSet(comm, [s * world for s in sizes], C.DT_F32, True)
    nb = len(sizes)
    state = torch.zeros(C.clip_state_floats(nb + 1), dtype=torch.float32, device=dev)
    state[0] = 1.0
    state.view(torch.int32)[3] = nb + 1
    slots = [nb - g for g in range(nb)]                              # engine-wide numbering need not be local order
    bs.set_clip(state, slots)
    g = torch.Generator().manual_seed(11 + rank)
    grads, shards = [], []
    for b, s in enumerate(sizes):
        shard = torch.zeros(s, dtype=torch.float32, device=dev)
        bs.set_shards(b, shard)
        gr = torch.randn(s * world, generator=g).to(dev)
        grads.append(gr)
        shards.append(shard)
        if b in absent:
            bs.set_pack(b, [0], [0], [s * world * 4], [1])                # zero-filled: no gradient on this rank
        else:
            bs.set_pack(b, [gr.data_ptr()], [0], [s * world * 4], [0])
        bs.reduce_scatter(b, True)
    bs.synchronize()
    st = state.cpu()
    out = []
    for b, s in enumerate(sizes):
        ref = float((shards[b].double() ** 2).sum())
        out.append((float(st[4 + slots[b]]), ref))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("algo", ["oneshot", "pipe"])
@pytest.mark.parametrize("world", [1, 2])
def test_gpu_bucket_slot_is_the_sum_of_squares_of_the_reduced_shard(algo, world):
    if world not in _gpu_worlds():
        pytest.skip("needs %d ranks" % world)
    sizes = [4, 1028, 3 * 65536 + 12, 1 << 20]
    outs = run_ranks(_slot_worker, world=world, backend="b200", args=(sizes, (1,), algo == "pipe"),
                     extra_env=_gpu_env(algo), timeout=300)
    for out in outs:
        for got, ref in out:
            assert abs(got - ref) <= 1e-5 * ref + 1e-6, (got, ref)
