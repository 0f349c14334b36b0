"""``dear.GradScaler``: dynamic loss scaling on the fused path == ``torch.amp.GradScaler`` around ``torch.optim``.

Overflows are injected into one parameter's gradient on ONE rank at chosen steps (a tensor hook keyed on the step);
the reference injects into the same parameter of a single process at the same steps.  Every rank must skip exactly
those steps, and the scale / growth-tracker sequences must be torch's, bit for bit."""
import os
import sys

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from _mp import run_ranks
from test_dear_equivalence import data, make_model

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INIT, GI = 2.0 ** 10, 3              # small growth interval: the scale grows within the test
POISON_PARAM = 0                     # first conv weight
INF, NAN = float("inf"), float("nan")


def _make_opt(kind, params):
    if kind == "sgd":
        return torch.optim.SGD(params, lr=0.05, momentum=0.8, dampening=0.3, weight_decay=5e-3)
    if kind == "sgd-nesterov":
        return torch.optim.SGD(params, lr=0.05, momentum=0.9, nesterov=True, weight_decay=1e-2)
    if kind == "adam":
        return torch.optim.Adam(params, lr=0.01, weight_decay=1e-3)
    return torch.optim.AdamW(params, lr=0.01)


def _poison_hook(state, poison, rank=None):
    """Replace element 0 of the gradient by ``poison[step]`` (first backward pass of the step only)."""
    def hook(g):
        v = poison.get(state["t"])
        if v is None or state.get("pass", 0) != 0 or (rank is not None and state.get("rank") != rank):
            return g
        g = g.clone()
        g.view(-1)[0] = v
        return g
    return hook


def reference(kind, steps, n, poison, passes=1, clip=None):
    m = make_model(); m.eval()
    opt = _make_opt(kind, m.parameters())
    sc = torch.amp.GradScaler("cpu", init_scale=INIT, growth_interval=GI)
    st = {"t": 0}
    list(m.parameters())[POISON_PARAM].register_hook(_poison_hook(st, poison))
    scales, trackers, norms = [], [], []
    for t in range(steps):
        st["t"] = t
        opt.zero_grad()
        for k in range(passes):
            st["pass"] = k
            x, y = data(t * passes + k, n)
            sc.scale(F.cross_entropy(m(x), y)).backward()
        if clip is not None:
            sc.unscale_(opt)
            norms.append(float(torch.nn.utils.clip_grad_norm_(m.parameters(), clip)))
        sc.step(opt)
        sc.update()
        scales.append(sc.get_scale())
        trackers.append(sc._get_growth_tracker())
    return [p.detach().clone() for p in m.parameters()], opt.state_dict()["state"], scales, trackers, norms


def scaler_worker(rank, world, kind, steps, n, poison, passes=1, clip=None, rebucket_at=None, mode="eager",
                  enabled=True, threshold=0.001):
    import dear_pytorch_b200 as dear
    dev = dear.device()
    m = make_model().to(dev); m.eval()
    opt = dear.DistributedOptimizer(_make_opt(kind, m.parameters()), m, threshold=threshold, norm_clip=clip,
                                    backward_passes_per_step=passes, verbose=False)
    dear.broadcast_parameters(m.state_dict(), 0)
    scaler = dear.GradScaler(opt, init_scale=INIT, growth_interval=GI, enabled=enabled) if mode != "none" else None
    st = {"t": 0, "rank": rank}
    list(m.parameters())[POISON_PARAM].register_hook(_poison_hook(st, poison, rank=world - 1))
    per = n // world
    step = None
    if mode in ("natural", "rotated"):
        step = dear.TrainStep(m, opt, F.cross_entropy, overlap_update=mode == "rotated", scaler=scaler)
    scales, trackers, norms = [], [], []
    for t in range(steps):
        if rebucket_at == t:
            opt.engine.rebucket(("threshold", 0.05))
        st["t"] = t
        if step is not None:
            x, y = data(t, n)
            step(x[rank * per:(rank + 1) * per].to(dev), y[rank * per:(rank + 1) * per].to(dev))
        else:
            opt.zero_grad()
            for k in range(passes):
                st["pass"] = k
                x, y = data(t * passes + k, n)
                loss = F.cross_entropy(m(x[rank * per:(rank + 1) * per].to(dev)), y[rank * per:(rank + 1) * per].to(dev))
                (scaler.scale(loss) if scaler is not None else loss).backward()
            if scaler is not None:
                scaler.unscale_(opt)
                scaler.step(opt)
                scaler.update()
            else:
                opt.step()
        if mode == "eager" and scaler is not None:
            scales.append(scaler.get_scale())
            trackers.append(scaler._get_growth_tracker())
        if clip is not None:
            norms.append(float(opt.engine.last_grad_norm))
    opt.synchronize()
    state = opt.state_dict()["state"]
    final = scaler.get_scale() if scaler is not None else None
    if dear.communicator() is not None:
        dear.communicator().check_status()
    return ([p.detach().float().cpu().clone() for p in m.parameters()],
            {i: {k: v.float().cpu() for k, v in s.items() if torch.is_tensor(v) and k != "master_param"} for i, s in state.items()},
            scales, trackers, norms, final)


def _check(outs, ref, check_seq=True, rtol=2e-5, atol=2e-6):
    ref_params, ref_state, ref_scales, ref_trackers, ref_norms = ref
    for params, state, scales, trackers, norms, final in outs:
        if check_seq:
            assert scales == ref_scales
            assert trackers == ref_trackers
        assert final == ref_scales[-1]
        for a, b in zip(params, ref_params):
            torch.testing.assert_close(a, b, rtol=rtol, atol=atol)
        for i, ent in ref_state.items():
            for k, v in ent.items():
                if k in ("momentum_buffer", "exp_avg", "exp_avg_sq", "step"):
                    torch.testing.assert_close(state[i][k], v.float(), rtol=rtol, atol=atol)
        if ref_norms:
            a, b = torch.tensor(norms), torch.tensor(ref_norms)
            fin = torch.isfinite(b)
            assert torch.equal(torch.isfinite(a), fin)        # inf / NaN exactly on the overflowing steps
            torch.testing.assert_close(a[fin], b[fin], rtol=1e-5, atol=1e-6)


# overflows on the first two steps (the first applied update comes late), a NaN, and one after growth
POISON = {0: INF, 1: NAN, 5: -INF}
STEPS, N = 8, 6


@pytest.mark.parametrize("backend,world", [("emu", 1), ("emu", 2), ("emu", 3), ("gloo", 2), ("gloo", 3)])
@pytest.mark.parametrize("kind", ["sgd", "sgd-nesterov", "adam", "adamw"])
def test_injected_overflow_matches_torch_grad_scaler(backend, world, kind):
    ref = reference(kind, STEPS, N, POISON)
    assert ref[2][:2] == [INIT / 2, INIT / 4] and max(ref[2]) > INIT / 4      # backs off, then grows
    _check(run_ranks(scaler_worker, world=world, backend=backend, args=(kind, STEPS, N, POISON)), ref)


@pytest.mark.parametrize("backend", ["emu", "gloo"])
def test_gradient_accumulation_with_an_overflow_in_the_first_pass(backend):
    ref = reference("sgd", 5, 4, {1: INF, 2: NAN}, passes=2)
    outs = run_ranks(_kw_worker, world=2, backend=backend, args=(dict(kind="sgd", steps=5, n=4, poison={1: INF, 2: NAN},
                                                                       passes=2),))
    _check(outs, ref)


def _kw_worker(rank, world, kw):
    return scaler_worker(rank, world, **kw)


@pytest.mark.parametrize("backend,kind", [("emu", "sgd"), ("emu", "adamw"), ("gloo", "adamw")])
def test_norm_clip_with_a_scaler(backend, kind):
    ref = reference(kind, 6, N, {0: INF, 3: NAN}, clip=0.5)
    outs = run_ranks(_kw_worker, world=2, backend=backend, args=(dict(kind=kind, steps=6, n=N, poison={0: INF, 3: NAN},
                                                                       clip=0.5),))
    _check(outs, ref)


@pytest.mark.parametrize("backend", ["emu", "gloo"])
@pytest.mark.parametrize("kind", ["sgd", "adam"])
def test_rebucket_mid_run_keeps_scale_tracker_and_applied_count(backend, kind):
    ref = reference(kind, STEPS, N, POISON)
    outs = run_ranks(_kw_worker, world=2, backend=backend, args=(dict(kind=kind, steps=STEPS, n=N, poison=POISON,
                                                                       rebucket_at=3),))
    _check(outs, ref)


@pytest.mark.parametrize("mode", ["natural", "rotated"])
def test_train_step_with_a_scaler_matches_the_eager_loop(mode):
    ref = reference("sgd", STEPS, N, POISON)
    outs = run_ranks(_kw_worker, world=2, backend="emu", args=(dict(kind="sgd", steps=STEPS, n=N, poison=POISON, mode=mode),))
    _check(outs, ref, check_seq=False)


def test_disabled_scaler_reproduces_the_unscaled_run_exactly():
    off = run_ranks(_kw_worker, world=2, backend="emu", args=(dict(kind="adam", steps=4, n=N, poison={}, enabled=False),))
    none = run_ranks(_kw_worker, world=2, backend="emu", args=(dict(kind="adam", steps=4, n=N, poison={}, mode="none"),))
    for (pa, sa, *_), (pb, sb, *_) in zip(off, none):
        assert all(torch.equal(a, b) for a, b in zip(pa, pb))
        assert all(torch.equal(sa[i][k], sb[i][k]) for i in sb for k in sb[i])


# ---- mixed dtypes: one decision for the fp16 and the fp32 bucket sets ------------------------------------------------------
class _Mixed(nn.Module):
    def __init__(self):
        super().__init__()
        torch.manual_seed(0)
        self.a = nn.Linear(8, 16).half()
        self.b = nn.Linear(16, 4)

    def forward(self, x):
        return self.b(self.a(x.half()).float())


def _mixed_worker(rank, world, poison, steps, device_type=None):
    import dear_pytorch_b200 as dear
    dev = dear.device()
    m = _Mixed().to(dev)
    opt = dear.DistributedOptimizer(torch.optim.SGD(m.parameters(), lr=0.1, momentum=0.9), m, threshold=0.001, verbose=False)
    scaler = dear.GradScaler(opt, init_scale=INIT, growth_interval=GI)
    st = {"t": 0, "rank": rank}
    m.a.weight.register_hook(_poison_hook(st, poison, rank=0))      # only the fp16 bucket overflows
    snaps, scales = [], []
    g = torch.Generator().manual_seed(7)
    for t in range(steps):
        st["t"] = t
        x, y = torch.randn(4, 8, generator=g), torch.randint(0, 4, (4,), generator=g)
        opt.zero_grad()
        scaler.scale(F.cross_entropy(m(x.to(dev)), y.to(dev))).backward()
        scaler.step(opt)
        scaler.update()
        opt.synchronize()
        snaps.append([p.detach().float().cpu().clone() for p in m.parameters()])
        scales.append(scaler.get_scale())
    dear.communicator().check_status()
    return snaps, scales, len(opt.engine.backend.sets) if hasattr(opt.engine.backend, "sets") else 2


def _check_mixed(outs, poison, steps):
    for snaps, scales, nsets in outs:
        assert nsets == 2
        s, expect = INIT, []
        tracker = 0
        for t in range(steps):
            if t in poison:
                s, tracker = s * 0.5, 0
            else:
                tracker += 1
                if tracker == GI:
                    s, tracker = s * 2, 0
            expect.append(s)
        assert scales == expect
        for t in range(1, steps):
            same = all(torch.equal(a, b) for a, b in zip(snaps[t], snaps[t - 1]))
            assert same == (t in poison), t                  # the fp32 bucket is skipped together with the fp16 one
    for a, b in zip(outs[0][0][-1], outs[-1][0][-1]):
        assert torch.equal(a, b)


@pytest.mark.parametrize("world", [1, 2])
def test_mixed_dtype_model_skips_every_bucket_set_together(world):
    poison = {2: INF, 3: NAN}
    _check_mixed(run_ranks(_mixed_worker, world=world, backend="emu", args=(poison, 6)), poison, 6)


# ---- state dict, argument checks -------------------------------------------------------------------------------------------
def _state_dict_worker(rank, world):
    import dear_pytorch_b200 as dear
    m = make_model(); m.eval()
    opt = dear.DistributedOptimizer(torch.optim.SGD(m.parameters(), lr=0.05), m, verbose=False)
    scaler = dear.GradScaler(opt, init_scale=INIT, growth_interval=GI)
    st = {"t": 0, "rank": rank}
    list(m.parameters())[0].register_hook(_poison_hook(st, {1: INF}))
    for t in range(5):
        st["t"] = t
        x, y = data(t, 4)
        scaler.scale(F.cross_entropy(m(x), y)).backward()
        scaler.step(opt)
        scaler.update()
    sd = scaler.state_dict()
    ts = torch.amp.GradScaler("cpu")
    ts.load_state_dict(sd)
    ts_sd = ts.state_dict()
    m1 = make_model()
    back = dear.GradScaler(dear.DistributedOptimizer(torch.optim.SGD(m1.parameters(), lr=0.05), m1, verbose=False))
    back.load_state_dict(dict(ts_sd, scale=3.0))
    errors = []
    try:
        dear.GradScaler(torch.optim.SGD(make_model().parameters(), lr=0.1))
    except TypeError as e:
        errors.append(str(e))
    m2 = make_model()
    try:
        dear.GradScaler(dear.DistributedOptimizer(torch.optim.SGD(m2.parameters(), lr=0.1), m2, loss_scale=64, verbose=False))
    except ValueError as e:
        errors.append(str(e))
    try:
        opt.set_loss_scale(64)
    except ValueError as e:
        errors.append(str(e))
    m3 = make_model()
    off = dear.GradScaler(dear.DistributedOptimizer(torch.optim.SGD(m3.parameters(), lr=0.1), m3, verbose=False), enabled=False)
    x = torch.ones(())
    return (sd, ts_sd, back.state_dict(), errors, off.state_dict(), off.get_scale(), off.is_enabled(),
            off.scale(x) is x, scaler.is_enabled())


def test_state_dict_round_trip_with_torch_grad_scaler_and_argument_checks():
    sd, ts_sd, back, errors, off_sd, off_scale, off_en, off_same, en = run_ranks(_state_dict_worker, world=1, backend="emu")[0]
    # steps 0..4, overflow at 1: 1024 -> 1024 (t=1) -> 512 -> 512 -> 512 -> 1024 (three clean steps)
    assert sd == {"scale": 1024.0, "growth_factor": 2.0, "backoff_factor": 0.5, "growth_interval": GI, "_growth_tracker": 0}
    assert ts_sd == sd
    assert back == dict(sd, scale=3.0)
    assert len(errors) == 3 and "DistributedOptimizer" in errors[0] and "static" in errors[1] and "GradScaler" in errors[2]
    assert off_sd == {} and off_scale == 1.0 and not off_en and off_same and en


# ---- single rank, fp32, static loss scale: the fp32 direct pack applies 1/S ----------------------------------------------
def _static_worker(rank, world, scale):
    import dear_pytorch_b200 as dear
    m = make_model(); m.eval()
    opt = dear.DistributedOptimizer(torch.optim.SGD(m.parameters(), lr=0.05, momentum=0.9), m, threshold=0.001,
                                    loss_scale=scale, verbose=False)
    for t in range(2):
        x, y = data(t, 4)
        opt.zero_grad()
        (F.cross_entropy(m(x), y) * scale).backward()
        opt.step()
    opt.synchronize()
    return [p.detach().clone() for p in m.parameters()]


def test_single_rank_static_loss_scale_with_fp32_parameters():
    m = make_model(); m.eval()
    opt = torch.optim.SGD(m.parameters(), lr=0.05, momentum=0.9)
    for t in range(2):
        x, y = data(t, 4)
        opt.zero_grad()
        F.cross_entropy(m(x), y).backward()
        opt.step()
    for a, b in zip(run_ranks(_static_worker, world=1, backend="emu", args=(64.0,))[0], m.parameters()):
        torch.testing.assert_close(a, b.detach(), rtol=2e-5, atol=2e-6)


# ---- the MNIST example's mixed-precision loop with the dynamic scaler ------------------------------------------------------
def _mnist_worker(rank, world):
    sys.path.insert(0, os.path.join(ROOT, "examples", "mnist"))
    import pytorch_mnist
    return pytorch_mnist.main(["--no-cuda", "--epochs", "2", "--train-size", "1500", "--test-size", "400", "--batch-size", "50",
                               "--log-interval", "1000", "--lr", "0.05", "--use-mixed-precision"])


@pytest.mark.parametrize("backend", ["gloo", "emu"])
def test_mnist_mixed_precision_with_dynamic_scaler_learns(backend):
    (l0, a0), (l1, a1) = run_ranks(_mnist_worker, world=2, backend=backend, timeout=400)
    assert abs(l0 - l1) < 1e-6 and abs(a0 - a1) < 1e-6
    assert a0 > 0.7, "accuracy %.3f: the run with dynamic loss scaling did not learn" % a0


# ---- on the H100: the sm_90a kernels (ranks share one GPU through CUDA IPC when the box has only one) ---------------------
GPU_ENV = {"DEAR_SPIN_TIMEOUT_S": "15"}


def _gpu_world():
    return 2 if torch.cuda.device_count() in (1, 2, 4, 8) else 1


def _gpu_worker(rank, world, kw):
    """scaler_worker on cuda, optionally under fp16 autocast or with a .half() model (fp32 masters)."""
    autocast, half = kw.pop("autocast", False), kw.pop("half", False)
    if autocast or half:
        import contextlib
        orig_make, orig_fwd = make_model, nn.Sequential.forward
        def fwd(self, x):
            ctx = torch.autocast("cuda", dtype=torch.float16) if autocast and x.is_cuda else contextlib.nullcontext()
            with ctx:
                return orig_fwd(self, x.half() if half else x).float()
        globals()["make_model"] = (lambda: orig_make().half()) if half else orig_make
        nn.Sequential.forward = fwd
    return scaler_worker(rank, world, **kw)


def _torch_cuda_reference_worker(rank, world, kind, steps, n, poison):
    """torch.optim + torch.amp.GradScaler under fp16 autocast on the GPU, one process, the whole batch."""
    m = make_model().cuda(); m.eval()
    opt = _make_opt(kind, m.parameters())
    sc = torch.amp.GradScaler("cuda", init_scale=INIT, growth_interval=GI)
    st = {"t": 0}
    list(m.parameters())[POISON_PARAM].register_hook(_poison_hook(st, poison))
    scales, trackers = [], []
    for t in range(steps):
        st["t"] = t
        x, y = data(t, n)
        opt.zero_grad()
        with torch.autocast("cuda", dtype=torch.float16):
            out = m(x.cuda())
        sc.scale(F.cross_entropy(out.float(), y.cuda())).backward()
        sc.step(opt)
        sc.update()
        scales.append(sc.get_scale())
        trackers.append(sc._get_growth_tracker())
    return ([p.detach().cpu().clone() for p in m.parameters()],
            {i: {k: v.float().cpu() for k, v in s.items() if torch.is_tensor(v)} for i, s in opt.state_dict()["state"].items()},
            scales, trackers, [])


@pytest.mark.gpu
@pytest.mark.parametrize("algo,world,kind", [("oneshot", 1, "sgd"), ("oneshot", 1, "adamw"), ("oneshot", 2, "sgd-nesterov"),
                                             ("pipe", 2, "adam"), ("nvls", 2, "sgd")])
def test_gpu_injected_overflow_matches_torch_grad_scaler(algo, world, kind):
    """Each Kernel A variant (one GPU: the direct fp32 pack) against torch.optim + torch.amp.GradScaler."""
    if world > _gpu_world():
        pytest.skip("needs ranks sharing a GPU")
    if algo == "nvls" and torch.cuda.device_count() < 2:
        pytest.skip("NVLS multicast needs at least 2 GPUs")
    ref = reference(kind, STEPS, N, POISON)
    outs = run_ranks(_gpu_worker, world=world, backend="b200", args=(dict(kind=kind, steps=STEPS, n=N, poison=POISON),),
                     extra_env=dict(GPU_ENV, DEAR_RS_ALGO=algo, DEAR_MULTICAST="1" if algo == "nvls" else "0"), timeout=300)
    _check(outs, ref, rtol=1e-4, atol=1e-5)


@pytest.mark.gpu
def test_gpu_fp16_autocast_with_fp32_parameters():
    world = _gpu_world()
    ref = run_ranks(_torch_cuda_reference_worker, world=1, backend="b200", args=("sgd", STEPS, N, POISON), extra_env=GPU_ENV,
                    timeout=300)[0]
    outs = run_ranks(_gpu_worker, world=world, backend="b200",
                     args=(dict(kind="sgd", steps=STEPS, n=N, poison=POISON, autocast=True),), extra_env=GPU_ENV, timeout=300)
    _check(outs, ref, rtol=1e-2, atol=2e-3)          # fp16 products over a different batch split; the scale sequence is exact


@pytest.mark.gpu
def test_gpu_half_model_with_fp32_masters_matches_the_emulation():
    """torch's GradScaler refuses fp16 gradients: the reference is the same run on the host emulation (tied to torch above).
    SGD: its update is linear in the gradient, so the fp16 rounding differences of GPU and host kernels stay small."""
    world = _gpu_world()
    kw = dict(kind="sgd", steps=STEPS, n=N, poison=POISON, half=True)
    emu = run_ranks(_gpu_worker, world=world, backend="emu", args=(dict(kw),), timeout=300)
    outs = run_ranks(_gpu_worker, world=world, backend="b200", args=(dict(kw),), extra_env=GPU_ENV, timeout=300)
    params, state, scales, trackers, _, _ = emu[0]
    assert scales[:2] == [INIT / 2, INIT / 4]
    _check(outs, (params, state, scales, trackers, []), rtol=1e-2, atol=2e-3)


@pytest.mark.gpu
def test_gpu_mixed_dtype_model_skips_every_bucket_set_together():
    poison = {2: INF, 3: NAN}
    _check_mixed(run_ranks(_mixed_worker, world=_gpu_world(), backend="b200", args=(poison, 6), extra_env=GPU_ENV,
                           timeout=300), poison, 6)


def _graph_worker(rank, world, use_graph, rotated, steps, poison):
    import dear_pytorch_b200 as dear
    dev = dear.device()
    m = make_model().to(dev); m.eval()
    opt = dear.DistributedOptimizer(_make_opt("sgd", m.parameters()), m, threshold=0.001, verbose=False)
    dear.broadcast_parameters(m.state_dict(), 0)
    scaler = dear.GradScaler(opt, init_scale=INIT, growth_interval=GI)
    poison_t = torch.ones((), device=dev)          # multiplied into the loss: changed between replays
    step = dear.TrainStep(m, opt, lambda out, y: F.cross_entropy(out, y) * poison_t, use_graph=use_graph, graph_warmup=2,
                          overlap_update=rotated, scaler=scaler)
    per = N // world
    for t in range(steps):
        poison_t.fill_(poison.get(t, 1.0))
        x, y = data(t, N)
        step(x[rank * per:(rank + 1) * per].to(dev), y[rank * per:(rank + 1) * per].to(dev))
    opt.synchronize()
    dear.communicator().check_status()
    return [p.detach().cpu().clone() for p in m.parameters()], scaler.get_scale(), step.eager_calls


@pytest.mark.gpu
@pytest.mark.parametrize("rotated", [False, True])
def test_gpu_cuda_graph_replays_match_the_eager_run(rotated):
    world, steps = _gpu_world(), 10
    poison = {1: INF, 5: NAN, 8: INF}               # an overflow during warm-up and two inside replays
    eager = run_ranks(_graph_worker, world=world, backend="b200", args=(False, rotated, steps, poison), extra_env=GPU_ENV,
                      timeout=300)
    graph = run_ranks(_graph_worker, world=world, backend="b200", args=(True, rotated, steps, poison), extra_env=GPU_ENV,
                      timeout=300)
    for (pe, se, _), (pg, sg, calls) in zip(eager, graph):
        assert calls < steps                        # the graph was replayed
        assert se == sg
        for a, b in zip(pe, pg):
            torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6)


# ---- resuming from a checkpoint with a scaler attached --------------------------------------------------------------------
RESUME_AT, RESUME_STEPS = 3, 5
RESUME_POISON = {RESUME_AT: INF, RESUME_AT + 3: NAN}      # the first step after the resume overflows


def _resume_reference(kind):
    """torch: RESUME_AT plain steps, checkpoint, then GradScaler steps (the same poison)."""
    import copy
    m = make_model(); m.eval()
    opt = _make_opt(kind, m.parameters())
    for t in range(RESUME_AT):
        x, y = data(t, N)
        opt.zero_grad()
        F.cross_entropy(m(x), y).backward()
        opt.step()
    ckpt = (copy.deepcopy(m.state_dict()), copy.deepcopy(opt.state_dict()))
    sc = torch.amp.GradScaler("cpu", init_scale=INIT, growth_interval=GI)
    st = {"t": 0}
    list(m.parameters())[POISON_PARAM].register_hook(_poison_hook(st, RESUME_POISON))
    scales, trackers = [], []
    for t in range(RESUME_AT, RESUME_AT + RESUME_STEPS):
        st["t"] = t
        x, y = data(t, N)
        opt.zero_grad()
        sc.scale(F.cross_entropy(m(x), y)).backward()
        sc.step(opt)
        sc.update()
        scales.append(sc.get_scale())
        trackers.append(sc._get_growth_tracker())
    return ckpt, ([p.detach().clone() for p in m.parameters()], opt.state_dict()["state"], scales, trackers, [])


def _resume_worker(rank, world, kind, ckpt):
    """The usual resume order: build the optimizer and the scaler, then load the checkpoint; re-bucket right after the
    overflowing first step (before the first applied update)."""
    import dear_pytorch_b200 as dear
    msd, osd = ckpt
    m = make_model(); m.load_state_dict(msd); m.eval()
    opt = dear.DistributedOptimizer(_make_opt(kind, m.parameters()), m, threshold=0.001, verbose=False)
    scaler = dear.GradScaler(opt, init_scale=INIT, growth_interval=GI)
    opt.load_state_dict(osd)
    st = {"t": 0, "rank": rank}
    list(m.parameters())[POISON_PARAM].register_hook(_poison_hook(st, RESUME_POISON, rank=world - 1))
    per = N // world
    scales, trackers = [], []
    for t in range(RESUME_AT, RESUME_AT + RESUME_STEPS):
        if t == RESUME_AT + 1:
            opt.engine.rebucket(("threshold", 0.05))
        st["t"] = t
        x, y = data(t, N)
        opt.zero_grad()
        scaler.scale(F.cross_entropy(m(x[rank * per:(rank + 1) * per]), y[rank * per:(rank + 1) * per])).backward()
        scaler.step(opt)
        scaler.update()
        scales.append(scaler.get_scale())
        trackers.append(scaler._get_growth_tracker())
    sd = opt.state_dict()
    state = {i: {k: v.float() for k, v in s.items() if torch.is_tensor(v) and k != "master_param"} for i, s in sd["state"].items()}
    return ([p.detach().clone() for p in m.parameters()], state, scales, trackers, [], scaler.get_scale()), \
        sd["dear"]["num_updates"]


@pytest.mark.parametrize("backend,world", [("emu", 1), ("emu", 2), ("gloo", 1), ("gloo", 2)])
@pytest.mark.parametrize("kind", ["adam", "sgd"])
def test_resume_with_a_scaler_keeps_the_step_count(backend, world, kind):
    ckpt, ref = _resume_reference(kind)
    applied = RESUME_AT + RESUME_STEPS - len(RESUME_POISON)
    if kind == "adam":
        assert all(int(e["step"]) == applied for e in ref[1].values())
    outs = run_ranks(_resume_worker, world=world, backend=backend, args=(kind, ckpt))
    _check([o for o, _ in outs], ref)
    if kind == "sgd":             # a stock torch.optim.SGD state carries no step count: momentum buffers count as one
        applied = 1 + RESUME_STEPS - len(RESUME_POISON)
    assert all(n == applied for _, n in outs)          # the checkpoint metadata counts applied updates only


def _new_scale_worker(rank, world, steps, poison, new_scale_at):
    import dear_pytorch_b200 as dear
    m = make_model(); m.eval()
    opt = dear.DistributedOptimizer(torch.optim.SGD(m.parameters(), lr=0.05), m, verbose=False)
    scaler = dear.GradScaler(opt, init_scale=INIT, growth_interval=GI)
    st = {"t": 0, "rank": rank}
    list(m.parameters())[POISON_PARAM].register_hook(_poison_hook(st, poison))
    seq = []
    for t in range(steps):
        st["t"] = t
        x, y = data(t, 4)
        scaler.scale(F.cross_entropy(m(x), y)).backward()
        scaler.step(opt)
        scaler.update(new_scale=new_scale_at.get(t))
        seq.append((scaler.get_scale(), scaler._get_growth_tracker()))
    m2 = make_model()
    off = dear.GradScaler(dear.DistributedOptimizer(torch.optim.SGD(m2.parameters(), lr=0.1), m2, verbose=False),
                          growth_factor=3.0, backoff_factor=0.25, growth_interval=7, enabled=False)
    return seq, (off.get_growth_factor(), off.get_backoff_factor(), off.get_growth_interval())


def test_update_with_new_scale_matches_torch_and_disabled_getters():
    steps, poison, new_scale_at = 8, {1: INF, 5: NAN}, {2: 100.0, 5: 8.0}
    m = make_model(); m.eval()
    opt = torch.optim.SGD(m.parameters(), lr=0.05)
    sc = torch.amp.GradScaler("cpu", init_scale=INIT, growth_interval=GI)
    st = {"t": 0}
    list(m.parameters())[POISON_PARAM].register_hook(_poison_hook(st, poison))
    ref = []
    for t in range(steps):
        st["t"] = t
        x, y = data(t, 4)
        sc.scale(F.cross_entropy(m(x), y)).backward()
        sc.step(opt)
        opt.zero_grad()
        sc.update(new_scale=new_scale_at.get(t))
        ref.append((sc.get_scale(), sc._get_growth_tracker()))
    seq, getters = run_ranks(_new_scale_worker, world=1, backend="emu", args=(steps, poison, new_scale_at))[0]
    assert seq == ref
    assert getters == (3.0, 0.25, 7)             # a disabled scaler reports its constructor arguments


# ---- on the H100: one GPU (direct 16-bit widening pack) and three ranks (generic-world kernels) -------------------------------
def _shared_gpu_world_ok(world):
    return world == 1 or torch.cuda.device_count() in (1, world) or torch.cuda.device_count() >= 8


@pytest.mark.gpu
@pytest.mark.parametrize("world", [1, 3])
def test_gpu_half_model_one_gpu_and_three_ranks_match_the_emulation(world):
    if not _shared_gpu_world_ok(world):
        pytest.skip("ranks cannot share the GPUs evenly")
    kw = dict(kind="sgd", steps=STEPS, n=N, poison=POISON, half=True)
    emu = run_ranks(_gpu_worker, world=world, backend="emu", args=(dict(kw),), timeout=300)
    outs = run_ranks(_gpu_worker, world=world, backend="b200", args=(dict(kw),), extra_env=GPU_ENV, timeout=300)
    params, state, scales, trackers, _, _ = emu[0]
    assert scales[:2] == [INIT / 2, INIT / 4]
    _check(outs, (params, state, scales, trackers, []), rtol=1e-2, atol=2e-3)


@pytest.mark.gpu
def test_gpu_three_ranks_fp32_match_torch_grad_scaler():
    if not _shared_gpu_world_ok(3):
        pytest.skip("ranks cannot share the GPUs evenly")
    ref = reference("adamw", STEPS, N, POISON)
    outs = run_ranks(_gpu_worker, world=3, backend="b200", args=(dict(kind="adamw", steps=STEPS, n=N, poison=POISON),),
                     extra_env=GPU_ENV, timeout=300)
    _check(outs, ref, rtol=1e-4, atol=1e-5)
