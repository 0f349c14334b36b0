"""Sharded torch.optim.RMSprop fused into the update kernel (Kernel B), against single-process torch.optim.RMSprop.

CPU: the host emulation (``emu``, the kernels' per-element math) and ``gloo`` (eager torch ops) at worlds 1-3: the option
matrix, absent gradients, composition with the scaler / clipping / 16-bit wire / 16-bit parameters / TrainStep /
accumulation / re-bucketing, checkpoints in torch's layout, rejections.  Bucket level: ``BucketSet`` driven directly and
Kernel B's result compared with a float64 RMSprop with an error bound derived from the magnitudes of the terms; every
RMSprop instantiation of ``ag_kernel`` reachable at worlds 1-4 (and 8 with eight GPUs) is run.
GPU: the same bucket matrix on the CUDA kernels, a small fp32 CNN end to end, and CUDA-graph replay against the eager
run."""
import collections
import copy
import hashlib

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from _mp import run_ranks
from test_dear_equivalence import data, make_model
from test_grad_comm_dtype import _WithSpare, _check, _kw_worker, reference as wire_reference
from test_kernel_matrix import (ALGO_ENV, CODE, DTS, ES, TORCH_DT, U, _bits, _gpu_world_ok, _within, make_grad,
                                std_layout, wide_layout)

ENV = {"DEAR_SPIN_TIMEOUT_S": "15"}
OPT_RMSPROP, HYPER_SKIP, HYPER_CENTERED = 3, 2, 4

# rtol / atol of test_adam.py
RTOL, ATOL = 1e-4, 2e-6


def make_opt(kind, params_or_model, kw=None):
    """RMSprop over two parameter groups with different hyper-parameters: the convolutions (kw) and the rest (the
    other centered setting, its own momentum / weight decay)."""
    m = params_or_model
    kw = dict(kw or dict(lr=1e-3, alpha=0.9, momentum=0.5, centered=True))
    named = list(m.named_parameters())
    first = [p for n, p in named if n.startswith("0.") or n.startswith("a.")]
    rest = [p for n, p in named if not (n.startswith("0.") or n.startswith("a."))]
    other = dict(lr=kw["lr"] * 0.7, alpha=kw.get("alpha", 0.99), centered=not kw.get("centered", False),
                 momentum=0.0 if kw.get("momentum", 0.0) else 0.9, weight_decay=0.0 if kw.get("weight_decay", 0.0) else 1e-2)
    groups = [dict(params=first, **kw), dict(params=rest, **other)]
    return torch.optim.RMSprop([g for g in groups if g["params"]], lr=kw["lr"])


# ------------------------------------------------------------------------------------------------ 1. option matrix
OPTIONS = [dict(lr=1e-3, alpha=alpha, centered=c, momentum=m, weight_decay=wd)
           for alpha in (0.99, 0.4) for c in (False, True) for m in (0.0, 0.9) for wd in (0.0, 1e-2)]


def _reference(kw, steps, world, per):
    model = make_model(); model.eval()
    opt = make_opt("rmsprop", model, kw)
    for t in range(steps):
        x, y = data(t, world * per)
        opt.zero_grad()
        F.cross_entropy(model(x), y).backward()
        opt.step()
    return [p.detach().clone() for p in model.parameters()], opt.state_dict()


def _matrix_worker(rank, world, cases, steps, per):
    import dear_pytorch_b200 as dear
    out = []
    for kw in cases:
        model = make_model(); model.eval()
        opt = dear.DistributedOptimizer(make_opt("rmsprop", model, kw), model, threshold=0.002, verbose=False)
        dear.broadcast_parameters(model.state_dict(), 0)
        for t in range(steps):
            x, y = data(t, world * per)
            opt.zero_grad()
            F.cross_entropy(model(x[rank * per:(rank + 1) * per]), y[rank * per:(rank + 1) * per]).backward()
            opt.step()
        opt.synchronize()
        assert len(opt.engine.plan.buckets) > 1
        out.append([p.detach().clone() for p in model.parameters()])
        opt.engine.close()
    return out


@pytest.mark.parametrize("backend", ["emu", "gloo"])
@pytest.mark.parametrize("world", [1, 2, 3])
def test_option_matrix_matches_torch(backend, world):
    steps, per = 4, 2
    refs = [_reference(kw, steps, world, per)[0] for kw in OPTIONS]
    outs = run_ranks(_matrix_worker, world=world, backend=backend, args=(OPTIONS, steps, per), timeout=600)
    for r, res in enumerate(outs):
        for kw, params, ref in zip(OPTIONS, res, refs):
            for a, b in zip(params, ref):
                torch.testing.assert_close(a, b, rtol=RTOL, atol=ATOL, msg=lambda m: "rank %d %s: %s" % (r, kw, m))
    for a, b in zip(outs[0], outs[-1]):
        assert all(torch.equal(x, y) for x, y in zip(a, b))        # replicas are bit-identical


# ------------------------------------------------------------------------------------------------ 2. absent gradients
class _Branchy(nn.Module):
    """``side`` only runs on every third step: torch leaves it (and its state) alone otherwise."""

    def __init__(self):
        super().__init__()
        torch.manual_seed(3)
        self.a, self.side, self.b = nn.Linear(10, 16), nn.Linear(16, 16), nn.Linear(16, 4)

    def forward(self, x, use_side):
        h = torch.tanh(self.a(x))
        if use_side:
            h = h + torch.relu(self.side(h))
        return self.b(h)


BRANCHY_KW = dict(lr=1e-2, alpha=0.9, momentum=0.5, centered=True, weight_decay=1e-2)


def _branchy_data(t, n):
    g = torch.Generator().manual_seed(900 + t)
    return torch.randn(n, 10, generator=g), torch.randint(0, 4, (n,), generator=g)


def _branchy_reference(steps, n):
    m = _Branchy()
    opt = make_opt("rmsprop", m, BRANCHY_KW)
    for t in range(steps):
        x, y = _branchy_data(t, n)
        opt.zero_grad()
        F.cross_entropy(m(x, t % 3 == 2), y).backward()
        opt.step()
    return [p.detach().clone() for p in m.parameters()], opt.state_dict()


def _branchy_worker(rank, world, steps, per, reload_at):
    import dear_pytorch_b200 as dear
    m = _Branchy()
    opt = dear.DistributedOptimizer(make_opt("rmsprop", m, BRANCHY_KW), m, threshold=0.0005, verbose=False)
    dear.broadcast_parameters(m.state_dict(), 0)
    for t in range(steps):
        x, y = _branchy_data(t, world * per)
        opt.zero_grad()
        F.cross_entropy(m(x[rank * per:(rank + 1) * per], t % 3 == 2), y[rank * per:(rank + 1) * per]).backward()
        opt.step()
        if t == reload_at:
            opt.load_state_dict(opt.state_dict())
    opt.synchronize()
    return [p.detach().clone() for p in m.parameters()], opt.state_dict()


def _steps(sd):
    return {int(i): int(float(e["step"])) for i, e in sd["state"].items()}


@pytest.mark.parametrize("backend", ["emu", "gloo"])
@pytest.mark.parametrize("world", [1, 2, 3])
def test_absent_gradients_and_per_parameter_steps(backend, world):
    steps, per = 7, 2
    ref, ref_sd = _branchy_reference(steps, world * per)
    assert sorted(set(_steps(ref_sd).values())) == [2, 7]
    for reload_at in (-1, 1, 3):                     # 1: before `side` ever had a gradient (no entry for it)
        for params, sd in run_ranks(_branchy_worker, world=world, backend=backend, args=(steps, per, reload_at)):
            for a, b in zip(params, ref):
                torch.testing.assert_close(a, b, rtol=RTOL, atol=ATOL)
            assert _steps(sd) == _steps(ref_sd)


# ------------------------------------------------------------------------------------------------ 3. composition
def _wire_opt(kind, m):
    # (test_grad_comm_dtype's model: `spare` never runs; two groups, centered and plain)
    if kind == "rmsprop-plain":
        return make_opt(kind, m, dict(lr=1e-3, alpha=0.99, momentum=0.0, centered=False))
    return make_opt(kind, m, dict(lr=1e-3, alpha=0.9, momentum=0.9, centered=True, weight_decay=1e-2))


STEPS, N = 5, 6


@pytest.mark.parametrize("kind", ["rmsprop", "rmsprop-plain"])
def test_bf16_wire_matches_the_rounded_reference(kind):
    ref = wire_reference(kind, STEPS, N, 2, "bf16", make_opt=_wire_opt)
    _check(run_ranks(_kw_worker, world=2, backend="emu",
                     args=(dict(kind=kind, wire="bf16", steps=STEPS, n=N, make_opt=_wire_opt),)), ref, rtol=RTOL, atol=ATOL)


@pytest.mark.parametrize("backend", ["emu", "gloo"])
def test_norm_clip_that_bites(backend):
    ref = wire_reference("rmsprop", STEPS, N, 2, None, clip=0.05, make_opt=_wire_opt)
    assert max(ref[1]) > 0.05
    _check(run_ranks(_kw_worker, world=2, backend=backend,
                     args=(dict(kind="rmsprop", wire=None, steps=STEPS, n=N, clip=0.05, make_opt=_wire_opt),)), ref,
           rtol=RTOL, atol=ATOL)


def test_gradient_accumulation():
    ref = wire_reference("rmsprop", 4, 4, 2, None, passes=2, make_opt=_wire_opt)
    _check(run_ranks(_kw_worker, world=2, backend="emu",
                     args=(dict(kind="rmsprop", wire=None, steps=4, n=4, passes=2, make_opt=_wire_opt),)), ref,
           rtol=RTOL, atol=ATOL)


@pytest.mark.parametrize("world", [2, 3])
def test_rebucket_mid_run(world):
    ref = wire_reference("rmsprop", STEPS, N, world, None, make_opt=_wire_opt)
    _check(run_ranks(_kw_worker, world=world, backend="emu",
                     args=(dict(kind="rmsprop", wire=None, steps=STEPS, n=N, rebucket_at=2, make_opt=_wire_opt),)), ref,
           rtol=RTOL, atol=ATOL)


def _scaler_worker(rank, world, steps, per, poison):
    import dear_pytorch_b200 as dear
    m = make_model(); m.eval()
    opt = dear.DistributedOptimizer(make_opt("rmsprop", m), m, threshold=0.002, verbose=False)
    dear.broadcast_parameters(m.state_dict(), 0)
    scaler = dear.GradScaler(opt, init_scale=2.0 ** 8, growth_interval=2)
    snaps = []
    for t in range(steps):
        x, y = data(t, world * per)
        loss = F.cross_entropy(m(x[rank * per:(rank + 1) * per]), y[rank * per:(rank + 1) * per])
        if t == poison and rank == world - 1:
            loss = loss * float("inf")
        scaler.scale(loss).backward()
        before = copy.deepcopy(opt.state_dict()) if t == poison else None
        scaler.step(opt)
        scaler.update()
        if before is not None:
            after = opt.state_dict()
            assert _same_state(before, after), "the skipped step moved the optimizer state"
        snaps.append(scaler.get_scale())
    opt.synchronize()
    return [p.detach().clone() for p in m.parameters()], snaps, opt.state_dict()


def _same_state(a, b):
    if a["state"].keys() != b["state"].keys():
        return False
    return all(a["state"][i].keys() == b["state"][i].keys() and
               all(torch.equal(a["state"][i][k], b["state"][i][k]) for k in a["state"][i]) for i in a["state"])


@pytest.mark.parametrize("backend", ["emu", "gloo"])
def test_grad_scaler_skip_leaves_every_shard_untouched(backend):
    world, per, steps, poison = 2, 2, 5, 2
    m = make_model(); m.eval()
    opt = make_opt("rmsprop", m)
    for t in range(steps):
        if t == poison:
            continue                                  # torch: the skipped step applies nothing
        x, y = data(t, world * per)
        opt.zero_grad()
        F.cross_entropy(m(x), y).backward()
        opt.step()
    ref = [p.detach().clone() for p in m.parameters()]
    for params, scales, sd in run_ranks(_scaler_worker, world=world, backend=backend, args=(steps, per, poison)):
        for a, b in zip(params, ref):
            torch.testing.assert_close(a, b, rtol=RTOL, atol=ATOL)
        assert scales[poison] == scales[poison - 1] * 0.5
        assert set(_steps(sd).values()) == {steps - 1}


class _Bf16Mlp(nn.Module):
    def __init__(self):
        super().__init__()
        torch.manual_seed(5)
        self.a, self.b = nn.Linear(12, 24), nn.Linear(24, 5)

    def forward(self, x):
        return self.b(torch.tanh(self.a(x)))


def _bf16_data(t, n):
    g = torch.Generator().manual_seed(400 + t)
    return torch.randn(n, 12, generator=g), torch.randint(0, 5, (n,), generator=g)


def _bf16_worker(rank, world, steps, per):
    import dear_pytorch_b200 as dear
    dev = dear.device()
    m = _Bf16Mlp().to(dev).to(torch.bfloat16)
    opt = dear.DistributedOptimizer(make_opt("rmsprop", m), m, threshold=0.0005, verbose=False)
    dear.broadcast_parameters(m.state_dict(), 0)
    for t in range(steps):
        x, y = _bf16_data(t, world * per)
        x, y = x[rank * per:(rank + 1) * per].to(dev, torch.bfloat16), y[rank * per:(rank + 1) * per].to(dev)
        opt.zero_grad()
        F.cross_entropy(m(x).float(), y).backward()
        opt.step()
    opt.synchronize()
    sd = opt.state_dict()
    masters = [sd["state"][i]["master_param"].float().cpu() for i in sorted(sd["state"])]
    return [p.detach().cpu().clone() for p in m.parameters()], masters


def _bf16_reference(world, steps, per):
    """fp32 master weights under torch.optim.RMSprop, the forward in bf16 from the rounded masters; the gradients are
    the bf16 ones averaged in fp32."""
    m = _Bf16Mlp().to(torch.bfloat16)
    master = _Bf16Mlp()
    with torch.no_grad():
        for p, q in zip(master.parameters(), m.parameters()):
            p.copy_(q.float())
    opt = make_opt("rmsprop", master)
    for t in range(steps):
        x, y = _bf16_data(t, world * per)
        acc = [torch.zeros_like(p) for p in master.parameters()]
        for r in range(world):
            m.zero_grad()
            F.cross_entropy(m(x[r * per:(r + 1) * per].to(torch.bfloat16)).float(), y[r * per:(r + 1) * per]).backward()
            for a, p in zip(acc, m.parameters()):
                a += p.grad.float()
        for a, p in zip(acc, master.parameters()):
            p.grad = a * (torch.tensor(1.0) / world)
        opt.step()
        with torch.no_grad():
            for p, q in zip(master.parameters(), m.parameters()):
                q.copy_(p.to(torch.bfloat16))
    return [p.detach().clone() for p in m.parameters()], [p.detach().clone() for p in master.parameters()]


@pytest.mark.parametrize("backend", ["emu", "gloo"])
def test_bf16_parameters_with_fp32_masters(backend):
    world, steps, per = 2, 4, 3
    ref_p, ref_m = _bf16_reference(world, steps, per)
    for params, masters in run_ranks(_bf16_worker, world=world, backend=backend, args=(steps, per)):
        for p, w in zip(params, masters):
            assert torch.equal(p, w.reshape(p.shape).to(torch.bfloat16))     # 16-bit parameters == rounded master
        for a, b in zip(masters, ref_m):
            torch.testing.assert_close(a.reshape(b.shape), b, rtol=2e-3, atol=1e-4)


def _sched_worker(rank, world, rotated, steps, per):
    import dear_pytorch_b200 as dear
    m = make_model(); m.eval()
    opt = dear.DistributedOptimizer(make_opt("rmsprop", m), m, threshold=0.002, verbose=False)
    dear.broadcast_parameters(m.state_dict(), 0)
    sched = torch.optim.lr_scheduler.StepLR(opt, step_size=1, gamma=0.7)
    step = dear.TrainStep(m, opt, F.cross_entropy, overlap_update=rotated)
    for t in range(steps):
        x, y = data(t, world * per)
        step(x[rank * per:(rank + 1) * per], y[rank * per:(rank + 1) * per])
        sched.step()
    opt.synchronize()
    return [p.detach().clone() for p in m.parameters()]


@pytest.mark.parametrize("backend", ["emu", "gloo"])
@pytest.mark.parametrize("rotated", [False, True])
def test_train_step_with_a_per_step_lr_schedule(backend, rotated):
    world, per, steps = 2, 2, 5
    m = make_model(); m.eval()
    opt = make_opt("rmsprop", m)
    sched = torch.optim.lr_scheduler.StepLR(opt, step_size=1, gamma=0.7)
    for t in range(steps):
        x, y = data(t, world * per)
        opt.zero_grad()
        F.cross_entropy(m(x), y).backward()
        opt.step()
        sched.step()
    ref = [p.detach().clone() for p in m.parameters()]
    for params in run_ranks(_sched_worker, world=world, backend=backend, args=(rotated, steps, per)):
        for a, b in zip(params, ref):
            torch.testing.assert_close(a, b, rtol=RTOL, atol=ATOL)


# ------------------------------------------------------------------------------------------------ 4. checkpoints
def _keys_ok(sd, opt):
    """torch.optim.RMSprop's layout: step + square_avg, momentum_buffer iff momentum > 0, grad_avg iff centered."""
    group = {}
    for g in sd["param_groups"]:
        for i in g["params"]:
            group[i] = g
    for i, e in sd["state"].items():
        g = group[int(i)]
        want = {"step", "square_avg"} | ({"momentum_buffer"} if g["momentum"] > 0 else set()) | \
            ({"grad_avg"} if g["centered"] else set())
        assert set(e) - {"master_param"} == want, (i, sorted(e), g)
        assert e["step"].dim() == 0 and e["step"].dtype == torch.float32


def _ckpt_worker(rank, world, steps, per, mode, sd_in, threshold):
    import dear_pytorch_b200 as dear
    m = make_model(); m.eval()
    opt = dear.DistributedOptimizer(make_opt("rmsprop", m), m, threshold=threshold, verbose=False)
    if sd_in is not None:
        msd, osd = sd_in
        m.load_state_dict(msd)
        opt.load_state_dict(osd)
    dear.broadcast_parameters(m.state_dict(), 0)
    t0 = 0 if mode == "first" else steps
    for t in range(t0, t0 + steps):
        x, y = data(t, world * per)
        opt.zero_grad()
        F.cross_entropy(m(x[rank * per:(rank + 1) * per]), y[rank * per:(rank + 1) * per]).backward()
        opt.step()
    opt.synchronize()
    return {k: v.clone() for k, v in m.state_dict().items()}, opt.state_dict()


def _torch_run(msd, osd, t0, steps, n):
    m = make_model(); m.eval()
    opt = make_opt("rmsprop", m)
    if msd is not None:
        m.load_state_dict(msd)
        opt.load_state_dict(osd)
    for t in range(t0, t0 + steps):
        x, y = data(t, n)
        opt.zero_grad()
        F.cross_entropy(m(x), y).backward()
        opt.step()
    return {k: v.clone() for k, v in m.state_dict().items()}, opt.state_dict()


def _strip(sd):
    return {"state": {int(i): {k: v.clone() for k, v in e.items() if k != "master_param"} for i, e in sd["state"].items()},
            "param_groups": copy.deepcopy(sd["param_groups"])}


def _close_state(a, b):
    assert sorted(a["state"]) == sorted(b["state"])
    for i in a["state"]:
        assert set(a["state"][i]) == set(b["state"][i])
        for k in a["state"][i]:
            torch.testing.assert_close(a["state"][i][k], b["state"][i][k], rtol=RTOL, atol=ATOL)


@pytest.mark.parametrize("backend", ["emu", "gloo"])
def test_checkpoint_round_trips_with_stock_torch(backend):
    world, per, steps = 2, 2, 3
    n = world * per
    # DeAR -> torch.optim.RMSprop: both continue identically
    (msd, osd), _ = run_ranks(_ckpt_worker, world=world, backend=backend, args=(steps, per, "first", None, 0.002))
    _keys_ok(osd, None)
    ref_first = _torch_run(None, None, 0, steps, n)
    _close_state(_strip(osd), _strip(ref_first[1]))
    cont_torch = _torch_run(msd, _strip(osd), steps, steps, n)
    for (m2, o2) in run_ranks(_ckpt_worker, world=world, backend=backend, args=(steps, per, "second", (msd, osd), 0.002)):
        for k in m2:
            torch.testing.assert_close(m2[k], cont_torch[0][k], rtol=RTOL, atol=ATOL)
        _close_state(_strip(o2), _strip(cont_torch[1]))
    # torch.optim.RMSprop -> DeAR, into another world size and bucket policy
    tm, to = ref_first
    cont_torch2 = _torch_run(tm, copy.deepcopy(to), steps, steps, n)     # (torch's load_state_dict aliases the tensors)
    for w2, thr in ((1, 25), (3, 0.001)):
        per2 = n // w2 if n % w2 == 0 else None
        if per2 is None:
            continue
        for (m2, o2) in run_ranks(_ckpt_worker, world=w2, backend=backend, args=(steps, per2, "second", (tm, to), thr)):
            for k in m2:
                torch.testing.assert_close(m2[k], cont_torch2[0][k], rtol=RTOL, atol=ATOL)
            _keys_ok(o2, None)
            _close_state(_strip(o2), _strip(cont_torch2[1]))


def test_checkpoint_resumes_into_another_world_size_and_buckets():
    world, per, steps = 2, 3, 3
    (msd, osd), _ = run_ranks(_ckpt_worker, world=world, backend="emu", args=(steps, per, "first", None, 0.002))
    want = _torch_run(*_torch_run(None, None, 0, steps, world * per), steps, steps, world * per)
    for (m2, o2) in run_ranks(_ckpt_worker, world=3, backend="emu", args=(steps, 2, "second", (msd, osd), 0.0005)):
        for k in m2:
            torch.testing.assert_close(m2[k], want[0][k], rtol=RTOL, atol=ATOL)
        _close_state(_strip(o2), _strip(want[1]))


# ------------------------------------------------------------------------------------------------ 5. rejections
def _reject_worker(rank, world):
    import dear_pytorch_b200 as dear
    out = []
    for kw in (dict(maximize=True), dict(capturable=True), dict(differentiable=True), dict(lr=torch.tensor(0.01))):
        m = make_model()
        try:
            dear.DistributedOptimizer(torch.optim.RMSprop(m.parameters(), **dict(dict(lr=0.01), **kw)), m, verbose=False)
            out.append(None)
        except ValueError as e:
            out.append(str(e))
    m = make_model()
    try:
        dear.DistributedOptimizer(torch.optim.Adagrad(m.parameters(), lr=0.01), m, verbose=False)
        out.append(None)
    except TypeError as e:
        out.append(str(e))
    return out


def test_rejections():
    msgs = run_ranks(_reject_worker, world=1, backend="emu")[0]
    assert all(msgs), msgs
    assert "maximize" in msgs[0] and "capturable" in msgs[1] and "differentiable" in msgs[2] and "tensor lr" in msgs[3]
    assert "RMSprop" in msgs[4]


# ------------------------------------------------------------------------------------------------ 6. bucket level
# Groups of the bucket-level matrix: centered with momentum, plain, centered without momentum, momentum with decay and
# alpha < 0.5 (the other lerp branch).  "nostate": no group centered and none with momentum, so no grad_avg and no
# momentum shard exist at all.
RMS_GROUPS = [dict(lr=1e-2, wd=1e-2, mu=0.9, alpha=0.99, centered=True, eps=1e-8),
              dict(lr=2e-2, wd=0.0, mu=0.0, alpha=0.9, centered=False, eps=1e-6),
              dict(lr=5e-3, wd=5e-3, mu=0.0, alpha=0.4, centered=True, eps=1.0),
              dict(lr=1e-2, wd=1e-2, mu=0.8, alpha=0.3, centered=False, eps=1e-8)]
NOSTATE_GROUPS = [RMS_GROUPS[1], dict(RMS_GROUPS[1], alpha=0.45, lr=1e-3)]
# Float64 bound: each fp32 operation rounds once (relative U); this many roundings per term bound the chain of sums and
# products (decay, square_avg, lerp, difference), then the sqrt, eps, division, momentum and step are propagated
# through their relative errors.  The device contracts a*b+c into FMA, which only removes roundings.
K = 6

Cfg = collections.namedtuple("Cfg", "pdt epi groups")


def configs(world):
    """(parameter dtype, epilogue, groups): every dtype with and without clipping (Kernel B's CLIP), a scaler with an
    injected inf (a skipped step and the count of applied updates; 16-bit parameters, so the master stays put too) and
    the configuration without optional state."""
    out = []
    for p in DTS:
        out += [Cfg(p, "none", "rms"), Cfg(p, "clip", "rms")]
    out += [Cfg("bf16", "amp", "rms"), Cfg("f32", "none", "nostate")]
    return out


def kernel_tuple(cfg, world, mc=False):
    W = world if world in (1, 2, 4, 8) else 0
    return ("ag_kernel", cfg.pdt, W, mc, "rmsprop", cfg.epi == "clip")


def reachable(worlds, mc=False):
    Ws = {w if w in (1, 2, 4, 8) else 0 for w in worlds}
    return {("ag_kernel", T, W, mc, "rmsprop", c) for T in DTS for W in Ws for c in (False, True) if not (mc and W == 1)}


def _rows(L, groups, rank, absent_rank):
    ends, rows = [], []
    for end, j, kind in L["hyper"]:
        h = dict(groups[j % len(groups)])
        h["skip"] = kind == "absent" or (kind == "zero_stale" and rank == absent_rank)
        ends.append(end)
        rows.append(h)
    return ends, rows


def _f32(x):
    return float(np.float32(x))


def _arrays(ends, rows, lo, hi):
    lens = torch.tensor(np.diff([0] + ends))
    out = {}
    for key in ("lr", "wd", "mu", "alpha", "eps"):
        vals = torch.tensor([_f32(r[key]) for r in rows], dtype=torch.float64)
        out[key] = torch.repeat_interleave(vals, lens)[lo:hi]
    out["w"] = torch.repeat_interleave(torch.tensor([_f32(1.0 - r["alpha"]) for r in rows], dtype=torch.float64), lens)[lo:hi]
    for key in ("centered", "skip"):
        out[key] = torch.repeat_interleave(torch.tensor([bool(r[key]) for r in rows]), lens)[lo:hi]
    return out


def rms_ref(p, g, sq, ga, buf, H, coef):
    """torch.optim.RMSprop in float64 from the state before the step, and the error bound of every result."""
    gc = g * coef
    g1 = gc + H["wd"] * p
    Mg = gc.abs() + (H["wd"] * p).abs()
    a, w = H["alpha"], H["w"]
    sq1 = a * sq + w * g1 * g1
    Msq = a * sq + w * Mg * Mg
    c = H["centered"]
    ga1 = torch.where(c, ga + w * (g1 - ga), ga)
    Mga = torch.where(c, ga.abs() + Mg, torch.zeros(()))
    var = torch.where(c, sq1 - ga1 * ga1, sq1)
    Mvar = torch.where(c, Msq + Mga * Mga, Msq)
    e_var = K * U * Mvar
    s = var.clamp(min=0).sqrt()
    # error of sqrt(var): e_var / (2 sqrt(var)) (var far from zero by construction), plus its own rounding
    e_s = torch.where(var > 0, e_var / (2 * s.clamp(min=1e-300)), e_var.sqrt()) + U * s
    den = s + H["eps"]
    e_den = e_s + U * den
    q = g1 / den
    e_q = K * U * Mg / den + q.abs() * (e_den / den + U)
    mom = H["mu"] > 0
    buf1 = torch.where(mom, H["mu"] * buf + q, buf)
    e_buf = torch.where(mom, K * U * (H["mu"] * buf.abs() + q.abs()) + e_q, torch.zeros(()))
    d = torch.where(mom, buf1, q)
    e_d = torch.where(mom, e_buf, e_q)
    p1 = p - H["lr"] * d
    e_p = K * U * (p.abs() + H["lr"] * d.abs()) + H["lr"] * e_d
    skip = H["skip"] & (g == 0)
    z = torch.zeros(())
    return dict(p=(torch.where(skip, p, p1), torch.where(skip, z, e_p)),
                sq=(torch.where(skip, sq, sq1), torch.where(skip, z, K * U * Msq)),
                ga=(torch.where(skip, ga, ga1), torch.where(skip, z, K * U * (Mga + Mg))),
                buf=(torch.where(skip, buf, buf1), torch.where(skip, z, e_buf)))


def run_config(C, comm, dev, rank, world, ci, cfg):
    tdt = TORCH_DT[cfg.pdt]
    es = ES[cfg.pdt]
    groups = RMS_GROUPS if cfg.groups == "rms" else NOSTATE_GROUPS
    has_mom = any(g["mu"] > 0 for g in groups)
    has_ga = any(g["centered"] for g in groups)
    amp, clip = cfg.epi == "amp", cfg.epi == "clip"
    lays = [std_layout(es, world), wide_layout(world, 384, 256, False)]
    bs = C.BucketSet(comm, [L["n"] for L in lays], getattr(C, CODE[cfg.pdt]), True)
    g0 = torch.Generator().manual_seed(3000 + ci)
    st = []
    for b, L in enumerate(lays):
        n = L["n"]
        sh = n // world
        init = torch.zeros(n)
        for s, k, _ in L["segs"]:
            init[s:s + k] = torch.randn(k, generator=g0)
        pbuf = bs.param_buffer(b)
        pbuf.copy_(init.to(tdt))
        S = dict(L=L, pbuf=pbuf, lo=rank * sh, sh=sh, gs=torch.zeros(sh, device=dev),
                 mom=torch.zeros(sh, device=dev) if has_mom else None, sq=torch.zeros(sh, device=dev),
                 ga=torch.zeros(sh, device=dev) if has_ga else None,
                 master=pbuf[rank * sh:(rank + 1) * sh].float().clone() if cfg.pdt != "f32" else None)
        bs.set_shards(b, S["gs"], S["mom"], S["master"], S["sq"], S["ga"])
        bs.set_step(b, 0)
        st.append(S)
    if amp:
        ampst = torch.zeros(9, dtype=torch.int32, device=dev)
        ampst.view(torch.float32)[2] = 1024.0
        ampst.view(torch.float32)[5] = 2.0
        ampst.view(torch.float32)[6] = 0.5
        ampst[7] = 1000
        bs.set_amp(ampst)
    if clip:
        clipst = torch.zeros(C.clip_state_floats(len(lays)), dtype=torch.float32, device=dev)
        clipst[0] = 1.0
        clipst.view(torch.int32)[3] = len(lays)
        bs.set_clip(clipst, list(range(len(lays))))
    recs, applied = [], 0
    nsteps = 3                                     # the scaler's injected inf lands on the last step
    for step in range(nsteps):
        inject = amp and step == 2
        absent_rank = step % world
        for b, S in enumerate(st):
            L = S["L"]
            seed = ((ci * 16 + step) * 16 + b) * 16 + 7
            gq = [make_grad(L, seed + q, q == absent_rank).to(tdt) for q in range(world)]
            if inject and b == 0:
                gq[world - 1][L["segs"][0][0] + 3] = float("inf")
            mine = gq[rank].to(dev)
            S["keep"] = mine
            src, off, nby, fl = [], [], [], []
            for s, k, kind in L["segs"]:
                off.append(s * es)
                nby.append(k * es)
                if kind == "absent" or (kind == "zero_stale" and rank == absent_rank):
                    src.append(0); fl.append(C.SEG_ZERO_FILL)
                else:
                    src.append(mine.data_ptr() + s * mine.element_size()); fl.append(0)
            bs.set_pack(b, src, off, nby, fl)
            ends, rows = _rows(L, groups, rank, absent_rank)
            bs.set_hyper(b, ends, [r["lr"] for r in rows], [r["wd"] for r in rows], [r["mu"] for r in rows],
                         [1.0 - r["alpha"] for r in rows],
                         [(HYPER_CENTERED if r["centered"] else 0) | (HYPER_SKIP if r["skip"] else 0) for r in rows],
                         opt=[OPT_RMSPROP] * len(rows), beta2=[r["alpha"] for r in rows], eps=[r["eps"] for r in rows])
            S["H"] = _arrays(ends, rows, S["lo"], S["lo"] + S["sh"])
            S["before"] = {k: (S[k].cpu().clone() if S[k] is not None else None) for k in ("mom", "sq", "ga", "master")}
            S["p0"] = S["pbuf"].cpu().clone()
        for b in range(len(st)):
            bs.reduce_scatter(b, True)
        bs.synchronize()
        for S in st:
            S["got"] = S["gs"].cpu().clone()               # Kernel A's shard: the input of the update
        for b in range(len(st)):
            bs.allgather_update(b, True, applied == 0, True, False, b == 0 and (amp or clip))
        bs.synchronize()
        coef = float(clipst[2]) if clip else 1.0
        if amp:
            a = ampst.cpu()
            assert int(a[1]) == int(inject) and int(a[4]) == applied + (0 if inject else 1), (cfg, step, a.tolist())
        if not inject:
            applied += 1
        hashes = []
        for b, S in enumerate(st):
            lo, sh = S["lo"], S["sh"]
            what = "%s step %d bucket %d" % (cfg, step, b)
            pb = S["pbuf"].cpu()
            master = S["master"].cpu() if S["master"] is not None else pb[lo:lo + sh].float()
            B = S["before"]
            if inject:
                assert torch.equal(_bits(pb, cfg.pdt), _bits(S["p0"], cfg.pdt)), what + ": parameters moved"
                for k in ("mom", "sq", "ga", "master"):
                    if S[k] is not None:
                        assert torch.equal(S[k].cpu(), B[k]), what + ": %s moved" % k
            else:
                p0 = (B["master"] if B["master"] is not None else S["p0"][lo:lo + sh].float()).double()
                zero = torch.zeros(sh, dtype=torch.float64)
                R = rms_ref(p0, S["got"].double(), B["sq"].double(), B["ga"].double() if has_ga else zero,
                            B["mom"].double() if has_mom else zero, S["H"], coef)
                _within(master.double(), *R["p"], what=what + " parameters vs float64")
                _within(S["sq"].cpu().double(), *R["sq"], what=what + " square_avg vs float64")
                if has_ga:
                    _within(S["ga"].cpu().double(), *R["ga"], what=what + " grad_avg vs float64")
                if has_mom:
                    _within(S["mom"].cpu().double(), *R["buf"], what=what + " momentum_buffer vs float64")
            if S["master"] is not None:
                assert torch.equal(_bits(pb[lo:lo + sh], cfg.pdt), _bits(master.to(tdt), cfg.pdt)), \
                    what + ": 16-bit parameters are not the master rounded"
            hashes.append(hashlib.sha1(pb.view(torch.uint8).numpy().tobytes()).hexdigest())
        recs.append(dict(cfg=tuple(cfg), step=step, hashes=hashes))
    del bs
    return recs


def bucket_worker(rank, world, mc):
    import dear_pytorch_b200 as dear
    from dear_pytorch_b200 import ops
    C = ops.require_native()
    assert (C.OPT_RMSPROP, C.HYPER_SKIP, C.HYPER_CENTERED) == (OPT_RMSPROP, HYPER_SKIP, HYPER_CENTERED)
    comm = dear.communicator()
    dev = dear.device()
    if mc:
        probe = C.BucketSet(comm, [world * 4096], C.DT_F32, True)
        ok = probe.has_multicast()
        del probe
        if not ok:
            return "no-multicast"
    recs = []
    for ci, cfg in enumerate(configs(world)):
        recs += run_config(C, comm, dev, rank, world, ci, cfg)
    comm.check_status()
    return recs


def check_ranks(outs):
    for recs in zip(*outs):
        assert all(r["hashes"] == recs[0]["hashes"] for r in recs), "%s step %d: parameter buffers differ between ranks" % (
            recs[0]["cfg"], recs[0]["step"])


def test_bucket_matrix_reaches_every_rmsprop_instantiation():
    ngpu = torch.cuda.device_count() if torch.cuda.is_available() else 0
    worlds = [1, 2, 3, 4] + ([8] if ngpu >= 8 else [])
    covered = {kernel_tuple(cfg, w) for w in worlds for cfg in configs(w)}
    missing = reachable(worlds) - covered
    assert not missing, sorted(missing)
    assert len(covered) == 24 + (6 if 8 in worlds else 0)


@pytest.mark.parametrize("world", [1, 2, 3])
def test_emulated_bucket_matrix(world):
    check_ranks(run_ranks(bucket_worker, world=world, backend="emu", args=(False,), extra_env=ENV, timeout=900))


# ------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_cuda_bucket_matrix(world):
    if not _gpu_world_ok(world):
        pytest.skip("ranks cannot share the GPUs evenly")
    check_ranks(run_ranks(bucket_worker, world=world, backend="b200", args=(False,), extra_env=ENV, timeout=900))


@pytest.mark.gpu
@pytest.mark.multigpu
def test_cuda_bucket_matrix_nvls():
    world = min(torch.cuda.device_count(), 8)
    missing = reachable([world], mc=True) - {kernel_tuple(cfg, world, mc=True) for cfg in configs(world)}
    assert not missing, sorted(missing)
    outs = run_ranks(bucket_worker, world=world, backend="b200", args=(True,), extra_env=dict(ENV, **ALGO_ENV["nvls"]),
                     timeout=900)
    if outs[0] == "no-multicast":
        pytest.skip("this box cannot create an NVLS multicast object")
    check_ranks(outs)


GPU_CASES = {"centered-momentum": dict(lr=1e-3, alpha=0.9, momentum=0.9, centered=True, weight_decay=1e-2),
             "plain": dict(lr=1e-3, alpha=0.99, momentum=0.0, centered=False)}


def _gpu_train_worker(rank, world, cases, steps, per):
    import dear_pytorch_b200 as dear
    dev = dear.device()
    out = []
    for kw in cases:
        m = make_model().to(dev); m.eval()
        opt = dear.DistributedOptimizer(make_opt("rmsprop", m, kw), m, threshold=0.002, verbose=False)
        dear.broadcast_parameters(m.state_dict(), 0)
        for t in range(steps):
            x, y = data(t, world * per)
            x, y = x[rank * per:(rank + 1) * per].to(dev), y[rank * per:(rank + 1) * per].to(dev)
            opt.zero_grad()
            F.cross_entropy(m(x), y).backward()
            opt.step()
        opt.synchronize()
        out.append([p.detach().cpu() for p in m.parameters()])
        opt.engine.close()
    dear.communicator().check_status()
    return out


# 16-bit parameters with fp32 masters are pinned on the GPU by the bucket matrix above (float64 oracle, master rounding
# invariant): a bf16 network's own forward / backward drifts from an fp32 trajectory by more than any fixed tolerance.


def _graph_worker(rank, world, steps, per):
    import dear_pytorch_b200 as dear
    dev = dear.device()
    res = []
    for use_graph in (False, True):
        m = make_model().to(dev); m.eval()
        opt = dear.DistributedOptimizer(make_opt("rmsprop", m), m, threshold=0.002, norm_clip=0.05, verbose=False)
        dear.broadcast_parameters(m.state_dict(), 0)
        scaler = dear.GradScaler(opt, init_scale=2.0 ** 10, growth_interval=3)
        step = dear.TrainStep(m, opt, F.cross_entropy, use_graph=use_graph, overlap_update=True, scaler=scaler,
                              graph_warmup=2)
        for t in range(steps):
            x, y = data(t, world * per)
            step(x[rank * per:(rank + 1) * per].to(dev), y[rank * per:(rank + 1) * per].to(dev))
        opt.synchronize()
        res.append(([p.detach().cpu().clone() for p in m.parameters()], float(opt.engine.last_grad_norm),
                    scaler.get_scale(), step._graph is not None))
        opt.engine.close()
    dear.communicator().check_status()
    return res


def _end_to_end_worker(rank, world, cases, steps, per, graph_steps):
    # one set of rank processes for both checks: starting CUDA in every rank costs more than the training itself
    return _gpu_train_worker(rank, world, cases, steps, per), (_graph_worker(rank, world, graph_steps, per) if graph_steps
                                                               else None)


@pytest.mark.gpu
@pytest.mark.parametrize("world", [1, 2])
def test_gpu_end_to_end(world):
    """A small fp32 CNN against torch.optim.RMSprop (centered with momentum, and plain) at worlds 1 and 2; at world 2 also
    CUDA-graph replay of the rotated TrainStep with GradScaler and norm_clip, bitwise equal to the eager run."""
    if not _gpu_world_ok(world):
        pytest.skip("ranks cannot share the GPUs evenly")
    names, steps, per = sorted(GPU_CASES), 5, 4
    cases = [GPU_CASES[n] for n in names]
    refs = [_reference(kw, steps, world, per)[0] for kw in cases]
    graph_steps = 8 if world == 2 else 0
    for res, graph in run_ranks(_end_to_end_worker, world=world, backend="b200", args=(cases, steps, per, graph_steps),
                                extra_env=ENV, timeout=300):
        for name, params, ref in zip(names, res, refs):
            for a, b in zip(params, ref):
                torch.testing.assert_close(a, b, rtol=2e-4, atol=5e-6, msg=lambda m: "%s: %s" % (name, m))
        if graph is not None:
            (pe, ne, se, _), (pg, ng, sg, captured) = graph
            assert captured
            assert ne == ng and se == sg
            assert all(torch.equal(a, b) for a, b in zip(pe, pg))
