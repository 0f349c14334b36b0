#!/usr/bin/env python
"""Randomised equivalence test of the distributed optimizers against single-process ``torch.optim`` (CPU, no GPU needed).

Every trial draws a model (depth / width / tied weight / a branch that only runs in some passes), an optimizer (SGD
flavours, Adam, AdamW, one or two parameter groups, optional LR schedule), a world size, a bucketing policy, gradient
accumulation, mid-run re-bucketing and a state-dict round trip, runs it on the ``emu`` (native runtime, kernels emulated
on the host) or ``gloo`` backend, and compares every parameter with the oracle trained on the concatenated batch.  This is
how the per-parameter Adam step count, the accumulation / bucket-view and the reduce-broadcast "unused parameter"
deviations were found.

    python tools/fuzz_equivalence.py --seed 1 --trials 40 [--variants dear,naive,wt,rb,bo,wfbp,horovod,bytescheduler]
"""
from __future__ import annotations

import argparse
import os
import random
import sys

import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
# rank processes that do not fork (spawn / fork server) import this module by name to find `worker`
sys.path.insert(0, os.path.join(ROOT, "tools"))
from _mp import run_ranks  # noqa: E402


class Net(nn.Module):
    def __init__(self, seed, depth, width, tie):
        super().__init__()
        torch.manual_seed(seed)
        self.inp = nn.Linear(12, width)
        self.blocks = nn.ModuleList(nn.Linear(width, width, bias=(i % 2 == 0)) for i in range(depth))
        self.norm = nn.LayerNorm(width)
        self.side = nn.Linear(width, width)              # runs in some passes only
        self.out = nn.Linear(width, 6)
        self.tie = tie

    def forward(self, x, use_side):
        h = torch.tanh(self.inp(x))
        for b in self.blocks:
            h = h + 0.2 * torch.tanh(b(h))
        if self.tie:
            h = h + 0.1 * nn.functional.linear(h, self.blocks[0].weight)      # second (functional) use of a weight
        h = self.norm(h)
        if use_side:
            h = h + 0.3 * torch.relu(self.side(h))
        return self.out(h)


def make_opt(kind, groups):
    if kind == "sgd":
        return torch.optim.SGD(groups, lr=0.05)
    if kind == "sgdm":
        return torch.optim.SGD(groups, lr=0.05, momentum=0.9, weight_decay=1e-3)
    if kind == "nesterov":
        return torch.optim.SGD(groups, lr=0.05, momentum=0.8, nesterov=True, weight_decay=1e-2)
    if kind == "damp":
        return torch.optim.SGD(groups, lr=0.05, momentum=0.8, dampening=0.3, weight_decay=5e-3)
    if kind == "adam":
        return torch.optim.Adam(groups, lr=0.01, weight_decay=1e-3)
    if kind == "rmsprop":
        return torch.optim.RMSprop(groups, lr=1e-3, alpha=0.9, weight_decay=1e-3)
    if kind == "rmsprop-centered-momentum":
        return torch.optim.RMSprop(groups, lr=1e-3, alpha=0.9, momentum=0.9, centered=True, weight_decay=1e-3)
    return torch.optim.AdamW(groups, lr=0.01, weight_decay=1e-2)


def param_groups(model, split):
    if not split:
        return [{"params": list(model.parameters())}]
    small = [p for n, p in model.named_parameters() if n.endswith("bias") or "norm" in n]
    big = [p for n, p in model.named_parameters() if not (n.endswith("bias") or "norm" in n)]
    return [{"params": big}, {"params": small, "lr": 0.02, "weight_decay": 0.0}]


def batch(i, n):
    g = torch.Generator().manual_seed(77 + i)
    return torch.randn(n, 12, generator=g), torch.randint(0, 6, (n,), generator=g)


def use_side(cfg, t, a):
    return cfg["branch"] and (t * cfg["accum"] + a) % cfg["mod"] == 1


def oracle(cfg):
    m = Net(cfg["seed"], cfg["depth"], cfg["width"], cfg["tie"])
    opt = make_opt(cfg["opt"], param_groups(m, cfg["split"]))
    sched = torch.optim.lr_scheduler.StepLR(opt, 2, 0.5) if cfg["sched"] else None
    k = cfg["accum"]
    for t in range(cfg["steps"]):
        opt.zero_grad()
        for a in range(k):
            x, y = batch(t * k + a, cfg["world"] * cfg["per"])
            (nn.functional.cross_entropy(m(x, use_side(cfg, t, a)), y) / k).backward()
        if cfg["clip"]:
            torch.nn.utils.clip_grad_norm_(m.parameters(), cfg["clip"])
        opt.step()
        if sched:
            sched.step()
    return [p.detach().clone() for p in m.parameters()]


def worker(rank, world, cfg):
    import dear_pytorch_b200 as dear
    from dear_pytorch_b200.parallel import variants
    dev = dear.device()                                  # cpu for emu / gloo, cuda:LOCAL_RANK for b200 / nccl
    m = Net(cfg["seed"], cfg["depth"], cfg["width"], cfg["tie"]).to(dev)
    base = make_opt(cfg["opt"], param_groups(m, cfg["split"]))
    v, k = cfg["variant"], cfg["accum"]
    if v == "naive":
        opt = variants.NaiveDistributedOptimizer(base, m, verbose=False)
    elif v == "wt":
        opt = variants.WaitTimeDistributedOptimizer(base, m, cycle_time_ms=0.05, warmup_steps=2, verbose=False)
    elif v == "rb":
        opt = variants.ReduceBroadcastDistributedOptimizer(base, m, threshold=cfg["thr"] or 0.002, verbose=False)
    elif v in ("wfbp", "horovod", "bytescheduler"):
        from dear_pytorch_b200.parallel import baselines
        if v == "wfbp":
            opt = baselines.WFBPDistributedOptimizer(base, model=m, threshold=cfg["elems"], verbose=False)
        elif v == "horovod":
            opt = baselines.HorovodOptimizer(base, m, cycle_time_ms=cfg["cycle"], fusion_threshold_mb=0.002, negotiation_steps=2,
                                             verbose=False)
        else:
            opt = baselines.ByteSchedulerOptimizer(base, m, partition=cfg["elems"] or 100000, credit=cfg["credit"], verbose=False)
    else:
        kw = dict(threshold=cfg["thr"]) if cfg["thr"] else dict(threshold=None, num_nearby_layers=cfg["nearby"])
        if v == "bo":
            kw.update(bo_tuning=True, bo_kwargs=dict(bound=(0.0003, 0.02), max_num_steps=3, interval=2))
        opt = dear.DistributedOptimizer(base, m, verbose=False, backward_passes_per_step=k, norm_clip=cfg["clip"] or None, **kw)
    sched = torch.optim.lr_scheduler.StepLR(opt, 2, 0.5) if cfg["sched"] else None
    dear.broadcast_parameters(m.state_dict(), 0)
    per = cfg["per"]
    train_step = None
    if cfg["trainstep"]:
        # the packaged iteration (utils/train.py), natural or rotated body; the branch flag travels as an input
        train_step = dear.TrainStep(m, opt, lambda out, y: nn.functional.cross_entropy(out, y), use_graph=False,
                                    overlap_update=cfg["rot"])
    for t in range(cfg["steps"]):
        if train_step is not None:
            x, y = batch(t, world * per)
            train_step(x[rank * per:(rank + 1) * per].to(dev), use_side(cfg, t, 0), y[rank * per:(rank + 1) * per].to(dev))
            if sched:
                sched.step()
            continue
        opt.zero_grad()
        for a in range(k):
            x, y = batch(t * k + a, world * per)
            (nn.functional.cross_entropy(m(x[rank * per:(rank + 1) * per].to(dev), use_side(cfg, t, a)),
                                         y[rank * per:(rank + 1) * per].to(dev)) / k).backward()
        opt.step()
        if sched:
            sched.step()
        if v == "dear" and cfg["rebucket"] and t == cfg["rebucket"]:
            opt.engine.rebucket(("threshold", cfg["thr2"]))
        if v in ("dear", "bo") and cfg["ckpt"] and t == cfg["ckpt"]:
            opt.load_state_dict(opt.state_dict())
    if train_step is not None:
        train_step.finish()
    if hasattr(opt, "synchronize"):
        opt.synchronize()
    return [p.detach().float().cpu().clone() for p in m.parameters()]


def draw(rnd, variants_allowed, backends=None, max_world=4):
    v = rnd.choice(variants_allowed)
    engine = v in ("dear", "bo", "naive", "wt", "wfbp", "horovod", "bytescheduler")
    cfg = dict(variant=v, seed=rnd.randint(0, 99), depth=rnd.randint(1, 5), width=rnd.choice([8, 17, 32]), tie=rnd.random() < 0.3,
               branch=rnd.random() < 0.5, mod=rnd.choice([2, 3, 5]),
               opt=rnd.choice(["sgd", "sgdm", "nesterov", "damp", "adam", "adamw"] if engine else ["sgd", "sgdm", "nesterov", "damp"]),
               split=rnd.random() < 0.5, world=rnd.choice([1, 2, 3, 4]), per=rnd.choice([1, 2]),
               steps=rnd.randint(6, 12) if v == "bo" else rnd.randint(3, 6), sched=rnd.random() < 0.3,
               thr=rnd.choice([None, 0.0005, 0.002, 0.01]), nearby=rnd.choice([1, 2, 3, -1]),
               accum=rnd.choice([1, 1, 2, 3]) if v == "dear" else 1, rebucket=rnd.choice([0, 0, 1, 2]),
               thr2=rnd.choice([0.0004, 0.003, 1.0]), ckpt=rnd.choice([0, 0, 1, 2]), backend=rnd.choice(["emu", "emu", "gloo"]),
               pipe=rnd.random() < 0.25, elems=rnd.choice([0, 50, 300, 5000]), cycle=rnd.choice([0.0, 0.2, 5.0]),
               credit=rnd.choice([100, 1000, 10 ** 7]))
    cfg["clip"] = rnd.choice([0, 0, 0.3, 2.0]) if v == "dear" else 0
    cfg["trainstep"] = rnd.random() < 0.3
    cfg["rot"] = rnd.random() < 0.6
    if cfg["trainstep"]:
        cfg.update(accum=1, rebucket=0, ckpt=0)
    if backends:
        cfg["backend"] = rnd.choice(backends)
    cfg["world"] = min(cfg["world"], max_world)
    if v in ("wfbp", "horovod", "bytescheduler"):
        # NCCL-style baselines: torch.distributed only; modules own their weights
        cfg.update(backend="nccl" if cfg["backend"] in ("b200", "nccl") else "gloo", tie=False)
    if v == "bo" and not cfg["thr"]:
        cfg["thr"] = 0.002
    # RMSprop takes the Adam family's slot half of the time: drawn from its own generator (seeded by the trial), so a
    # seed's sequence of trials keeps every other dimension — and its cost — as before
    if cfg["opt"] in ("adam", "adamw") and random.Random("rmsprop:%d:%d:%d" % (cfg["seed"], cfg["depth"], cfg["width"])).random() < 0.5:
        cfg["opt"] = "rmsprop" if cfg["opt"] == "adam" else "rmsprop-centered-momentum"
    return cfg


def run_trial(cfg):
    env = {"DEAR_RS_ALGO": "pipe", "DEAR_STRIPE_MB": "0.001"} if (cfg["pipe"] and cfg["backend"] == "emu") else None
    gpu = cfg["backend"] in ("b200", "nccl")
    if gpu:
        env = dict(env or {}, DEAR_SPIN_TIMEOUT_S="15")
    ref = oracle(cfg)
    outs = run_ranks(worker, world=cfg["world"], backend=cfg["backend"], args=(cfg,), timeout=300 if gpu else 180, extra_env=env)
    tol = dict(rtol=1e-3, atol=5e-5) if cfg["opt"].startswith(("adam", "rmsprop")) else dict(rtol=5e-5, atol=5e-6)
    if gpu:                                                # other reduction orders in the GEMMs than the CPU oracle
        tol = dict(rtol=2e-3, atol=1e-4)
    for params in outs:
        for a, b in zip(params, ref):
            torch.testing.assert_close(a, b, **tol)
    for other in outs[1:]:
        for a, b in zip(outs[0], other):
            assert torch.equal(a, b), "replicas are not bit-identical"


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--trials", type=int, default=20)
    ap.add_argument("--variants", default="dear,dear,dear,bo,naive,wt,rb,wfbp,horovod,bytescheduler")
    ap.add_argument("--quiet", action="store_true")
    ap.add_argument("--backends", default=None, help="comma list; default emu,emu,gloo.  b200 runs the fused kernels (GPU box)")
    ap.add_argument("--max-world", type=int, default=4)
    args = ap.parse_args(argv)
    rnd = random.Random(args.seed)
    failures = []
    for i in range(args.trials):
        cfg = draw(rnd, args.variants.split(","), args.backends.split(",") if args.backends else None, args.max_world)
        try:
            run_trial(cfg)
            if not args.quiet:
                print(i, "ok", {k: cfg[k] for k in ("variant", "opt", "world", "backend", "accum", "branch", "tie", "split", "sched", "rebucket", "ckpt", "trainstep", "rot", "clip")},
                      flush=True)
        except Exception as e:      # noqa: BLE001 - report and continue
            failures.append((cfg, str(e)[-800:]))
            print(i, "FAIL", cfg, str(e)[-800:], flush=True)
    print("failures: %d / %d" % (len(failures), args.trials))
    return failures


if __name__ == "__main__":
    sys.exit(1 if main() else 0)
