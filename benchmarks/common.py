"""Shared pieces of the synthetic benchmark drivers (imagenet_benchmark.py / bert_benchmark.py).

The drivers keep the reference's command line (dear/imagenet_benchmark.py:24-56) and its log lines
("Iter #k: ... img/sec per GPU", "Total img/sec on N GPU(s)", scraped by benchmarks.py), but
  * the optimizer variant is a flag (``--method``), not an edited import line;
  * timing is CUDA events on the compute stream, max over ranks, without a device synchronise
    inside the step (the reference calls torch.cuda.synchronize() in benchmark_step and times with
    host timeit, dear/imagenet_benchmark.py:126-136,151-164).
"""
from __future__ import annotations

import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import dear_pytorch_b200 as dear  # noqa: E402

METHODS = ("dear", "dear-bo", "dear-notf", "dear-naive", "dear-wt", "dear-rb", "wfbp", "mgwfbp", "asc",
           "ddp", "ddp-zero", "horovod", "bytescheduler", "single")


def add_common_args(ap):
    ap.add_argument("--method", default="dear", choices=METHODS, help="distributed optimizer variant / baseline")
    ap.add_argument("--fp16", action="store_true", default=False, help="(reference flag) bf16 parameters with fp32 master shards")
    ap.add_argument("--dtype", default=None, choices=[None, "fp32", "bf16", "amp"])
    ap.add_argument("--batch-size", type=int, default=32)
    ap.add_argument("--num-warmup-batches", type=int, default=10)
    ap.add_argument("--num-batches-per-iter", type=int, default=10)
    ap.add_argument("--num-iters", type=int, default=5)
    ap.add_argument("--no-cuda", action="store_true", default=False)
    ap.add_argument("--mgwfbp", action="store_true", default=False, help="(reference flag) same as --method mgwfbp")
    ap.add_argument("--asc", action="store_true", default=False, help="(reference flag) same as --method asc")
    ap.add_argument("--nstreams", type=int, default=1)
    ap.add_argument("--threshold", type=float, default=25.0, help="fusion threshold: MB for dear*, elements for wfbp")
    ap.add_argument("--rdma", action="store_true", default=False)
    ap.add_argument("--compressor", type=str, default="none")
    ap.add_argument("--density", type=float, default=1.0)
    ap.add_argument("--momentum-correction", action="store_true", default=False,
                    help="sparse WFBP: accumulate the velocity before sparsification (wfbp/dopt.py:906-953)")
    ap.add_argument("--exclude-parts", type=str, default="", help="reducescatter, allgather (time breakdown)")
    ap.add_argument("--momentum", type=float, default=0.0)
    ap.add_argument("--optimizer", choices=["sgd", "adam", "adamw", "rmsprop"], default="sgd",
                    help="adam/adamw/rmsprop: sharded Adam / RMSprop fused into the all-gather kernel (dear methods only); "
                         "RMSprop takes its momentum from --momentum")
    ap.add_argument("--rmsprop-alpha", type=float, default=0.99, help="--optimizer rmsprop: smoothing constant alpha")
    ap.add_argument("--rmsprop-eps", type=float, default=1e-8, help="--optimizer rmsprop: eps")
    ap.add_argument("--rmsprop-centered", action="store_true", default=False, help="--optimizer rmsprop: centered")
    ap.add_argument("--graph", type=int, default=0, help="capture the whole iteration in a CUDA graph")
    ap.add_argument("--norm-clip", type=float, default=None,
                    help="dear, dear-bo, dear-notf: clip the global gradient norm to this value (clip_grad_norm_ semantics, "
                         "inside the fused kernels)")
    ap.add_argument("--grad-comm-dtype", choices=["fp32", "bf16", "fp16"], default="fp32",
                    help="dear, dear-bo, dear-notf: dtype in which fp32 gradients are sent to the reduce-scatter (rounded "
                         "on every rank, summed in fp32)")
    # flags of the reference's baseline drivers (horovod/, bytescheduler/, pytorch-ddp/ imagenet_benchmark.py)
    ap.add_argument("--fp16-allreduce", action="store_true", default=False,
                    help="--method horovod: fused buffers travel as fp16 (hvd.Compression.fp16)")
    ap.add_argument("--use-adasum", action="store_true", default=False,
                    help="--method horovod: Adasum reduction (hvd.Adasum); like the reference, the lr is then not scaled by "
                         "the number of ranks")
    ap.add_argument("--use-zero", type=int, default=0, help="--method ddp: ZeroRedundancyOptimizer (= --method ddp-zero)")
    ap.add_argument("--partition", type=int, default=None, help="--method bytescheduler: partition size in elements")
    ap.add_argument("--json", type=str, default=None, help="also write the result as JSON to this file")
    return ap


def resolve_method(args):
    if args.mgwfbp:
        return "mgwfbp"
    if args.asc:
        return "asc"
    if args.method == "ddp" and getattr(args, "use_zero", 0):
        return "ddp-zero"
    return args.method


def init_runtime(args):
    method = resolve_method(args)
    cuda = not args.no_cuda and torch.cuda.is_available()
    if not cuda:
        backend = os.environ.get("DEAR_BACKEND", "gloo")
    elif method.startswith("dear"):
        backend = os.environ.get("DEAR_BACKEND", "b200")
    else:
        backend = "nccl"
    dear.init(backend=backend, nstreams=args.nstreams)
    torch.backends.cudnn.benchmark = True
    return method, cuda


def wrap_optimizer(method, args, model, optimizer, profile_fn=None):
    """Returns (model, optimizer) for the chosen method."""
    from dear_pytorch_b200.parallel import variants
    from dear_pytorch_b200.parallel import baselines
    from dear_pytorch_b200.parallel.compression import compressors
    world = dear.size()
    if method == "single" or (world == 1 and not method.startswith("dear")):
        return model, optimizer
    wire = {"fp32": None, "bf16": torch.bfloat16, "fp16": torch.float16}[getattr(args, "grad_comm_dtype", "fp32")]
    if method == "dear":
        return model, dear.DistributedOptimizer(optimizer, model, threshold=args.threshold, exclude_parts=args.exclude_parts,
                                                norm_clip=args.norm_clip, grad_comm_dtype=wire)
    if method == "dear-bo":
        return model, dear.DistributedOptimizer(optimizer, model, threshold=args.threshold, exclude_parts=args.exclude_parts,
                                                bo_tuning=True, norm_clip=args.norm_clip, grad_comm_dtype=wire)
    if method == "dear-notf":
        return model, dear.DistributedOptimizer(optimizer, model, threshold=None, num_nearby_layers=1,
                                                exclude_parts=args.exclude_parts, norm_clip=args.norm_clip,
                                                grad_comm_dtype=wire)
    if method == "dear-naive":
        return model, variants.NaiveDistributedOptimizer(optimizer, model, exclude_parts=args.exclude_parts)
    if method == "dear-wt":
        return model, variants.WaitTimeDistributedOptimizer(optimizer, model, exclude_parts=args.exclude_parts)
    if method == "dear-rb":
        return model, variants.ReduceBroadcastDistributedOptimizer(optimizer, model, threshold=args.threshold,
                                                                   nstreams=args.nstreams, exclude_parts=args.exclude_parts)
    if method in ("wfbp", "mgwfbp", "asc"):
        seq, times = (None, None)
        if method in ("mgwfbp", "asc"):
            seq, times, _ = profile_fn()
            seq, times = dear.runtime.broadcast_object((seq, times), src=0)
        thr = 0 if method == "wfbp" and args.threshold == 25.0 else int(args.threshold)
        comp = compressors[args.compressor]()
        return model, baselines.WFBPDistributedOptimizer(
            optimizer, model=model, compression=comp, is_sparse=args.density < 1, density=args.density,
            seq_layernames=seq, layerwise_times=times, threshold=thr, mgwfbp=(method == "mgwfbp"), asc=(method == "asc"),
            rdma=args.rdma, momentum_correction=getattr(args, "momentum_correction", False))
    if method == "horovod":
        return model, baselines.HorovodOptimizer(                         # HOROVOD_FUSION_THRESHOLD / HOROVOD_CYCLE_TIME
            optimizer, model, fp16_allreduce=getattr(args, "fp16_allreduce", False),
            op="adasum" if getattr(args, "use_adasum", False) else "average")
    if method == "bytescheduler":
        return model, baselines.ByteSchedulerOptimizer(                   # BYTESCHEDULER_PARTITION / BYTESCHEDULER_CREDIT
            optimizer, model, partition=getattr(args, "partition", None))
    if method in ("ddp", "ddp-zero"):
        kw = dict(optimizer.defaults)
        ddp_model, opt = baselines.wrap_ddp(model, type(optimizer), {k: v for k, v in kw.items() if k in
                                            ("lr", "momentum", "weight_decay", "dampening", "nesterov")},
                                            zero=(method == "ddp-zero"))
        return ddp_model, opt
    raise ValueError(method)


def log(s, nl=True):
    if dear.rank() != 0:
        return
    print(s, end="\n" if nl else "", flush=True)


def run_timing(step_fn, args, unit_name, batch_size, sync_fn):
    """The reference's loop (warm-up, num_iters x num_batches_per_iter) with device timing."""
    cuda = dear.device().type == "cuda"
    log("Running warmup...")
    for _ in range(args.num_warmup_batches):
        step_fn()
    sync_fn()
    log("Running benchmark...")
    rates, iter_times = [], []
    for x in range(args.num_iters):
        dear.barrier()
        if cuda:
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
        t0 = time.perf_counter()
        for _ in range(args.num_batches_per_iter):
            step_fn()
        sync_fn(host=False)
        if cuda:
            e1.record()
            torch.cuda.synchronize()
            dt = e0.elapsed_time(e1) / 1e3
        else:
            dt = time.perf_counter() - t0
        if dear.size() > 1:
            import torch.distributed as dist
            t = torch.tensor([dt], dtype=torch.float64)
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            dt = float(t)
        rate = batch_size * args.num_batches_per_iter / dt
        log("Iter #%d: %.1f %s/sec per GPU" % (x, rate, unit_name))
        rates.append(rate)
        iter_times.append(dt / args.num_batches_per_iter)
    mean, conf = float(np.mean(rates)), float(1.96 * np.std(rates))
    log("Iteraction time: %.3f +-%.3f" % (np.mean(iter_times), 1.96 * np.std(iter_times)))
    log("%s/sec per %s: %.1f +-%.1f" % (unit_name.capitalize(), "GPU" if cuda else "CPU", mean, conf))
    log("Total %s/sec on %d %s(s): %.1f +-%.1f" % (unit_name, dear.size(), "GPU" if cuda else "CPU",
                                                    dear.size() * mean, dear.size() * conf))
    return {"per_gpu": mean, "total": dear.size() * mean, "conf": conf, "iter_time_s": float(np.mean(iter_times))}


def finish(args, result, extra):
    if dear.rank() == 0 and args.json:
        import json
        with open(args.json, "w") as f:
            json.dump(dict(result, **extra), f, indent=1)


def make_base_optimizer(args, params, lr):
    """The reference benchmarks always use SGD (dear/imagenet_benchmark.py:94, dear/bert_benchmark.py:122)."""
    import torch
    if getattr(args, "optimizer", "sgd") == "adamw":
        return torch.optim.AdamW(params, lr=lr)
    if getattr(args, "optimizer", "sgd") == "adam":
        return torch.optim.Adam(params, lr=lr)
    if getattr(args, "optimizer", "sgd") == "rmsprop":
        return torch.optim.RMSprop(params, lr=lr, alpha=args.rmsprop_alpha, eps=args.rmsprop_eps, momentum=args.momentum,
                                   centered=args.rmsprop_centered)
    return torch.optim.SGD(params, lr=lr, momentum=args.momentum)
