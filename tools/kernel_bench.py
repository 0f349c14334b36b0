#!/usr/bin/env python
"""Micro-benchmark of the two fused kernels against their roofline and against NCCL.

    torchrun --nproc-per-node N tools/kernel_bench.py [--sizes-mb 1,4,16,24,64,392] [--dtype fp32]
                                                      [--grad-comm-dtype fp32|bf16|fp16]

For every bucket size it times (CUDA events, after warm-up, max over ranks)
  Kernel A  rs_kernel : pack + reduce-scatter + fp32 accumulate + 1/P scale
  Kernel B  ag_kernel : sharded SGD(momentum) + all-gather push
and the NCCL collectives the reference issues for the same bucket
(reduce_scatter_tensor / all_gather_into_tensor, without the reference's extra elementwise kernels).
Bus bandwidth = bytes * (P-1)/P / time, reported against the H100 SXM data sheet's 450 GB/s per direction
(utils/perf_model.py); at P = 1 the HBM roofline applies instead.  ``--grad-comm-dtype bf16|fp16`` (fp32 buckets, P > 1)
sends the gradients at 16 bits: the pack reads fp32 and writes 16-bit wire elements, the pull reads wire bytes.
``rs_link_bytes`` / ``rs_hbm_bytes`` are the byte model of Kernel A per rank.  With ranks sharing one GPU, "peer" loads
read local HBM, so those times say nothing about the link.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import dear_pytorch_b200 as dear  # noqa: E402
from dear_pytorch_b200 import ops  # noqa: E402
from dear_pytorch_b200.utils import perf_model  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes-mb", default="1,4,16,24,64,392")
    ap.add_argument("--dtype", default="fp32", choices=["fp32", "bf16"])
    ap.add_argument("--grad-comm-dtype", default="fp32", choices=["fp32", "bf16", "fp16"],
                    help="--dtype fp32 only: dtype of the gradient buckets (the pack rounds the fp32 gradients)")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--nccl", type=int, default=1)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    dear.init(backend="b200")
    C = ops.require_native()
    rank, world, dev = dear.rank(), dear.size(), dear.device()
    comm = dear.communicator()
    tdt = torch.float32 if args.dtype == "fp32" else torch.bfloat16
    es = 4 if args.dtype == "fp32" else 2
    sizes_mb = [float(s) for s in args.sizes_mb.split(",")]
    quantum = world * 128 // es
    numels = [max(quantum, int(mb * 2 ** 20 / es) // quantum * quantum) for mb in sizes_mb]
    wire = args.grad_comm_dtype if args.dtype == "fp32" and world > 1 and args.grad_comm_dtype != "fp32" else None
    wes = 2 if wire else es                      # bytes per gradient element in the bucket (on the wire)
    bs = C.BucketSet(comm, numels, C.DT_F32 if args.dtype == "fp32" else C.DT_BF16, True,
                     {"bf16": C.DT_BF16, "fp16": C.DT_F16}.get(wire))
    results = []
    peaks = perf_model.measured_peaks()

    def maxr(v):
        if world == 1:
            return v
        t = torch.tensor([v], dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t)

    def timed(fn, iters):
        for _ in range(3):
            fn()
        bs.wait_all()
        torch.cuda.synchronize()
        dear.barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        bs.wait_all()
        e1.record()
        torch.cuda.synchronize()
        return maxr(e0.elapsed_time(e1) / iters * 1e3)      # us

    for g, n in enumerate(numels):
        nbytes = n * es
        wbytes = n * wes
        shard = n // world
        grad_src = torch.randn(n, device=dev).to(tdt)                   # "autograd output" to be packed
        gs = torch.zeros(shard, device=dev)
        mom = torch.zeros(shard, device=dev)
        master = torch.zeros(shard, device=dev) if args.dtype != "fp32" else None
        bs.set_shards(g, gs, mom, master)
        bs.set_pack(g, [grad_src.data_ptr()], [0], [wbytes], [0])
        bs.set_hyper(g, [n], [0.01], [1e-4], [0.9], [0.0], [0])
        bs.param_buffer(g).normal_()
        torch.cuda.synchronize()
        t_rs = timed(lambda: bs.reduce_scatter(g, True), args.iters)
        t_rs_nopack = timed(lambda: bs.reduce_scatter(g, False), args.iters)
        t_ag = timed(lambda: bs.allgather_update(g, True, False, True, False), args.iters)
        row = {"bucket_mb": round(nbytes / 2 ** 20, 2), "dtype": args.dtype, "grad_comm_dtype": wire or args.dtype,
               "world": world, "rs_plan": bs.rs_plan(g),
               "rs_us": round(t_rs, 2), "rs_nopack_us": round(t_rs_nopack, 2), "ag_sgd_us": round(t_ag, 2)}
        rr = perf_model.rs_roofline_us(wbytes, world, wes, peaks, src_elem_bytes=es)
        row["rs_link_bytes"] = int(rr["link_bytes"])
        row["rs_hbm_bytes"] = int(rr["hbm_bytes"])
        ar = perf_model.ag_roofline_us(nbytes, world, es, True, peaks)
        row["rs_roofline_us"] = round(rr["bound_us"], 2)
        row["ag_roofline_us"] = round(ar["bound_us"], 2)
        row["rs_frac_of_roofline"] = round(rr["bound_us"] / t_rs, 3)
        row["ag_frac_of_roofline"] = round(ar["bound_us"] / t_ag, 3)
        if world > 1:
            link = nbytes * (world - 1) / world
            row["rs_busbw_gbs"] = round(wbytes * (world - 1) / world / t_rs / 1e3, 1)
            row["ag_busbw_gbs"] = round(link / t_ag / 1e3, 1)
        if args.nccl and world > 1:
            full = torch.randn(n, device=dev).to(tdt)
            out = torch.empty(shard, device=dev, dtype=tdt)

            def nccl_timed(fn):
                for _ in range(3):
                    fn()
                torch.cuda.synchronize(); dear.barrier()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.iters):
                    fn()
                e1.record(); torch.cuda.synchronize()
                return maxr(e0.elapsed_time(e1) / args.iters * 1e3)
            row["nccl_rs_us"] = round(nccl_timed(lambda: dist.reduce_scatter_tensor(out, full)), 2)
            row["nccl_ag_us"] = round(nccl_timed(lambda: dist.all_gather_into_tensor(full, out)), 2)
            # the work Kernel A actually replaces (dear/dear_dopt.py:265 + communicator.cpp:157-169 + :306): copy the
            # gradients into the flat buffer (ONE copy kernel here; the reference launches one per parameter), the
            # NCCL reduce-scatter, and the division by the world size
            src = torch.randn(n, device=dev).to(tdt)

            def ref_path():
                full.copy_(src)
                dist.reduce_scatter_tensor(out, full)
                out.div_(world)
            row["nccl_copy_rs_div_us"] = round(nccl_timed(ref_path), 2)
            row["rs_vs_nccl"] = round(t_rs / row["nccl_rs_us"], 3)
            # gradients that a GEMM wrote straight into the bucket (ops/direct_wgrad.py: Linear layers) skip the pack
            row["rs_nopack_vs_nccl"] = round(t_rs_nopack / row["nccl_rs_us"], 3)
            row["rs_vs_nccl_copy_rs_div"] = round(t_rs / row["nccl_copy_rs_div_us"], 3)
            del src
        results.append(row)
        if rank == 0:
            print(json.dumps(row), flush=True)
        del grad_src
    comm.check_status()
    if rank == 0 and args.out:
        with open(args.out, "w") as f:
            json.dump({"peaks": peaks, "rows": results, "multicast": bs.has_multicast()}, f, indent=1)
    del bs
    dear.shutdown()


if __name__ == "__main__":
    main()
