"""Kernel A (reduce-scatter) and Kernel B (update + all-gather) time with and without dynamic loss scaling.

    python tools/grad_scaler_bench.py [--world 1 2] [--mb 1 25 100] [--root DIR] [--out FILE]

Times one fp32 bucket of each size through ``BucketSet`` with CUDA events (mean over --iters launches after --warmup),
scaler off (static path) and on (``set_amp``: the update kernel decides, every step applies).  ``--root`` imports the
package from another checkout, so two builds can be timed in the same run; a build without ``BucketSet.set_amp``
reports the scaler-off rows only.  Ranks of --world 2 share the GPU through CUDA IPC.  Prints one JSON line per row.
"""
import argparse
import json
import os
import socket
import sys

import torch
import torch.multiprocessing as mp


def _bench(rank, world, port, root, mbs, iters, warmup, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank), LOCAL_WORLD_SIZE=str(world))
    sys.path.insert(0, root)
    import dear_pytorch_b200 as dear
    from dear_pytorch_b200 import ops
    dear.init(backend="b200")
    C, comm, dev = ops.require_native(), dear.communicator(), dear.device()
    rows = []
    for mb in mbs:
        n = int(mb * (1 << 20)) // 4 // (16 * world) * (16 * world)
        bs = C.BucketSet(comm, [n], C.DT_F32, True)
        shard = n // world
        gshard, mom = torch.zeros(shard, device=dev), torch.zeros(shard, device=dev)
        bs.set_shards(0, gshard, mom, None, None)
        bs.set_hyper(0, [n], [1e-3], [0.0], [0.9], [0.0], [0])
        grad = torch.randn(n, device=dev) * 1e-3
        bs.set_pack(0, [grad.data_ptr()], [0], [n * 4], [0])
        for amp_on in ((False, True) if hasattr(bs, "set_amp") else (False,)):
            if amp_on:
                st = torch.zeros(9, dtype=torch.int32, device=dev)
                f = st.view(torch.float32)
                f[2], f[5], f[6], st[7] = 1024.0, 2.0, 0.5, 1 << 30
                bs.set_amp(st)
            times = {}
            for kernel in ("A", "B"):
                ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
                for i in range(warmup + iters):
                    if i == warmup:
                        ev[0].record()
                    if kernel == "A":
                        bs.reduce_scatter(0, True)
                        bs.wait_rs(0)
                    else:
                        kw = {"decide": True} if amp_on else {}
                        bs.allgather_update(0, True, False, True, False, **kw)
                        bs.wait_bucket(0)
                ev[1].record()
                torch.cuda.synchronize()
                times[kernel] = ev[0].elapsed_time(ev[1]) * 1e3 / iters
                if kernel == "A":
                    bs.allgather_update(0, True, False, True, False, **({"decide": True} if amp_on else {}))
                    bs.wait_bucket(0)
                    torch.cuda.synchronize()
            rows.append(dict(root=root, world=world, rank=rank, mb=mb, scaler=amp_on, kernel_a_us=round(times["A"], 2),
                             kernel_b_us=round(times["B"], 2)))
        comm.synchronize()
        del bs
    comm.check_status()
    dear.shutdown()
    q.put(rows)


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--world", type=int, nargs="+", default=[1, 2])
    ap.add_argument("--mb", type=float, nargs="+", default=[1, 25, 100])
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("grad_scaler_bench needs a GPU")
    ctx = mp.get_context("spawn")
    for world in args.world:
        s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
        q = ctx.Queue()
        procs = [ctx.Process(target=_bench, args=(r, world, port, os.path.abspath(args.root), args.mb, args.iters,
                                                    args.warmup, q)) for r in range(world)]
        for p in procs:
            p.start()
        rows = [r for _ in procs for r in q.get(timeout=600)]
        for p in procs:
            p.join()
        for r in sorted(rows, key=lambda r: (r["mb"], r["scaler"], r["rank"])):
            if r["rank"] != 0:
                continue
            line = json.dumps(r)
            print(line, flush=True)
            if args.out:
                with open(args.out, "a") as f:
                    f.write(line + "\n")


if __name__ == "__main__":
    main()
