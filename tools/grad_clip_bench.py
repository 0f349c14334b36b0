"""Kernel A (reduce-scatter) and Kernel B (update + all-gather) time with and without global-norm clipping.

    python tools/grad_clip_bench.py [--world 1 2] [--mb 1 25 100] [--repeats 3] [--out FILE]

Times one fp32 bucket of each size through ``BucketSet`` with CUDA events (mean over --iters launches after --warmup),
clipping off and on (``set_clip``: Kernel A sums the squares of the shard, the update kernel decides and applies the
coefficient).  Off and on alternate --repeats times in the same process, so the spread between repeats of one setting
can be compared with the difference between the settings.  Ranks of --world 2 share the GPU through CUDA IPC.  Prints
one JSON line per row, with the GPU's name and power limit.
"""
import argparse
import json
import os
import socket
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch
import torch.multiprocessing as mp


def _card():
    """(name, power limit in W) of the GPU the numbers were measured on."""
    import subprocess
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        name, power = [x.strip() for x in out.strip().split(",")[:2]]
        return name, float(power)
    except Exception:                                     # no nvidia-smi: the name alone
        return torch.cuda.get_device_name(), None


def _bench(rank, world, port, mbs, iters, warmup, repeats, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank), LOCAL_WORLD_SIZE=str(world))
    import dear_pytorch_b200 as dear
    from dear_pytorch_b200 import ops
    dear.init(backend="b200")
    C, comm, dev = ops.require_native(), dear.communicator(), dear.device()
    gpu, power = _card()
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
        st = torch.zeros(C.clip_state_floats(1), dtype=torch.float32, device=dev)
        st[0] = 1e-3                                      # well below the norm: the clip bites on every step
        st.view(torch.int32)[3] = 1
        for rep in range(repeats):
            for clip_on in (False, True):
                bs.set_clip(st if clip_on else None, [0])
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
                            bs.allgather_update(0, True, False, True, False, clip_on)
                            bs.wait_bucket(0)
                    ev[1].record()
                    torch.cuda.synchronize()
                    times[kernel] = ev[0].elapsed_time(ev[1]) * 1e3 / iters
                    if kernel == "A":
                        bs.allgather_update(0, True, False, True, False, clip_on)
                        bs.wait_bucket(0)
                        torch.cuda.synchronize()
                rows.append(dict(gpu=gpu, power_limit_w=power, world=world, rank=rank, mb=mb, repeat=rep, clip=clip_on,
                                 kernel_a_us=round(times["A"], 2), kernel_b_us=round(times["B"], 2)))
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
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("grad_clip_bench needs a GPU")
    ctx = mp.get_context("spawn")
    for world in args.world:
        s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
        q = ctx.Queue()
        procs = [ctx.Process(target=_bench, args=(r, world, port, args.mb, args.iters, args.warmup,
                                                    args.repeats, q)) for r in range(world)]
        for p in procs:
            p.start()
        rows = [r for _ in procs for r in q.get(timeout=600)]
        for p in procs:
            p.join()
        for r in sorted(rows, key=lambda r: (r["mb"], r["repeat"], r["clip"], r["rank"])):
            if r["rank"] != 0:
                continue
            line = json.dumps(r)
            print(line, flush=True)
            if args.out:
                with open(args.out, "a") as f:
                    f.write(line + "\n")


if __name__ == "__main__":
    main()
