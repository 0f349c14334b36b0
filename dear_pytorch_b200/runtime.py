"""Process-group runtime: rendezvous, device pinning, backend selection.

Reference behaviour being replaced: importing ``dear`` runs ``MPI_Init``
(dear/dear_dopt.py:37), ``dear.init()`` builds three NCCL communicators
(dear/dear_dopt.py:45-51) and drivers pin ``rank() % 4`` (dear/imagenet_benchmark.py:65).

Here:
  * launch is ``torchrun`` / env:// (RANK, WORLD_SIZE, LOCAL_RANK, MASTER_ADDR, MASTER_PORT);
    no MPI.  A process started without those variables is a world of one.
  * the device is pinned from LOCAL_RANK (not a hard-coded ``% 4``).
  * ``backend`` selects the data path of the decoupled all-reduce:
      "b200"  our fused sm_90a kernels over peer-mapped NVLink memory  (default on GPU)
      "emu"   the same native runtime executed on the host over POSIX shm (CPU tests)
      "nccl"  torch.distributed NCCL collectives + eager update          (baseline)
      "gloo"  torch.distributed gloo collectives + eager update          (CPU plumbing)
"""
from __future__ import annotations

import datetime
import os
from dataclasses import dataclass, field
from typing import Optional

import torch
import torch.distributed as dist

from . import ops

_BACKENDS = ("b200", "emu", "nccl", "gloo")


@dataclass
class _State:
    backend: str
    rank: int
    world: int
    local_rank: int
    local_size: int
    device: torch.device
    comm: object = None            # native Communicator (b200 / emu)
    group: object = None           # torch.distributed group (object broadcast, baselines)
    owns_pg: bool = False
    options: dict = field(default_factory=dict)


_state: Optional[_State] = None


def _env_int(name, default):
    v = os.environ.get(name)
    return default if v in (None, "") else int(v)


def is_initialized() -> bool:
    return _state is not None


def _require() -> _State:
    if _state is None:
        raise RuntimeError("dear is not initialised: call dear.init() first")
    return _state


def init(backend: Optional[str] = None, device: Optional[torch.device] = None, *, nstreams: int = 1,
         staging_mb: Optional[int] = None, provider: Optional[str] = None,
         multicast: Optional[bool] = None, timeout_s: float = 600.0) -> None:
    """Initialise the runtime (idempotent).

    Must be called by every rank.  Unlike the reference there is no ordering
    constraint with device selection: the device is pinned here.
    """
    global _state
    if _state is not None:
        return
    timeout_s = float(os.environ.get("DEAR_TIMEOUT_S", timeout_s))
    rank = _env_int("RANK", 0)
    world = _env_int("WORLD_SIZE", 1)
    local_rank = _env_int("LOCAL_RANK", rank)
    local_size = _env_int("LOCAL_WORLD_SIZE", world)

    use_cuda = torch.cuda.is_available() and (device is None or torch.device(device).type == "cuda")
    backend = select_backend(backend or os.environ.get("DEAR_BACKEND"), use_cuda, world, local_size, verbose=(rank == 0))
    if backend in ("b200", "nccl") and not torch.cuda.is_available():
        raise RuntimeError("backend %r needs a CUDA device" % backend)
    if backend in ("emu", "gloo"):
        use_cuda = False

    if use_cuda:
        if device is None:
            device = torch.device("cuda", local_rank % torch.cuda.device_count())
        device = torch.device(device)
        torch.cuda.set_device(device)
    else:
        device = torch.device("cpu")

    global _kept_pg
    owns_pg = _kept_pg and dist.is_initialized()       # a group this module created and kept over a shutdown()
    _kept_pg = False
    group = None
    store = None
    if world > 1 or dist.is_initialized():
        if not dist.is_initialized():
            os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
            os.environ.setdefault("MASTER_PORT", "29500")
            # NCCL is registered for CUDA tensors but initialised lazily: the fused
            # path never touches it, only the baselines (nccl backend, DDP, WFBP) do.
            pg_backend = "cpu:gloo,cuda:nccl" if use_cuda else "gloo"
            dist.init_process_group(pg_backend, rank=rank, world_size=world,
                                    timeout=datetime.timedelta(seconds=timeout_s))
            owns_pg = True
        rank, world = dist.get_rank(), dist.get_world_size()
        group = dist.group.WORLD
        from torch.distributed.distributed_c10d import _get_default_store
        store = _get_default_store()

    comm = None
    opts = {}
    if backend in ("b200", "emu"):
        C = ops.require_native()
        if world > C.MAX_RANKS:
            raise RuntimeError("the symmetric-memory backend spans one NVSwitch domain (<= %d ranks)" % C.MAX_RANKS)
        o = C.CommOptions()
        o.device = device.index if backend == "b200" else -1
        o.nstreams = max(1, int(nstreams))
        o.staging_bytes = int(staging_mb if staging_mb is not None else _env_int("DEAR_STAGING_MB", 32)) << 20
        prov = (provider or os.environ.get("DEAR_PROVIDER") or "ipc").lower()
        if prov not in ("ipc", "vmm"):
            raise ValueError("DEAR_PROVIDER must be 'ipc' or 'vmm'")
        o.provider = C.PROVIDER_CUDA_VMM if prov == "vmm" else C.PROVIDER_CUDA_IPC
        if multicast is None:
            multicast = os.environ.get("DEAR_MULTICAST", "0") not in ("0", "", "false", "False")
        o.multicast = bool(multicast) and prov == "vmm"
        o.spin_timeout_s = float(os.environ.get("DEAR_SPIN_TIMEOUT_S", "60"))
        o.rendezvous_timeout_s = float(timeout_s)
        # CTAs of the fused kernels (upper bounds; small buckets get fewer, csrc/communicator.cpp: grid_for).  On one GPU
        # nothing ever spins, so the kernels may take most of the chip for a few microseconds (HBM-bound).  With peers
        # the pull is NVLink-bound from ~32 CTAs on, but the PACK phase of Kernel A and the push of Kernel B scale with
        # the CTA count (tools/kernel_bench.py sweeps it).
        o.rs_grid = _env_int("DEAR_RS_GRID", 128 if world == 1 else 64)
        o.ag_grid = _env_int("DEAR_AG_GRID", 128 if world == 1 else 48)
        o.gen_grid = _env_int("DEAR_GEN_GRID", 8)
        # Kernel A variant per bucket: by size unless forced (DEAR_RS_ALGO=oneshot|pipe|nvls); csrc/communicator.h
        algo = os.environ.get("DEAR_RS_ALGO", "auto").lower()
        if algo not in ("auto", "oneshot", "pipe", "nvls"):
            raise ValueError("DEAR_RS_ALGO must be auto, oneshot, pipe or nvls")
        o.rs_algo = {"auto": -1, "oneshot": 0, "pipe": 1, "nvls": 2}[algo]
        if "DEAR_PIPE_MIN_MB" in os.environ:      # auto mode: buckets at least this large use the pipelined variant
            o.pipe_min_bytes = int(float(os.environ["DEAR_PIPE_MIN_MB"]) * (1 << 20))
        o.rs_grid_big = _env_int("DEAR_RS_GRID_BIG", 128)
        o.stripe_target_bytes = int(float(os.environ.get("DEAR_STRIPE_MB", "8")) * (1 << 20))
        o.separate_ag_stream = os.environ.get("DEAR_AG_STREAM", "1") not in ("0", "false", "False")
        # rendezvous keys must be unique per init(): a re-initialised process group can land on the SAME TCPStore server
        # (multi-tenant stores are shared per port), where the previous communicator's barrier counters still exist
        global _init_seq
        _init_seq += 1
        comm = C.Communicator(rank, world, store, "dear%d_%d" % (_env_int("DEAR_JOB_SEQ", 0), _init_seq), o)
        opts = dict(provider=prov, multicast=o.multicast, rs_grid=o.rs_grid, ag_grid=o.ag_grid, rs_algo=algo,
                    separate_ag_stream=o.separate_ag_stream)

    _state = _State(backend=backend, rank=rank, world=world, local_rank=local_rank, local_size=local_size,
                    device=device, comm=comm, group=group, owns_pg=owns_pg, options=opts)


_kept_pg = False       # shutdown(destroy_process_group=False) left a group that this module owns
_init_seq = 0          # init() calls that created a native communicator in this process (identical on every rank)


def select_backend(requested: Optional[str], use_cuda: bool, world: int, local_size: int, verbose: bool = False) -> str:
    """Resolve the data path.  The fused kernels move data through peer-mapped memory, which exists inside ONE
    NVLink/NVSwitch domain (one node): a job that spans several nodes (``LOCAL_WORLD_SIZE < WORLD_SIZE``, e.g.
    ``scripts/launch_multinode.sh``) runs the same engine on the ``nccl`` backend instead — the reference's own
    transport (common/comm_core/communicator.cpp:85-127) — unless ``b200`` was requested explicitly."""
    multi_node = 0 < local_size < world
    if requested is None:
        if not use_cuda:
            return "gloo"
        if multi_node:
            if verbose:
                print("[dear] %d ranks over %d nodes: the symmetric-memory kernels span one NVSwitch domain; "
                      "using the nccl backend" % (world, world // local_size), flush=True)
            return "nccl"
        return "b200"
    if requested not in _BACKENDS:
        raise ValueError("unknown backend %r (choose from %s)" % (requested, ", ".join(_BACKENDS)))
    if requested in ("b200", "emu") and multi_node:
        raise RuntimeError("backend %r needs all %d ranks on one node (LOCAL_WORLD_SIZE=%d); use DEAR_BACKEND=nccl "
                           "across nodes" % (requested, world, local_size))
    return requested


def shutdown(destroy_process_group: bool = True) -> None:
    """Tear the runtime down (streams, arenas, process group).

    To re-initialise inside the same process pass ``destroy_process_group=False``: the next ``init()`` then reuses the
    ``torch.distributed`` group (re-creating one on the same MASTER_PORT races with peers that still see the old
    rendezvous store), while the native communicator, its streams and every symmetric arena are released — provided the
    engines were closed first (``optimizer.engine.close()`` hands the parameters back from the buckets)."""
    global _state
    if _state is None:
        return
    st = _state
    try:
        if st.comm is not None:
            st.comm.synchronize()
        if st.owns_pg and destroy_process_group and dist.is_initialized() and st.world > 1:
            # leave together: rank 0 hosts the rendezvous store, and a later init() in the same process re-creates it
            # on the same port — a rank still inside the old group would see its connection reset
            try:
                dist.barrier(group=st.group)
            except Exception:      # a peer already died: tear down anyway
                pass
    finally:
        _state = None
        st.comm = None
        if st.owns_pg and dist.is_initialized():
            if destroy_process_group:
                dist.destroy_process_group()
            else:
                global _kept_pg
                _kept_pg = True


def rank() -> int:
    return _require().rank if _state is not None else _env_int("RANK", 0)


def size() -> int:
    return _require().world if _state is not None else _env_int("WORLD_SIZE", 1)


def local_rank() -> int:
    return _require().local_rank if _state is not None else _env_int("LOCAL_RANK", 0)


def local_size() -> int:
    return _require().local_size if _state is not None else _env_int("LOCAL_WORLD_SIZE", 1)


def backend() -> str:
    return _require().backend


def device() -> torch.device:
    return _require().device


def communicator():
    """The native Communicator (``None`` for the nccl / gloo backends)."""
    return _require().comm


def group():
    return _require().group


def barrier() -> None:
    st = _require()
    if st.world == 1:
        return
    if st.comm is not None:
        st.comm.barrier()
    else:
        dist.barrier()


def broadcast_object(obj, src: int = 0):
    """Broadcast a small picklable Python object from ``src`` (tuner decisions, flags)."""
    st = _require()
    if st.world == 1:
        return obj
    box = [obj]
    try:
        dist.broadcast_object_list(box, src=src, group=st.group, device=torch.device("cpu"))
    except (RuntimeError, ValueError):
        # a user-created NCCL-only process group has no CPU backend: stage through the GPU
        dist.broadcast_object_list(box, src=src, group=st.group, device=st.device)
    return box[0]
