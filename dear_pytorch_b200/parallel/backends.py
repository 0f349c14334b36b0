"""Data-path backends of the DeAR engine.

``NativeBackend``  (b200 / emu): symmetric buckets + the two fused kernels of
                   csrc/kernels.cu (or their host emulation) — no NCCL call and no separate
                   elementwise kernel on either the backward or the forward path.
``TorchBackend``   (nccl / gloo): the same bucket layout driven by
                   ``torch.distributed.reduce_scatter_tensor`` / ``all_gather_into_tensor`` and
                   the optimizer family's eager sharded update (parallel/families.py) — the
                   comparison baseline and the CPU plumbing path.  This is what the reference
                   does per bucket (dear/tensorfusion.py:469-482, dear/dear_dopt.py:293-336),
                   minus its per-parameter loops.

Both expose the same interface to ``parallel.optimizer``:
  param_buffer(g) / grad_buffer(g)      flat bucket tensors (parameters / gradients are views)
  reduce_scatter(g, pack)               backward-path collective (+ 1/P scale)
  allgather_update(g, ...)              forward-path collective (+ sharded update)
  wait_bucket(g) / wait_all() / fence() / synchronize()
"""
from __future__ import annotations

from typing import Dict, List, Optional, Tuple

import torch
import torch.distributed as dist

from .. import ops
from .bucket import BucketPlan
from .families import HYPER_SKIP, HyperRow

_DT_CODE = {torch.float32: "DT_F32", torch.bfloat16: "DT_BF16", torch.float16: "DT_F16"}
SHARD_KINDS = ("mom", "var", "gavg", "master")    # a bucket's fp32 shards: family state (parallel/families.py), master


class _BackendBase:
    steal_grads = False

    def __init__(self, family, plan: BucketPlan, rank: int, world: int, device: torch.device,
                 grad_comm_dtype: Optional[torch.dtype] = None):
        self.family = family            # parallel/families.py: which state shards a bucket needs, the eager update
        self.plan = plan
        self.rank = rank
        self.world = world
        self.device = device
        # fp32 gradients travel as this 16-bit dtype (DearEngine.grad_comm_dtype); one rank has no wire
        self.wire = grad_comm_dtype if world > 1 else None
        nb = len(plan.buckets)
        self.grad_shard: List[torch.Tensor] = [None] * nb
        self.shards: List[Dict[str, torch.Tensor]] = [{} for _ in range(nb)]     # per bucket: kind -> fp32 shard
        self.hyper: List[Optional[Tuple[HyperRow, ...]]] = [None] * nb
        self.grad_scale = 1.0
        self.amp: Optional[torch.Tensor] = None     # dynamic loss scaler state (parallel/grad_scaler.py), engine-owned
        self.clip: Optional[torch.Tensor] = None    # global-norm clipping state (ClipState, csrc/dear_common.h), engine-owned

    # -- shard state ------------------------------------------------------------------
    def _alloc_shards(self):
        for b in self.plan.buckets:
            self.grad_shard[b.index] = torch.zeros(b.shard_numel, dtype=torch.float32, device=self.device)

    def init_master_shards(self):
        """fp32 master copy of this rank's shard for low-precision parameter buckets."""
        for b in self.plan.buckets:
            if b.dtype != torch.float32:
                lo = self.rank * b.shard_numel
                self.shards[b.index]["master"] = self.param_buffer(b.index)[lo:lo + b.shard_numel].float().clone()
        self._shards_changed()

    def ensure_state(self, g: int, kind: str) -> torch.Tensor:
        """The ``kind`` state shard of bucket g, allocated (zeroed) on first use."""
        shard = self.shards[g].get(kind)
        if shard is None:
            shard = self.shards[g][kind] = torch.zeros(self.plan.buckets[g].shard_numel, dtype=torch.float32,
                                                       device=self.device)
            self._shards_changed(g)
        return shard

    def _shards_changed(self, g: Optional[int] = None):
        pass

    def set_step(self, t: int) -> None:
        """Number of updates already applied (Adam bias correction); called after (re)building buckets."""
        pass

    def set_hyper(self, g: int, rows: Tuple[HyperRow, ...]) -> None:
        """Hyper-parameter rows of bucket g (sorted by ``end``, covering the bucket); allocates the state they need."""
        self.hyper[g] = rows
        for kind in self.family.shard_kinds(rows):
            self.ensure_state(g, kind)

    def launches(self) -> int:
        return 0

    def set_grad_scale(self, s: float) -> None:
        """Extra factor applied to the averaged gradient (1/loss_scale for static loss scaling)."""
        self.grad_scale = float(s)

    def stream_key(self, g: int) -> int:
        """Buckets with the same key share one communication stream (ordering domain)."""
        return 0

    def set_amp(self, state: Optional[torch.Tensor]) -> None:
        """Dynamic loss scaling: ``state`` is the engine's int32[9] AmpState (csrc/dear_common.h), or None."""
        self.amp = state

    def clip_state_numel(self) -> int:
        """float32 elements of the engine's clipping state (words 0-2: max_norm, total_norm, coef)."""
        return 4

    def set_clip(self, state: Optional[torch.Tensor]) -> None:
        """Global-norm clipping: ``state`` is the engine's float32 ClipState, or None."""
        self.clip = state


# =====================================================================================
# native: b200 kernels / host emulation
# =====================================================================================
class NativeBackend(_BackendBase):
    steal_grads = True

    def __init__(self, comm, family, plan: BucketPlan, rank: int, world: int, device: torch.device,
                 grad_comm_dtype: Optional[torch.dtype] = None):
        super().__init__(family, plan, rank, world, device, grad_comm_dtype)
        C = ops.require_native()
        self.C = C
        self.comm = comm
        # one native BucketSet per dtype; bucket g -> (set, local index)
        by_dtype: Dict[torch.dtype, List[int]] = {}
        for b in plan.buckets:
            if b.dtype not in _DT_CODE:
                raise TypeError("unsupported parameter dtype %s" % b.dtype)
            by_dtype.setdefault(b.dtype, []).append(b.index)
        self.sets = {}
        self.where: List[Tuple[object, int]] = [None] * len(plan.buckets)
        for dt, idxs in by_dtype.items():
            # fp32 sets with a wire dtype are converting sets: 16-bit gradient buckets, the pack rounds
            wire = self.wire if dt == torch.float32 and self.wire is not None else dt
            bs = C.BucketSet(comm, [plan.buckets[g].padded_numel for g in idxs], getattr(C, _DT_CODE[dt]), True,
                             getattr(C, _DT_CODE[wire]))
            self.sets[dt] = bs
            for li, g in enumerate(idxs):
                self.where[g] = (bs, li)
        self._pbuf = [bs.param_buffer(li) for bs, li in self.where]
        self._gbuf = [bs.grad_buffer(li) for bs, li in self.where]
        self._alloc_shards()
        self._shards_changed()
        self._first_in_set = {id(bs): min(g for g, (s, _) in enumerate(self.where) if s is bs)
                              for bs in self.sets.values()}

    @property
    def has_multicast(self) -> bool:
        return any(bs.has_multicast() for bs in self.sets.values())

    def param_buffer(self, g):
        return self._pbuf[g]

    def grad_buffer(self, g):
        return self._gbuf[g]

    def _shards_changed(self, g=None):
        for i in (range(len(self.where)) if g is None else (g,)):
            bs, li = self.where[i]
            if self.grad_shard[i] is not None:
                sh = self.shards[i]
                bs.set_shards(li, self.grad_shard[i], sh.get("mom"), sh.get("master"), sh.get("var"), sh.get("gavg"))

    def set_hyper(self, g, rows):
        if self.hyper[g] == rows:
            return
        super().set_hyper(g, rows)
        bs, li = self.where[g]
        bs.set_hyper(li, *(list(col) for col in zip(*rows)))    # one list per HyperRow field

    def set_step(self, t: int):
        for i, (bs, li) in enumerate(self.where):
            bs.set_step(li, int(t))

    def set_pack(self, g, src_ptrs, dst_off, nbytes, flags):
        bs, li = self.where[g]
        bs.set_pack(li, src_ptrs, dst_off, nbytes, flags)

    def reduce_scatter(self, g, pack=True):
        bs, li = self.where[g]
        bs.reduce_scatter(li, pack)

    def set_amp(self, state):
        self.amp = state
        for bs in self.sets.values():
            bs.set_amp(state)

    def clip_state_numel(self):
        return self.C.clip_state_floats(len(self.where))

    def set_clip(self, state):
        # slots are the engine-wide bucket indices: Kernel A of bucket g writes its sum of squares to slot g
        self.clip = state
        for bs in self.sets.values():
            bs.set_clip(state, [g for g, (s, _) in enumerate(self.where) if s is bs])

    def allgather_update(self, g, do_update=True, first_step=False, zero_grad=False):
        bs, li = self.where[g]
        # the first bucket of every set carries the entry rendezvous: nobody overwrites a
        # peer's parameters before that peer has finished its backward pass.
        entry = self._first_in_set[id(bs)] == g
        # dynamic loss scaling and global-norm clipping: bucket 0's update decides for the whole step.  With several
        # dtype sets it waits for every set's reduce-scatters, and the other sets' first updates wait for it.
        deciding = self.amp is not None or self.clip is not None
        decide = deciding and g == 0 and do_update
        if deciding and entry and len(self.sets) > 1:
            for other in (self.sets.values() if decide else (self.where[0][0],)):
                bs.join(other)
        bs.allgather_update(li, do_update, first_step, entry, zero_grad, decide)

    def fence(self):
        for bs in self.sets.values():
            bs.fence_current_to_comm()

    def wait_bucket(self, g):
        bs, li = self.where[g]
        bs.wait_bucket(li)

    def wait_all(self):
        for bs in self.sets.values():
            bs.wait_all()

    def synchronize(self):
        for bs in self.sets.values():
            bs.synchronize()

    def launches(self):
        return self.comm.launches()

    def set_grad_scale(self, s):
        self.grad_scale = float(s)
        for bs in self.sets.values():
            bs.set_grad_scale(float(s))

    def stream_key(self, g):
        return id(self.where[g][0])


# =====================================================================================
# torch.distributed: nccl / gloo
# =====================================================================================
class TorchBackend(_BackendBase):
    steal_grads = False

    def __init__(self, group, family, plan: BucketPlan, rank: int, world: int, device: torch.device,
                 grad_comm_dtype: Optional[torch.dtype] = None):
        super().__init__(family, plan, rank, world, device, grad_comm_dtype)
        self.group = group
        self.cuda = device.type == "cuda"
        self._pbuf = [torch.zeros(b.padded_numel, dtype=b.dtype, device=device) for b in plan.buckets]
        self._gbuf = [torch.zeros(b.padded_numel, dtype=b.dtype, device=device) for b in plan.buckets]
        self._rs_out = [torch.zeros(b.shard_numel, dtype=b.dtype, device=device) for b in plan.buckets]
        self._alloc_shards()
        self._n_launch = 0
        self._t = 0                      # updates applied so far (Adam bias correction)
        if self.cuda:
            self.stream = torch.cuda.Stream(device=device, priority=-1)
            self.ag_done = [torch.cuda.Event() for _ in plan.buckets]
            self._pending = [False] * len(plan.buckets)

    def param_buffer(self, g):
        return self._pbuf[g]

    def grad_buffer(self, g):
        return self._gbuf[g]

    def set_step(self, t: int):
        self._t = int(t)

    def set_amp(self, state):
        self.amp = state
        self._overflow = None if state is None else torch.zeros((), dtype=torch.float32, device=self.device)
        self._skip = False

    def _amp_decide(self):
        """One decision per step: did any rank see a non-finite reduced gradient?  Then skip every bucket's update;
        the scale and growth tracker follow torch.amp.GradScaler (torch._amp_update_scale_)."""
        found = self._overflow.reshape(1).clone()
        if self.world > 1:
            dist.all_reduce(found, op=dist.ReduceOp.MAX, group=self.group)
        st, f32 = self.amp, self.amp.view(torch.float32)
        st[8] = st[3]
        torch._amp_update_scale_(f32[2:3], st[3:4], found, float(f32[5]), float(f32[6]), int(st[7]))
        self._skip = bool(found.item())
        st[1] = int(self._skip)
        if not self._skip:
            st[4] += 1
        self._overflow.zero_()

    @torch.no_grad()
    def _clip_decide(self):
        """``torch.nn.utils.clip_grad_norm_`` over the averaged gradient: after the reduce-scatters every rank holds 1/P
        of it exactly once, so the norm is one pass over the fp32 shards plus a one-element all-reduce.  The
        coefficient is applied in the update (``_update_shard``).  Eager steps only."""
        if self.cuda and torch.cuda.is_current_stream_capturing():
            raise RuntimeError("norm_clip is not supported inside a CUDA-graph capture on the nccl backend")
        shards = [s for s in self.grad_shard if s is not None]
        sq = torch.stack(torch._foreach_norm(shards)).pow(2).sum().reshape(1)       # no shard-sized temporaries
        if self.world > 1:
            dist.all_reduce(sq, group=self.group)
        total = sq.sqrt()
        self.clip[1:2].copy_(total)
        self.clip[2:3].copy_((self.clip[0:1] / (total + 1e-6)).clamp(max=1.0))

    def set_pack(self, g, src_ptrs, dst_off, nbytes, flags):
        pass    # gradients are accumulated straight into the bucket views

    def _on_comm_stream(self):
        if self.cuda:
            return torch.cuda.stream(self.stream)
        import contextlib
        return contextlib.nullcontext()

    def reduce_scatter(self, g, pack=True):
        if self.cuda:
            self.stream.wait_stream(torch.cuda.current_stream(self.device))
        with self._on_comm_stream():
            if self.wire is not None and self._gbuf[g].dtype == torch.float32:
                # the fused backends' rounding (grad_comm_dtype) before the same fp32 collective: same arithmetic up to
                # the summation order, no bandwidth saved
                self._gbuf[g].copy_(self._gbuf[g].to(self.wire))
            if self.world > 1:
                dist.reduce_scatter_tensor(self._rs_out[g], self._gbuf[g], op=dist.ReduceOp.SUM, group=self.group)
            else:
                self._rs_out[g].copy_(self._gbuf[g])
            torch.mul(self._rs_out[g].float(), self.grad_scale / self.world, out=self.grad_shard[g])
            if self.amp is not None:
                self.grad_shard[g].mul_(self.amp.view(torch.float32)[2].reciprocal())
                torch.maximum(self._overflow, (~torch.isfinite(self.grad_shard[g])).any().float(), out=self._overflow)
            self._gbuf[g].zero_()
        self._n_launch += 3

    @torch.no_grad()
    def _update_shard(self, g, first_step):
        if self.amp is not None:
            if self._skip:
                return
            first_step = self._t == 0             # counts applied updates only
        b = self.plan.buckets[g]
        lo, hi = self.rank * b.shard_numel, (self.rank + 1) * b.shard_numel
        master = self.shards[g].get("master")
        start = 0
        for row in self.hyper[g]:
            a, z = max(start, lo), min(row.end, hi)
            start = row.end
            if a >= z:
                continue
            if row.flags & HYPER_SKIP and not bool(self.grad_shard[g][a - lo:z - lo].any()):
                continue                          # no gradient on ANY rank this step: parameter and state stay as they are
            sl = slice(a - lo, z - lo)
            p = master[sl] if master is not None else self._pbuf[g][a:z]
            d = self.grad_shard[g][sl]
            if self.clip is not None:
                d = d * self.clip[2]
            self._n_launch += self.family.update(row, p, d, self.shards[g], sl, first_step, self._t)

    def allgather_update(self, g, do_update=True, first_step=False, zero_grad=False):
        b = self.plan.buckets[g]
        lo = self.rank * b.shard_numel
        with self._on_comm_stream():
            if do_update and g == 0 and self.amp is not None:
                self._amp_decide()
            if do_update and g == 0 and self.clip is not None:
                self._clip_decide()
            if do_update:
                self._update_shard(g, first_step)
            if "master" in self.shards[g]:
                src = self.shards[g]["master"].to(b.dtype)
            else:
                src = self._pbuf[g][lo:lo + b.shard_numel].clone()
            if self.world > 1:
                dist.all_gather_into_tensor(self._pbuf[g], src, group=self.group)
            else:
                self._pbuf[g][lo:lo + b.shard_numel].copy_(src)
            if do_update and g == len(self.plan.buckets) - 1 and not (self.amp is not None and self._skip):
                self._t += 1
            if self.cuda:
                self.ag_done[g].record(self.stream)
                self._pending[g] = True
        self._n_launch += 2

    def fence(self):
        if self.cuda:
            self.stream.wait_stream(torch.cuda.current_stream(self.device))

    def wait_bucket(self, g):
        if self.cuda and self._pending[g]:
            torch.cuda.current_stream(self.device).wait_event(self.ag_done[g])

    def wait_all(self):
        if self.cuda:
            torch.cuda.current_stream(self.device).wait_stream(self.stream)

    def synchronize(self):
        if self.cuda:
            self.stream.synchronize()

    def launches(self):
        return self._n_launch
