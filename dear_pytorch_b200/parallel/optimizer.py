"""DeAR distributed optimizer: decoupled all-reduce with tensor fusion.

Public behaviour follows the reference's ``dear.DistributedOptimizer``
(dear/dear_dopt.py:56-398): gradients of iteration *t* are reduce-scattered per fusion
bucket while the backward pass is still running, and the matching all-gather plus the
SGD update are overlapped with the forward pass of iteration *t+1*.  The result is
mathematically identical to synchronous data-parallel SGD.

GPU-first redesign (SURVEY.md §7, §9):
  * parameters live in flat symmetric *parameter buckets* (``p.data`` is a view) and the
    update is **sharded**: each rank updates 1/P of every bucket (momentum and fp32 master
    state are sharded too) and pushes the result into every peer's bucket — Kernel B;
  * gradients are handed to Kernel A by pointer (``p.grad`` is whatever autograd produced;
    no per-parameter copy/scale/zero kernels), reduced over NVLink and scaled by 1/P once;
  * nothing on the hot path blocks the host: ordering is stream events and in-kernel flags.
    The reference blocks on ``cudaStreamSynchronize`` per bucket (dear/dear_dopt.py:284,352);
  * all parameter updates are issued at ``step()`` (asynchronously, in forward order), so the
    last iteration's update is not lost (reference defect, dear/dear_dopt.py:371) and an
    extra forward pass never re-applies a gradient (reference defect, :278);
  * each parameter uses the hyper-parameters of *its own* param group (the reference loops
    over all groups for every parameter, dear/dear_dopt.py:312-335);
  * reduce-scatters are issued in a rank-consistent order (descending bucket index), and
    buckets whose parameters received no gradient are flushed at ``step()`` with zeros.
"""
from __future__ import annotations

import math
import os
from typing import Dict, List, Optional

import torch
import torch.nn as nn

from .. import runtime
from .backends import HYPER_SKIP, OPT_ADAM, OPT_ADAMW, OPT_SGD, HyperSpec, NativeBackend, TorchBackend
from .bucket import BucketPlan

import weakref

THRESHOLD = 25            # MB, reference default (dear/dear_dopt.py:43)
_LIVE_ENGINES = weakref.WeakSet()   # engines whose buckets currently hold their model's parameters


def live_engines():
    return [e for e in list(_LIVE_ENGINES) if not e._closed and e.backend is not None]
NUM_NEARBY_LAYERS = 4     # reference default (dear/dear_dopt.py:42)


def _dense_like(p: torch.Tensor) -> bool:
    return p.is_contiguous() or p.is_contiguous(memory_format=torch.channels_last) or \
        (p.dim() == 5 and p.is_contiguous(memory_format=torch.channels_last_3d))


class DearEngine:
    """Buffers, hooks and the per-bucket state machine behind ``DistributedOptimizer``."""

    def __init__(self, optimizer: torch.optim.Optimizer, model: nn.Module, *, threshold=THRESHOLD,
                 num_nearby_layers=NUM_NEARBY_LAYERS, exclude_parts: str = "", policy=None, verbose=True,
                 backward_passes_per_step: int = 1, grad_comm_dtype: Optional[torch.dtype] = None):
        if grad_comm_dtype not in (None, torch.float32, torch.bfloat16, torch.float16):
            raise ValueError("grad_comm_dtype must be None, torch.float32, torch.bfloat16 or torch.float16; got %r"
                             % (grad_comm_dtype,))
        # fp32 gradients cross the wire as this 16-bit dtype (None: as fp32); fixed for the engine's lifetime
        self._grad_comm_dtype = None if grad_comm_dtype in (None, torch.float32) else grad_comm_dtype
        if not runtime.is_initialized():
            runtime.init()
        self.opt = optimizer
        self.model = model
        self.rank = runtime.rank()
        self.world = runtime.size()
        self.device = runtime.device()
        self.backend_name = runtime.backend()
        self.exclude_reducescatter = "reducescatter" in exclude_parts
        self.exclude_allgather = "allgather" in exclude_parts
        self.verbose = verbose and self.rank == 0
        self.num_steps = 0
        self.threshold = threshold
        self.num_nearby_layers = num_nearby_layers
        self._mom_initialised = False
        self.num_updates = 0               # parameter updates applied so far (Adam bias correction)
        self.amp: Optional[torch.Tensor] = None   # dynamic loss scaler state (attach_scaler), survives re-bucketing
        self._norm_clip: Optional[float] = None    # global-norm clipping (the norm_clip property)
        self.clip: Optional[torch.Tensor] = None  # its device state (ClipState), rebuilt with the buckets
        self.flush_callbacks = []          # run by flush(): deferred work of the training loop (TrainStep.finish)
        if int(backward_passes_per_step) < 1:
            raise ValueError("backward_passes_per_step must be >= 1")
        self.passes_per_step = int(backward_passes_per_step)   # gradient accumulation: reduce on the last pass only
        self._passes_seen = {}             # parameter -> backward passes since the last step()
        if isinstance(optimizer, torch.optim.AdamW):
            self.opt_kind = OPT_ADAMW
        elif isinstance(optimizer, torch.optim.Adam):
            self.opt_kind = OPT_ADAM
        else:
            self.opt_kind = OPT_SGD
        self._hooks = []
        self._closed = False
        self._wt = None                    # optional wait-time recorder (variants.WaitTimeBucketing)
        self._step_callbacks = []          # called at the re-bucketing safe point
        self._safe_point_actions = []

        for p in model.parameters():
            if p.requires_grad and p.device.type != self.device.type:
                raise RuntimeError("model parameters live on %s but the runtime device is %s" % (p.device, self.device))
        # Adam / AdamW: updates a parameter did NOT take part in (no gradient on any rank).  torch.optim keeps the step
        # count per parameter, the kernels keep one per bucket set: _refresh_hyper folds the difference into the
        # parameter's hyper segment (see _adam_lag_adjust)
        self._lag: Dict[nn.Parameter, int] = {}
        # SGD with momentum AND dampening: torch initialises a parameter's momentum buffer with its first gradient
        # (undampened); the kernels know one global "first step".  Parameters that start later get dampening 0 in
        # their hyper segment for that one update (buf = m * 0 + 1 * g).  Filled below, empties after the first steps.
        self._virgin = set()
        self.group_of: Dict[nn.Parameter, int] = {}
        for gi, grp in enumerate(optimizer.param_groups):
            for p in grp["params"]:
                self.group_of[p] = gi

        # true grad-as-bucket-view for GEMM-produced gradients (fused backends, one backward pass per step)
        from ..ops import direct_wgrad
        self._direct_wgrad = (self.backend_name in ("b200", "emu") and self.passes_per_step == 1 and direct_wgrad.enabled()
                              and not self.exclude_reducescatter)
        if self._direct_wgrad:
            direct_wgrad.install(model)
        self.plan = BucketPlan(model, self.world)
        for s in self.plan.slots:
            if s.param not in self.group_of:
                raise ValueError("parameter %s requires grad but is not in any optimizer param group" % s.name)
        if policy is not None:
            self._apply_policy(policy)
        elif threshold is not None:
            self.plan.group_by_threshold(threshold)
        else:
            self.plan.group_by_nearby_layers(num_nearby_layers)
        if self.verbose:
            print("# of parameters: ", self.plan.num_parameters)
        self._check_plan_consistency()
        if self.opt_kind == OPT_SGD and any(g.get("momentum", 0) != 0 and g.get("dampening", 0) != 0 for g in optimizer.param_groups):
            self._virgin = {s.param for s in self.plan.slots}
        self._build(initial=True)
        self._register_hooks()
        _LIVE_ENGINES.add(self)
        # model.load_state_dict() after wrapping writes into the bucket views: the fp32 master shards follow
        self._hooks.append(model.register_load_state_dict_post_hook(lambda module, incompatible: self.params_changed()))
        if os.environ.get("DEAR_TIMELINE"):
            from ..utils import trace
            trace.attach(self)

    # ------------------------------------------------------------------ plan / buffers
    def _apply_policy(self, policy):
        kind = policy[0]
        if kind == "threshold":
            self.plan.group_by_threshold(policy[1])
        elif kind == "nearby":
            self.plan.group_by_nearby_layers(policy[1])
        elif kind == "flags":
            self.plan.group_by_flags(policy[1])
        elif kind == "per_module":
            self.plan.group_per_module()
        elif kind == "explicit":
            self.plan.group_explicit(policy[1])
        else:
            raise ValueError("unknown bucketing policy %r" % (policy,))

    def _check_plan_consistency(self):
        if self.world == 1 or os.environ.get("DEAR_SKIP_PLAN_CHECK"):
            return
        import hashlib
        h = hashlib.sha1(repr(self.plan.signature()).encode()).hexdigest()
        h0 = runtime.broadcast_object(h, src=0)
        if h != h0:
            raise RuntimeError("rank %d built a different bucket plan than rank 0 (models differ?)" % self.rank)
        # ranks that disagree would pack gradients of different formats into each other's buckets: every rank learns
        # every setting, so all of them raise
        wires = [None] * self.world
        torch.distributed.all_gather_object(wires, str(self._grad_comm_dtype), group=runtime.group())
        if len(set(wires)) != 1:
            raise RuntimeError("the ranks disagree on grad_comm_dtype: %s (rank order)" % ", ".join(wires))

    @property
    def grad_comm_dtype(self) -> Optional[torch.dtype]:
        """16-bit dtype in which fp32 gradients are sent to the reduce-scatter (None: fp32, the default)."""
        return self._grad_comm_dtype

    def _make_backend(self):
        if self.backend_name in ("b200", "emu"):
            return NativeBackend(runtime.communicator(), self.plan, self.rank, self.world, self.device,
                                 self._grad_comm_dtype)
        return TorchBackend(runtime.group(), self.plan, self.rank, self.world, self.device, self._grad_comm_dtype)

    @torch.no_grad()
    def _build(self, initial: bool, carry: Optional[dict] = None):
        """Allocate buckets for the current plan and move parameters (and state) into them."""
        plan = self.plan
        self.backend = self._make_backend()
        be = self.backend
        be.set_grad_scale(1.0 / getattr(self, "loss_scale", 1.0))
        be.set_amp(self.amp)
        self.clip = None
        self._attach_clip()
        self.steal = be.steal_grads
        self._param_view: Dict[nn.Parameter, torch.Tensor] = {}
        self._grad_view: Dict[nn.Parameter, torch.Tensor] = {}
        self._direct_params: List[nn.Parameter] = []
        for b in plan.buckets:
            pbuf, gbuf = be.param_buffer(b.index), be.grad_buffer(b.index)
            for s in b.slots:
                p = s.param
                if not _dense_like(p.data):
                    p.data = p.data.contiguous()
                pv = torch.as_strided(pbuf, p.shape, p.stride(), s.start)
                gv = torch.as_strided(gbuf, p.shape, p.stride(), s.start)
                pv.copy_(p.data)
                p.data = pv
                self._param_view[p] = pv
                self._grad_view[p] = gv
                if self.steal:
                    p.grad = None
                else:
                    p.grad = gv
                # Linear weights: the wgrad GEMM writes its slice of the gradient bucket directly (ops/direct_wgrad.py).
                # Not into a 16-bit bucket of fp32 gradients (grad_comm_dtype): those go through the converting pack.
                if self._direct_wgrad and p.dim() == 2 and gv.is_contiguous() and gv.dtype == p.dtype:
                    p._dear_grad_view = gv
                    p._dear_grad_written = False
                    self._direct_params.append(p)
                elif hasattr(p, "_dear_grad_view"):
                    del p._dear_grad_view
        be.init_master_shards()
        if carry is not None:
            self._restore_state(carry)
        self.set_step(self.num_updates)
        nb = len(plan.buckets)
        self._n_params = [len(b.slots) for b in plan.buckets]
        self._arrived = [[False] * n for n in self._n_params]
        self._n_arrived = [0] * nb
        self._complete = [False] * nb
        self._rs_launched = [False] * nb
        self._next_rs = nb - 1
        self._pending = [False] * nb
        self._any_pending = False
        # stolen gradients still read by Kernel A, per communication stream (one BucketSet per dtype)
        self._inflight: Dict[int, List[torch.Tensor]] = {}
        self._src = [[0] * n for n in self._n_params]
        self._flags = [[0] * n for n in self._n_params]
        # pack tables count gradient-bucket bytes (2 per element when fp32 gradients travel at 16 bits)
        es = [be.grad_buffer(b.index).element_size() for b in plan.buckets]
        self._dst_off = [[s.start * es[b.index] for s in b.slots] for b in plan.buckets]
        self._nbytes = [[s.numel * es[b.index] for s in b.slots] for b in plan.buckets]
        self._hyper_key = [None] * nb
        self._absent = [()] * nb           # per bucket: slots that received no gradient in the current step
        self._module_bucket = list(plan.module_bucket)
        if getattr(self, "timeline", None) is not None:
            from ..utils import trace
            trace.attach_backend(self)
        if self.verbose:
            print(plan.describe())

    # ------------------------------------------------------------------ hooks
    def _register_hooks(self):
        if not self.exclude_allgather:
            for mi, module in enumerate(self.plan.modules):
                self._hooks.append(module.register_forward_pre_hook(self._make_pre_hook(mi)))
        if not self.exclude_reducescatter:
            for s in self.plan.slots:
                self._hooks.append(s.param.register_post_accumulate_grad_hook(self._on_grad))

    def _make_pre_hook(self, mi):
        def hook(module, inputs):
            if self._any_pending:
                self._wait_bucket(self._module_bucket[mi])
            if self._safe_point_actions and mi == len(self._module_bucket) - 1 and torch.is_grad_enabled():
                self._run_safe_point()
        return hook

    def _wait_bucket(self, g):
        if self._pending[g]:
            self.backend.wait_bucket(g)
            self._pending[g] = False
            # inside ONE BucketSet every all-gather is queued behind every reduce-scatter of the same step, so
            # once the compute stream has waited on one of its all-gathers that set's gradients may be released;
            # another dtype's set has its own stream and keeps its gradients until one of ITS buckets was waited on
            self._inflight.pop(self.backend.stream_key(g), None)
            if not any(self._pending):
                self._any_pending = False

    def _on_grad(self, p):
        s = self.plan.slot_of[p]
        g, i = s.bucket, s.index_in_bucket
        if self.passes_per_step > 1:
            # gradient accumulation: autograd keeps summing into p.grad; only the last pass hands it over
            seen = self._passes_seen.get(p, 0) + 1
            self._passes_seen[p] = seen
            if seen < self.passes_per_step:
                return
        if self._rs_launched[g] or self._arrived[g][i]:
            raise RuntimeError(
                "gradient for %s arrived %s before step(): pass backward_passes_per_step=k to DistributedOptimizer to "
                "accumulate gradients over k backward passes (the reference has no accumulation: one backward per "
                "step)" % (s.name, "twice" if self.passes_per_step == 1 else "more than %d times" % self.passes_per_step))
        grad = p.grad
        if self.steal:
            self._hand_over(g, i, p, grad)
        else:
            gv = self._grad_view[p]
            if grad.data_ptr() != gv.data_ptr():
                gv.copy_(grad)
                p.grad = gv
        self._arrived[g][i] = True
        if self._wt is not None:
            self._wt.param_in(s)
        self._n_arrived[g] += 1
        if self._n_arrived[g] == self._n_params[g]:
            self._complete[g] = True
            self._drain_rs()

    def _hand_over(self, g, i, p, grad):
        """Steal mode: point the pack table of bucket g at this gradient (or stage it in the bucket view)."""
        if grad.data_ptr() == self._grad_view[p].data_ptr():
            # already in the bucket: the layer's wgrad GEMM wrote it there (ops/direct_wgrad.py)
            self._src[g][i] = 0
            self._flags[g][i] = 0
            return
        if (grad.dtype == p.dtype and grad.stride() == p.stride() and grad.data_ptr() % 16 == 0
                and not grad.is_sparse):
            self._src[g][i] = grad.data_ptr()
        else:
            self._grad_view[p].copy_(grad)
            self._src[g][i] = 0
        self._flags[g][i] = 0
        self._inflight.setdefault(self.backend.stream_key(g), []).append(grad)

    def _drain_rs(self, force=False):
        """Launch reduce-scatters in descending bucket order (identical on every rank)."""
        while self._next_rs >= 0 and (force or self._complete[self._next_rs]):
            g = self._next_rs
            absent = []
            if not self._complete[g]:
                for i, ok in enumerate(self._arrived[g]):
                    if ok:
                        continue
                    # (bucket-view mode keeps p.grad alive between steps: whether autograd produced anything in THIS
                    # step is what the hook counted)
                    q = self.plan.buckets[g].slots[i].param
                    late = q.grad if (self.passes_per_step > 1 and self._passes_seen.get(q, 0) > 0) else None
                    if late is not None:
                        # accumulated over fewer passes than passes_per_step (unused in some): still a gradient
                        p = self.plan.buckets[g].slots[i].param
                        if self.steal:
                            self._hand_over(g, i, p, late)
                        elif late.data_ptr() != self._grad_view[p].data_ptr():
                            self._grad_view[p].copy_(late)
                            p.grad = self._grad_view[p]
                    else:                # no gradient this iteration: contribute zeros, skip the update
                        self._src[g][i] = 0
                        self._flags[g][i] = 1 if self.steal else 0
                        absent.append(i)
            self._absent[g] = tuple(absent)
            if self.steal:
                self.backend.set_pack(g, self._src[g], self._dst_off[g], self._nbytes[g], self._flags[g])
            self.backend.reduce_scatter(g, True)
            self._rs_launched[g] = True
            if self._wt is not None:
                self._wt.bucket_out(g)
            self._next_rs -= 1

    # ------------------------------------------------------------------ hyper-parameters
    @staticmethod
    def _adam_lag_adjust(k, t: int, lag: int):
        """Hyper-parameters that make the kernel's update with the GLOBAL step count ``t`` equal to Adam's update with
        the parameter's own count ``s = t - lag`` (torch.optim counts steps per parameter and skips a parameter without
        gradient):   lr/bc1(s) * m / (sqrt(v)/sqrt(bc2(s)) + eps)  ==  lr'/bc1(t) * m / (sqrt(v)/sqrt(bc2(t)) + eps')
        with  r = sqrt(bc2(s)/bc2(t)),  eps' = eps r,  lr' = lr r bc1(t)/bc1(s);  AdamW's decoupled decay keeps
        lr' wd' = lr wd."""
        lr, wd, b1, damp, nest, opt, b2, eps = k
        s = t - lag
        r = math.sqrt((1.0 - b2 ** s) / (1.0 - b2 ** t)) if b2 < 1.0 else 1.0
        lr2 = lr * r * ((1.0 - b1 ** t) / (1.0 - b1 ** s) if 0.0 < b1 < 1.0 else 1.0)
        wd2 = wd * lr / lr2 if (opt == OPT_ADAMW and lr2 != 0.0) else wd
        return (lr2, wd2, b1, damp, nest, opt, b2, eps * r)

    def _refresh_hyper(self):
        key_all = self._hyper_key_now()
        t = self.num_updates + 1                     # the step count the kernels will use for the coming update
        for b in self.plan.buckets:
            absent = self._absent[b.index]
            lags = None
            if self.opt_kind != OPT_SGD and self._lag:
                # (a parameter that sits this step out as well needs no correction now: no table churn for a branch
                # that never runs)
                gone_now = set(absent)
                lags = tuple(0 if i in gone_now else self._lag.get(sl.param, 0) for i, sl in enumerate(b.slots))
                lags = (t, lags) if any(lags) else None
            fresh = ()
            if self._virgin and self._mom_initialised and self.opt_kind == OPT_SGD:
                gone_now = set(absent)
                fresh = tuple(i for i, sl in enumerate(b.slots) if i not in gone_now and sl.param in self._virgin)
            key = (key_all, absent, lags, fresh)
            if self._hyper_key[b.index] == key:
                continue
            segs = []
            if not absent and lags is None and not fresh:
                for end, gi in self.plan.hyper_segments(b.index, self.group_of):
                    segs.append((int(end),) + key_all[gi])
            else:
                # parameters that received no gradient on this rank carry HYPER_SKIP: where the reduced gradient is
                # zero as well (absent on every rank) the update leaves them alone, like torch.optim skips
                # ``p.grad is None`` (no weight decay, no momentum / moment decay)
                gone, prev = set(absent), None
                for i, sl in enumerate(b.slots):
                    gi, skip = self.group_of[sl.param], i in gone
                    lag = lags[1][i] if (lags is not None and not skip) else 0
                    end = b.slots[i + 1].start if i + 1 < len(b.slots) else b.padded_numel
                    k = key_all[gi]
                    if lag and t - lag >= 1:
                        k = self._adam_lag_adjust(k, t, lag)
                    first_own = i in fresh
                    if first_own:
                        k = k[:3] + (0.0,) + k[4:]          # this parameter's first gradient: buf = g
                    seg = (int(end),) + k[:4] + (int(k[4]) | (HYPER_SKIP if skip else 0),) + k[5:]
                    if prev == (gi, skip, lag, first_own) and not lag:
                        segs[-1] = seg
                    else:
                        segs.append(seg)
                    prev = (gi, skip, lag, first_own)
            self.backend.set_hyper(b.index, HyperSpec(segs))
            self._hyper_key[b.index] = key

    def freeze_hyper(self):
        """A loop that DEFERS ``step()`` past the point where the user's code may change ``param_groups`` (the rotated
        ``TrainStep``: the update of call t runs at the start of call t+1, after ``scheduler.step()``) snapshots the
        hyper-parameters when the gradients are complete; the deferred update then uses the snapshot, like
        ``optimizer.step(); scheduler.step()`` would have."""
        self._frozen_hyper = self._hyper_key_live()

    # ------------------------------------------------------------------ global-norm clipping
    # Semantics of ``torch.nn.utils.clip_grad_norm_`` on the AVERAGED (and, with a scaler, unscaled) gradient (the
    # reference's WFBP optimizer clips per tensor after its all-reduce, wfbp/dopt.py:855-862; its DeAR factory accepts
    # ``norm_clip`` and ignores it).  On the fused backends Kernel A sums the squares of the reduced shard per bucket and
    # the step's first update kernel agrees on the norm with every rank at its entry rendezvous; every update kernel
    # multiplies the coefficient into the gradient.  No extra pass over memory, no host synchronisation, and it can be
    # captured in a CUDA graph.  ClipState words (csrc/dear_common.h): 0 max_norm, 1 total_norm, 2 coef, 3 slots.
    @property
    def norm_clip(self) -> Optional[float]:
        return self._norm_clip

    @norm_clip.setter
    def norm_clip(self, value: Optional[float]):
        """Takes effect at the next step; the value is written to the device on the current stream (outside any CUDA
        graph), after every queued update."""
        if value is not None:
            value = float(value)
            if not value > 0:
                raise ValueError("norm_clip must be positive")
        was_on = self._norm_clip is not None
        self._norm_clip = value
        if getattr(self, "backend", None) is None:
            return
        self.synchronize(host=False)
        if value is not None and was_on and self.clip is not None:
            self.clip[0].fill_(value)
        else:
            self.clip = None
            self._attach_clip()

    def _attach_clip(self):
        """(Re)allocate the device clipping state for the current buckets and hand it to the backend."""
        be = self.backend
        if self._norm_clip is None or self.exclude_reducescatter or self.exclude_allgather:
            be.set_clip(None)
            return
        st = torch.zeros(be.clip_state_numel(), dtype=torch.float32, device=self.device)
        st[0] = self._norm_clip
        st.view(torch.int32)[3] = len(self.plan.buckets)
        self.clip = st
        be.set_clip(st)

    @property
    def last_grad_norm(self) -> Optional[torch.Tensor]:
        """2-norm of the last step's averaged gradient before clipping: a fresh 0-dim fp32 tensor, ordered on the
        current stream after that step's deciding update.  None without clipping."""
        if self.clip is None:
            return None
        if self._pending and self._pending[0]:
            self._wait_bucket(0)                         # bucket 0's update decides the step
        return self.clip[1].clone()

    def unfreeze_hyper(self):
        self._frozen_hyper = None

    def _hyper_key_now(self):
        frozen = getattr(self, "_frozen_hyper", None)
        return frozen if frozen is not None else self._hyper_key_live()

    def _hyper_key_live(self):
        """Per param group: (lr, wd, momentum|beta1, dampening, nesterov, opt, beta2, eps)."""
        keys = []
        for g in self.opt.param_groups:
            if self.opt_kind == OPT_SGD:
                keys.append((float(g["lr"]), float(g.get("weight_decay", 0.0)), float(g.get("momentum", 0.0)),
                             float(g.get("dampening", 0.0)), bool(g.get("nesterov", False)), OPT_SGD, 0.0, 0.0))
            else:
                b1, b2 = g["betas"]
                keys.append((float(g["lr"]), float(g.get("weight_decay", 0.0)), float(b1), 0.0, False, self.opt_kind,
                             float(b2), float(g["eps"])))
        return tuple(keys)

    def hyper_changed(self) -> bool:
        key = self._hyper_key_now()
        return any(k is None or k[0] != key for k in self._hyper_key)

    def refresh_hyper_outside_graph(self):
        """An LR scheduler changed ``param_groups`` while the step is replayed from a CUDA graph:
        re-upload the device hyper-parameter tables and order the replay after the upload."""
        # a replayed graph advances the device step counter on its own; a per-parameter correction computed here for
        # one value of it would go stale, so under graphs Adam's bias correction follows the global count
        self._lag.clear()
        self._refresh_hyper()
        self.backend.wait_all()

    def set_loss_scale(self, scale: float):
        """Static loss scaling (the reference's ImageNet driver runs apex O2 with ``loss_scale=128.0``,
        dear/imagenet_benchmark.py:116-117,131): back-propagate ``loss * scale`` and the un-scaling is folded into the
        1/P of the reduce-scatter epilogue — no extra pass over the gradients.  Call it before ``backward()``."""
        if scale <= 0:
            raise ValueError("loss scale must be positive")
        if self.amp is not None:
            raise ValueError("this optimizer has a dynamic loss scaler (GradScaler); a static loss scale cannot be combined "
                             "with it")
        self.loss_scale = float(scale)
        if self.backend is not None:
            self.backend.set_grad_scale(1.0 / self.loss_scale)

    # ------------------------------------------------------------------ dynamic loss scaling (GradScaler)
    # AmpState words (csrc/dear_common.h): 0 overflow, 1 found_inf, 2 scale (f32), 3 growth tracker, 4 applied updates,
    # 5 growth factor (f32), 6 backoff factor (f32), 7 growth interval, 8 growth tracker before the last step's rule
    _AMP_F32 = {"scale": 2, "growth_factor": 5, "backoff_factor": 6}
    _AMP_I32 = {"growth_tracker": 3, "applied": 4, "growth_interval": 7, "prev_growth_tracker": 8}

    def set_step(self, t: int):
        """Number of updates applied so far, set from the host (build, re-bucketing, checkpoint resume): the kernels'
        step counters and, with a scaler, its count of applied updates (the source of the step count from then on)."""
        self.num_updates = int(t)
        self.backend.set_step(self.num_updates)
        if self.amp is not None:
            self.write_scaler(applied=self.num_updates)

    def attach_scaler(self, init_scale: float, growth_factor: float, backoff_factor: float, growth_interval: int):
        """Switch to dynamic loss scaling: the kernels divide the reduced gradient by a device-resident scale, skip
        the update of a step in which any rank saw a non-finite value, and adjust the scale like torch's GradScaler."""
        if getattr(self, "loss_scale", None) is not None:
            raise ValueError("this optimizer has a static loss_scale; a dynamic loss scaler (GradScaler) cannot be "
                             "combined with it")
        if self.amp is not None:
            raise ValueError("this optimizer already has a GradScaler")
        self.synchronize(host=False)
        self.amp = torch.zeros(9, dtype=torch.int32, device=self.device)
        self.write_scaler(scale=init_scale, growth_factor=growth_factor, backoff_factor=backoff_factor,
                          growth_interval=growth_interval, growth_tracker=0, prev_growth_tracker=0,
                          applied=self.num_updates)
        self.backend.set_amp(self.amp)

    def scaler_scale(self) -> torch.Tensor:
        """The device scale as a 0-dim fp32 tensor, usable by the current stream (ordered after the last update)."""
        self.synchronize(host=False)
        return self.amp.view(torch.float32)[2]

    def write_scaler(self, **fields):
        """Set AmpState fields from the host, in current-stream order after every queued update."""
        self.synchronize(host=False)
        f32 = self.amp.view(torch.float32)
        for k, v in fields.items():
            if k in self._AMP_F32:
                f32[self._AMP_F32[k]].fill_(float(v))
            else:
                self.amp[self._AMP_I32[k]].fill_(int(v))

    def read_scaler(self) -> dict:
        """Host copy of the AmpState fields (synchronises the host)."""
        self.synchronize(host=True)
        st = self.amp.cpu()
        f32 = st.view(torch.float32)
        out = {k: float(f32[i]) for k, i in self._AMP_F32.items()}
        out.update({k: int(st[i]) for k, i in self._AMP_I32.items()})
        return out

    def params_changed(self):
        """The parameter VALUES were overwritten from outside (``broadcast_parameters``, ``load_state_dict``,
        manual ``p.data.copy_``): re-derive the fp32 master shards of low-precision buckets from the bucket
        contents, otherwise the next update would push the stale masters back over the new values."""
        if self.backend is None:
            return
        self.synchronize(host=True)
        self.backend.init_master_shards()

    # ------------------------------------------------------------------ step
    def step(self):
        if self.backend is None:
            raise RuntimeError("this DistributedOptimizer was closed (engine.close()): its buckets are released")
        be = self.backend
        nb = len(self.plan.buckets)
        if not self.exclude_reducescatter:
            self._drain_rs(force=True)
        if not self.exclude_allgather:
            self._refresh_hyper()
            be.fence()
            first = not self._mom_initialised
            for g in range(nb):
                be.allgather_update(g, True, first, zero_grad=not self.steal)
                self._pending[g] = True
            self._any_pending = True
            self._mom_initialised = True
            self.num_updates += 1
            if self._virgin:
                for g in range(nb):
                    gone = set(self._absent[g])
                    for i, sl in enumerate(self.plan.buckets[g].slots):
                        if i not in gone:
                            self._virgin.discard(sl.param)
            if self.opt_kind != OPT_SGD:
                for g in range(nb):
                    if self._absent[g]:
                        slots = self.plan.buckets[g].slots
                        for i in self._absent[g]:
                            self._lag[slots[i].param] = self._lag.get(slots[i].param, 0) + 1
        else:
            # time-breakdown mode (no all-gather): peers may still be pulling from this rank's
            # gradient buckets, so rendezvous on the device before the next backward reuses them
            be.wait_all()
            comm = runtime.communicator()
            if comm is not None and self.world > 1:
                comm.waitStream(comm.deviceBarrier())
            self._inflight.clear()
        if self.steal:
            for s in self.plan.slots:
                s.param.grad = None
        self._passes_seen.clear()
        for p in self._direct_params:
            p._dear_grad_written = False
        # reset the per-iteration state machine
        for g in range(nb):
            if self._n_arrived[g]:
                self._arrived[g] = [False] * self._n_params[g]
                self._n_arrived[g] = 0
            self._complete[g] = False
            self._rs_launched[g] = False
        self._next_rs = nb - 1
        self.num_steps += 1
        for cb in self._step_callbacks:
            cb()

    def flush_reduce_scatter(self):
        """Issue the reduce-scatter of every bucket that has not been issued yet (absent gradients count as
        zeros).  ``step()`` does this itself; a loop that defers ``step()`` (utils/train.py, rotated mode)
        calls it right after backward."""
        if not self.exclude_reducescatter:
            self._drain_rs(force=True)

    def join_comm_stream(self):
        """The current stream waits for everything queued on the communication stream so far."""
        self.backend.wait_all()

    def flush(self):
        """User-facing barrier: apply deferred updates (rotated training loops register a callback), then
        wait until every update is visible to the host."""
        for cb in list(self.flush_callbacks):
            cb()
        self.synchronize(host=True)

    def synchronize(self, host: bool = True):
        """Make all outstanding updates visible to the current stream (and the host)."""
        if self.backend is None:           # closed: everything was synchronised and handed back in close()
            return
        if self._any_pending:
            self.backend.wait_all()
            self._pending = [False] * len(self._pending)
            self._any_pending = False
        self._inflight.clear()
        if host:
            self.backend.synchronize()
            if self.device.type == "cuda":
                torch.cuda.current_stream(self.device).synchronize()

    # ------------------------------------------------------------------ re-bucketing
    def request_rebucket(self, policy):
        """Re-lay-out the buckets at the next safe point (last module's forward pre-hook of a
        training forward; reference dear/dopt_rsag_bo.py:317-320)."""
        self._safe_point_actions.append(policy)

    def _run_safe_point(self):
        policy = self._safe_point_actions[-1]
        self._safe_point_actions.clear()
        self.rebucket(policy)

    @torch.no_grad()
    def _gather_state(self) -> dict:
        """Full (un-sharded) optimizer state per parameter name: momentum and fp32 master."""
        from ..utils.checkpoint import gather_sharded
        out = {"momentum": {}, "master": {}, "var": {}, "mom_init": self._mom_initialised, "num_updates": self.num_updates}
        if self.amp is not None:
            # skipped steps applied nothing: the device count of applied updates is the step count of the new buckets
            applied = self.read_scaler()["applied"]
            out.update(num_updates=applied, mom_init=applied > 0)
        for b in self.plan.buckets:
            g = b.index
            for kind, shard in (("momentum", self.backend.mom_shard[g]), ("master", self.backend.master_shard[g]),
                                ("var", self.backend.var_shard[g])):
                if shard is None:
                    continue
                full = gather_sharded(shard, self.world)
                for s in b.slots:
                    out[kind][s.name] = full[s.start:s.end].clone()
        return out

    @torch.no_grad()
    def _restore_state(self, carry: dict):
        be = self.backend
        self._mom_initialised = bool(carry.get("mom_init", False))

        self.num_updates = int(carry.get("num_updates", self.num_updates))
        for b in self.plan.buckets:
            g = b.index
            lo, hi = self.rank * b.shard_numel, (self.rank + 1) * b.shard_numel
            for kind in ("momentum", "master", "var"):
                vals = carry.get(kind, {})
                if not any(s.name in vals for s in b.slots):
                    continue
                if kind == "momentum":
                    be.ensure_momentum(g)
                    shard = be.mom_shard[g]
                elif kind == "var":
                    be.ensure_var(g)
                    shard = be.var_shard[g]
                else:
                    shard = be.master_shard[g]
                    if shard is None:
                        continue
                for s in b.slots:
                    if s.name not in vals:
                        continue
                    a, z = max(s.start, lo), min(s.end, hi)
                    if a < z:
                        shard[a - lo:z - lo].copy_(vals[s.name].reshape(-1)[a - s.start:z - s.start])

    def rebucket(self, policy):
        """Collective: switch to a new bucketing policy, migrating parameters and sharded state."""
        self.synchronize(host=True)
        carry = self._gather_state()
        old_backend = self.backend
        self._apply_policy(policy)
        self._build(initial=False, carry=carry)
        del old_backend
        runtime.barrier()

    def close(self):
        if self._closed:
            return
        self._closed = True
        for h in self._hooks:
            h.remove()
        self._hooks.clear()
        self.flush()                       # deferred updates of a rotated training loop, then wait for everything
        if getattr(self, "timeline", None) is not None:
            self.timeline.close()
        # Hand the parameters back: they are views of the (symmetric) parameter buckets, which must be released before
        # the communicator — and with it the rendezvous store — can go away (runtime.shutdown, re-initialisation).
        with torch.no_grad():
            for s in self.plan.slots:
                s.param.data = s.param.data.clone(memory_format=torch.preserve_format)
                s.param.grad = None
                if hasattr(s.param, "_dear_grad_view"):
                    del s.param._dear_grad_view
        self._inflight.clear()
        self._grad_view = {}
        self.backend = None


# =====================================================================================
# optimizer facade
# =====================================================================================
class _DistributedOptimizer(torch.optim.Optimizer):
    """Mixed into a dynamic subclass of the user's optimizer class (the Horovod idiom the
    reference uses, dear/dear_dopt.py:395-398)."""

    def __init__(self, params, model, threshold=THRESHOLD, num_nearby_layers=NUM_NEARBY_LAYERS,
                 exclude_parts="", policy=None, verbose=True, backward_passes_per_step=1, grad_comm_dtype=None):
        super(self.__class__, self).__init__(params)
        if not isinstance(self, (torch.optim.SGD, torch.optim.Adam, torch.optim.AdamW)):
            raise TypeError(
                "the decoupled all-reduce fuses the parameter update into the all-gather kernel; supported: "
                "torch.optim.SGD (the reference's only DeAR optimizer, dear/dear_dopt.py:310-336), Adam and AdamW; "
                "got %s. Use parallel.baselines for other optimizers." % type(self).__mro__[1].__name__)
        for g in self.param_groups:
            if g.get("amsgrad", False) or g.get("capturable", False) or g.get("differentiable", False):
                raise ValueError("amsgrad / capturable / differentiable Adam variants are not supported")
        for g in self.param_groups:
            if g.get("maximize", False):
                raise ValueError("maximize=True is not supported")
        self._dear = DearEngine(self, model, threshold=threshold, num_nearby_layers=num_nearby_layers,
                                exclude_parts=exclude_parts, policy=policy, verbose=verbose,
                                backward_passes_per_step=backward_passes_per_step, grad_comm_dtype=grad_comm_dtype)

    # -- torch.optim.Optimizer API ---------------------------------------------------
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        self._dear.step()
        return loss

    def zero_grad(self, set_to_none: bool = True):
        """No-op, like the reference (dear/dear_dopt.py:338-339): gradients are consumed by the
        reduce-scatter and released by ``step()``."""
        return None

    def synchronize(self):
        """Block until every outstanding parameter update has landed (host-visible)."""
        self._dear.flush()

    flush = synchronize

    def skip_synchronize(self):
        """Horovod-style context manager used by mixed-precision loops (examples/mnist/pytorch_mnist.py:80 of the
        reference: ``optimizer.synchronize(); scaler.unscale_(optimizer); with optimizer.skip_synchronize(): ...``).
        ``step()`` never blocks here, so there is nothing to skip; kept for source compatibility."""
        import contextlib
        return contextlib.nullcontext()

    def set_loss_scale(self, scale: float):
        self._dear.set_loss_scale(scale)

    @property
    def engine(self) -> DearEngine:
        return self._dear

    def state_dict(self):
        from ..utils.checkpoint import optimizer_state_dict
        return optimizer_state_dict(self)

    def load_state_dict(self, state_dict):
        from ..utils.checkpoint import load_optimizer_state_dict
        return load_optimizer_state_dict(self, state_dict)


def DistributedOptimizer(optimizer, model, compression=None, is_sparse=False, density=0.001, seq_layernames=None,
                         layerwise_times=None, norm_clip=None, threshold=None, writer=None, gradient_path=None,
                         fp16=False, mgwfbp=False, rdma=False, multi_job_scheduling=False, exclude_parts="",
                         num_nearby_layers=None, policy=None, verbose=True, bo_tuning=False, bo_kwargs=None,
                         backward_passes_per_step=1, loss_scale=None, grad_comm_dtype=None):
    """Wrap ``optimizer`` (``torch.optim.SGD`` / ``Adam`` / ``AdamW``) for DeAR data-parallel training of ``model``.

    Signature-compatible with the reference factory (dear/dear_dopt.py:381-398): the Horovod-era
    keyword arguments are accepted; those that have no meaning here are ignored.  Unlike the
    reference, ``threshold`` (MB; default 25) and ``num_nearby_layers`` are honoured instead of
    being module constants:  ``threshold=None, num_nearby_layers=k`` selects the nearby-layer
    policy (``k=1`` is "DeAR without tensor fusion").  ``bo_tuning=True`` enables the Bayesian
    buffer-size tuner (the reference's separate ``dopt_rsag_bo`` module).  ``backward_passes_per_step=k``
    (Horovod's name; not in the reference) accumulates gradients locally over k backward passes and
    reduce-scatters them during the k-th; call ``step()`` once per k passes.  ``norm_clip=c`` (accepted and ignored by the
    reference's DeAR factory) clips the global norm of the averaged gradient to ``c`` like
    ``torch.nn.utils.clip_grad_norm_`` before the update, inside the fused kernels (``DearEngine.norm_clip``; the norm
    before clipping is ``engine.last_grad_norm``).  ``grad_comm_dtype=torch.bfloat16`` or ``torch.float16`` sends the
    gradients of fp32 parameters to the reduce-scatter rounded to that dtype (``.to(dtype)`` on every rank, summed in
    fp32): half the bytes over the link, like DDP's ``bf16_compress_hook`` / ``fp16_compress_hook``.  bf16 keeps fp32's
    range; fp16 is meant to be paired with loss scaling (an overflow in the cast is an inf that ``GradScaler`` skips).
    16-bit parameters and a single rank are unaffected.  ``compression=`` and ``fp16=`` are still ignored.
    """
    if threshold in (None, 0) and num_nearby_layers is None:
        threshold = float(os.environ.get("DEAR_THRESHOLD_MB", THRESHOLD))
    elif threshold in (None, 0):
        threshold = None
    cls = type(optimizer.__class__.__name__, (optimizer.__class__,), dict(_DistributedOptimizer.__dict__))
    opt = cls(optimizer.param_groups, model, threshold=threshold,
              num_nearby_layers=num_nearby_layers if num_nearby_layers is not None else NUM_NEARBY_LAYERS,
              exclude_parts=exclude_parts, policy=policy, verbose=verbose,
              backward_passes_per_step=backward_passes_per_step, grad_comm_dtype=grad_comm_dtype)
    if norm_clip is not None:
        opt._dear.norm_clip = norm_clip             # global-norm clipping of the averaged gradients
    if loss_scale is not None:
        opt.set_loss_scale(loss_scale)
    if bo_tuning:
        # dopt_rsag_bo: Bayesian optimisation of the fusion threshold (dear/dopt_rsag_bo.py:100-101)
        from .tuner import attach_tuner
        attach_tuner(opt, verbose=verbose, **(bo_kwargs or {}))
    return opt
