"""``TrainStep`` — one training iteration (zero_grad → forward → loss → backward → step) as a
callable, optionally captured into a single CUDA graph.

Why a graph: the reference's iteration issues ≈1.1 k tiny kernels and several host-blocking
stream synchronisations for ResNet-50 (SURVEY.md §3.3).  With the fused kernels the optimizer
needs ~2 launches per bucket and no host synchronisation, and because the cross-GPU epochs live in
device memory (csrc/kernels.cu) the whole iteration — cuDNN/cuBLAS kernels, Kernel A per bucket on
the communication stream, Kernel B per bucket — replays as ONE graph launch.

``overlap_update=True`` rotates the loop body to ``step(previous gradients) → forward → backward``.
Graph launches serialise, so with the natural body the update + all-gather of iteration *t* (issued
by ``step()`` at the END of the graph) cannot overlap the forward of iteration *t+1* the way it does
in eager mode — the decoupling the whole method is about would be lost inside a graph.  Rotated, the
all-gathers are the FIRST nodes of the graph and the forward's per-bucket waits let them overlap
layer by layer.  Every call still performs one forward/backward and (from the second call on) one
parameter update; ``finish()`` — also run by ``optimizer.synchronize()`` / ``state_dict()`` — applies
the last pending update, so nothing is dropped at the end of training.  The update for batch *t* runs at the
start of call *t+1*, i.e. after the user's ``scheduler.step()``; it nevertheless uses the hyper-parameters that were
in force at the end of call *t* (``DearEngine.freeze_hyper``; a snapshot of ``param_groups`` for other optimizers), so
``step(x, y); scheduler.step()`` trains exactly like the natural loop (tests/test_train_step.py).

With ``bo_tuning=True`` the wrapper stays eager while the tuner explores (its timing and re-bucketing live
in Python hooks) and captures the graph once the final bucket layout is in place.
"""
from __future__ import annotations

import os
from typing import Callable, Optional

import torch


def _tree_map(fn, obj):
    if torch.is_tensor(obj):
        return fn(obj)
    if isinstance(obj, (tuple, list)):
        return type(obj)(_tree_map(fn, o) for o in obj)
    return obj


def _tree_zip_apply(fn, a, b):
    if torch.is_tensor(a):
        fn(a, b)
    elif isinstance(a, (tuple, list)):
        for x, y in zip(a, b):
            _tree_zip_apply(fn, x, y)


def _first_tensor(obj):
    if torch.is_tensor(obj):
        return obj
    if isinstance(obj, (tuple, list)):
        for o in obj:
            t = _first_tensor(o)
            if t is not None:
                return t
    return None


class TrainStep:
    def __init__(self, model: torch.nn.Module, optimizer, loss_fn: Callable, autocast_dtype: Optional[torch.dtype] = None,
                 use_graph: bool = False, graph_warmup: int = 3, overlap_update: bool = False, scaler=None):
        self.model = model
        self.scaler = scaler               # dear.GradScaler: back-propagate scaler.scale(loss) (dynamic loss scaling)
        self.opt = optimizer
        self.loss_fn = loss_fn
        self.autocast_dtype = autocast_dtype
        self.use_graph = use_graph
        self.graph_warmup = graph_warmup
        self._calls = 0
        self._graph = None
        self._static_in = None
        self._static_loss = None
        self._engine = getattr(optimizer, "_dear", None)
        self._debug = bool(os.environ.get("DEAR_GRAPH_DEBUG"))
        self._side = None
        self.eager_calls = 0               # how many times the Python step body ran (incl. the capture)
        self.overlap_update = overlap_update
        self._pending_update = False       # rotated mode: gradients reduced, update not yet applied
        self._clip_at_capture = None       # the engine's clipping state when the graph was captured
        if overlap_update and self._engine is not None:
            self._engine.flush_callbacks.append(self.finish)

    def _forward_backward(self, *batch):
        *inputs, target = batch
        self.opt.zero_grad()
        if self.autocast_dtype is not None:
            with torch.autocast("cuda" if inputs[0].is_cuda else "cpu", dtype=self.autocast_dtype):
                out = self.model(*inputs)
        else:
            out = self.model(*inputs)
        loss = self.loss_fn(out, target)
        (self.scaler.scale(loss) if self.scaler is not None else loss).backward()
        return loss.detach()

    def _eager(self, *batch):
        self.eager_calls += 1
        if not self.overlap_update:
            loss = self._forward_backward(*batch)
            self.opt.step()
            return loss
        if self._pending_update:
            self._deferred_step()                         # update from the previous call's gradients
        loss = self._forward_backward(*batch)
        if self._engine is not None:
            self._engine.flush_reduce_scatter()           # incomplete buckets (unused parameters) too
            self._engine.freeze_hyper()                   # the deferred update belongs to THIS call's learning rate
        else:
            self._frozen_groups = [{k: v for k, v in g.items() if k != "params"} for g in self.opt.param_groups]
        self._pending_update = True
        # the update of this call is deferred, not skipped, and will use this call's hyper-parameters: an LR scheduler
        # stepped now must not warn that it runs "before optimizer.step()" (torch checks this flag)
        self.opt._opt_called = True
        return loss

    def _deferred_step(self):
        """``optimizer.step()`` for the gradients of the previous call, with the hyper-parameters that were in force when
        that call ended (an LR scheduler stepped by the user in between must not leak into it)."""
        frozen = getattr(self, "_frozen_groups", None)
        if self._engine is not None or frozen is None:
            self.opt.step()                               # (the DeAR engine holds its own snapshot: freeze_hyper)
            return
        live = [{k: g[k] for k in f} for g, f in zip(self.opt.param_groups, frozen)]
        try:
            for g, f in zip(self.opt.param_groups, frozen):
                g.update(f)
            self.opt.step()
        finally:
            for g, v in zip(self.opt.param_groups, live):
                g.update(v)

    def _tuning_active(self) -> bool:
        tuner = getattr(self.opt, "tuner", None)
        if tuner is None or self._graph is not None:
            return False
        return (not tuner.finished) or bool(getattr(self._engine, "_safe_point_actions", None))

    def finish(self):
        """Rotated mode: apply the update of the last call's gradients (no-op otherwise)."""
        if self._pending_update:
            self._pending_update = False
            self._deferred_step()
            if self._engine is not None:
                self._engine.unfreeze_hyper()
            self._frozen_groups = None

    def _log(self, msg):
        if self._debug:
            print("[TrainStep] " + msg, flush=True)

    def _eager_on_side_stream(self, batch):
        """Warm-up iterations of the graph mode run on a side stream (the PyTorch whole-network
        capture recipe): allocator pools, cuDNN autotuning and autograd streams settle on the stream
        family the capture will use.  They are ordinary training steps on the caller's batches."""
        dev = _first_tensor(batch).device
        if self._side is None:
            self._side = torch.cuda.Stream(device=dev)
        cur = torch.cuda.current_stream(dev)
        self._side.wait_stream(cur)
        with torch.cuda.stream(self._side):
            loss = self._eager(*batch)
            if self._engine is not None:
                self._engine.synchronize(host=False)
                self._engine.join_comm_stream()
        cur.wait_stream(self._side)
        _tree_map(lambda t: t.record_stream(self._side), batch)
        return loss

    def _capture(self, batch):
        eng = self._engine
        dev = _first_tensor(batch).device
        self._static_in = _tree_map(lambda t: torch.empty_like(t).copy_(t), batch)
        if eng is not None:
            # hyper-parameter tables are uploaded OUTSIDE the graph (before the capture and after every change), so
            # an LR scheduler keeps working on a replayed graph; the native runtime refuses to capture such an upload
            eng.refresh_hyper_outside_graph()
            eng.synchronize(host=True)
            self._clip_at_capture = eng.clip        # the captured kernels hold this clipping state's address
        torch.cuda.synchronize(dev)
        self._log("capturing")
        self._graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self._graph, capture_error_mode="thread_local"):
            loss = self._eager(*self._static_in)
            if eng is not None:
                eng.synchronize(host=False)     # join the communication stream back into the capture
                eng.join_comm_stream()          # (rotated body: the reduce-scatters are its last nodes)
            self._static_loss = loss
        self._log("capture done; first replay")
        # the capture only records: replaying it IS this call's training step
        self._graph.replay()
        return self._static_loss

    def __call__(self, *batch):
        self._calls += 1
        if not self.use_graph:
            return self._eager(*batch)
        if self._tuning_active():
            # the Bayesian buffer-size tuner times iterations and re-buckets from Python hooks, which a replayed
            # graph never runs: stay eager until it has settled, then warm up and capture the final layout
            self._calls = 0
            return self._eager_on_side_stream(batch)
        if self.overlap_update and not self._pending_update:
            # nothing to apply yet (first call, or right after finish()): the captured body starts with an
            # update, so prime it with a plain forward/backward
            return self._eager_on_side_stream(batch)
        if self._graph is None:
            if self._calls <= self.graph_warmup:
                return self._eager_on_side_stream(batch)
            return self._capture(batch)
        eng = self._engine
        if eng is not None and eng.clip is not self._clip_at_capture:
            raise RuntimeError("norm_clip was switched on or off after the training step was captured in a CUDA graph; "
                               "its value may change between calls, but set it (or None) before the first call")
        if eng is not None and eng.hyper_changed():
            eng.refresh_hyper_outside_graph()
        _tree_zip_apply(lambda s, t: s.copy_(t, non_blocking=True) if s.data_ptr() != t.data_ptr() else None,
                        self._static_in, batch)
        self._graph.replay()
        if eng is not None:
            eng.num_steps += 1          # the replay ran the step; Python-side callbacks (tuner) do not run
            eng.num_updates += 1        # mirrors the device-resident Adam step counter (checkpointing)
            if self.overlap_update:
                eng.freeze_hyper()      # the update that opens the NEXT replay uses the values in force now
        return self._static_loss
