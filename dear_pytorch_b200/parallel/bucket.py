"""Tensor-fusion bucket planner.

Reproduces the reference's module discovery and grouping rules and adds the
memory layout the fused kernels need.

Reference rules (SURVEY.md §8.2-8.3):
  * discovery      dear/dear_dopt.py:207-222  ``model.modules()`` pre-order; a module is
                   registered iff it owns >=1 direct trainable parameter not already claimed
                   by an earlier module (tied weights belong to their first owner).
  * threshold      dear/dear_dopt.py:109-139  module size in MB = numel*4/2**20 (always 4
                   bytes); append while ``tot == 0 or tot + size < threshold``.
  * nearby layers  dear/dear_dopt.py:94-107   close a group every k modules; k<0 => one group.
  * flags          dear/dopt_rsag_wt.py:216-241 a boundary flag per module.
  * per tensor     dear/dopt_rsag_naive.py     one bucket per module ("w/o tensor fusion").

Layout differences (deliberate, GPU-first):
  * every parameter starts on a 256-byte boundary inside its bucket so that the views handed
    to cuDNN/cuBLAS (and TMA-based kernels) are aligned and so that hyper-parameter segments
    never straddle a 128-bit vector;
  * the bucket is padded so that each rank's shard is a multiple of 128 bytes (the reference
    pads to a multiple of P elements, dear/dear_dopt.py:186-194);
  * a bucket never mixes dtypes (a dtype change closes the bucket).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Sequence

import torch
import torch.nn as nn

PARAM_ALIGN_BYTES = 256
SHARD_ALIGN_BYTES = 128


@dataclass
class ParamSlot:
    name: str
    param: nn.Parameter
    module_index: int
    bucket: int = -1
    index_in_bucket: int = -1
    start: int = 0          # element offset inside the bucket
    numel: int = 0

    @property
    def end(self) -> int:
        return self.start + self.numel


@dataclass
class Bucket:
    index: int
    dtype: torch.dtype
    module_indices: List[int] = field(default_factory=list)
    slots: List[ParamSlot] = field(default_factory=list)
    numel: int = 0           # sum of parameter numels (no padding)
    padded_numel: int = 0    # what is allocated: multiple of world * shard alignment
    shard_numel: int = 0

    @property
    def size_mb(self) -> float:
        return self.padded_numel * 4 / 1024 / 1024


class BucketPlan:
    """Assignment of a model's trainable parameters to fusion buckets."""

    def __init__(self, model: nn.Module, world: int):
        self.world = int(world)
        self.modules: List[nn.Module] = []
        self.module_names: List[str] = []
        self.module_params: List[List[ParamSlot]] = []
        self.slots: List[ParamSlot] = []
        self.slot_of: Dict[nn.Parameter, ParamSlot] = {}
        self.module_index: Dict[nn.Module, int] = {}
        self.buckets: List[Bucket] = []
        self.module_bucket: List[int] = []
        self.policy = None
        self._discover(model)

    # ------------------------------------------------------------------ discovery
    def _discover(self, model: nn.Module) -> None:
        names = {p: n for n, p in model.named_parameters()}
        claimed = set()
        for module in model.modules():
            direct = []
            for p in module.parameters(recurse=False):
                if not p.requires_grad or p in claimed:
                    continue
                claimed.add(p)
                direct.append(p)
            if not direct:
                continue
            mi = len(self.modules)
            self.modules.append(module)
            self.module_names.append("module_name_%s_%d" % (module.__class__.__name__, mi))
            self.module_index[module] = mi
            slots = []
            for p in direct:
                s = ParamSlot(name=names.get(p, "param.noname.%d" % len(self.slots)), param=p,
                              module_index=mi, numel=p.numel())
                slots.append(s)
                self.slots.append(s)
                self.slot_of[p] = s
            self.module_params.append(slots)

    @property
    def num_parameters(self) -> int:
        return sum(s.numel for s in self.slots)

    def module_size_mb(self, mi: int) -> float:
        # the reference always charges 4 bytes per element (dear/dear_dopt.py:121)
        return sum(s.numel for s in self.module_params[mi]) * 4 / 1024 / 1024

    # ------------------------------------------------------------------ grouping policies
    def _split_on_dtype(self, groups: Sequence[Sequence[int]]) -> List[List[int]]:
        """A bucket never mixes dtypes: every group is partitioned into one sub-bucket per dtype
        (module order preserved inside each).  With bf16 convolutions and fp32 BatchNorm this gives
        one large bf16 bucket and one small fp32 bucket per group instead of a bucket per layer."""
        out: List[List[int]] = []
        for g in groups:
            by_dt: Dict[torch.dtype, List[int]] = {}
            for mi in g:
                dts = {s.param.dtype for s in self.module_params[mi]}
                if len(dts) != 1:
                    raise ValueError("module %s mixes parameter dtypes %s" % (self.module_names[mi], dts))
                by_dt.setdefault(next(iter(dts)), []).append(mi)
            out.extend(by_dt.values())
        return out

    def group_by_threshold(self, threshold_mb: float) -> "BucketPlan":
        groups: List[List[int]] = []
        cur: List[int] = []
        tot = 0.0
        for mi in range(len(self.modules)):
            sz = self.module_size_mb(mi)
            if tot == 0 or tot + sz < threshold_mb:
                cur.append(mi)
                tot += sz
            else:
                groups.append(cur)
                cur = [mi]
                tot = sz
        if cur:
            groups.append(cur)
        self.policy = ("threshold", float(threshold_mb))
        return self._layout(groups)

    def group_by_nearby_layers(self, k: int) -> "BucketPlan":
        groups: List[List[int]] = []
        cur: List[int] = []
        for i in range(len(self.modules)):
            cur.append(i)
            if not k < 0 and (i + 1) % k == 0:
                groups.append(cur)
                cur = []
        if cur:
            groups.append(cur)
        self.policy = ("nearby", int(k))
        return self._layout(groups)

    def group_by_flags(self, flags: Sequence[int]) -> "BucketPlan":
        """``flags[i] == 1`` closes a bucket after module i (wait-time variant)."""
        if len(flags) != len(self.modules):
            raise ValueError("need one flag per registered module")
        groups: List[List[int]] = []
        cur: List[int] = []
        for i, f in enumerate(flags):
            cur.append(i)
            if f:
                groups.append(cur)
                cur = []
        if cur:
            groups.append(cur)
        self.policy = ("flags", tuple(int(f) for f in flags))
        return self._layout(groups)

    def group_per_module(self) -> "BucketPlan":
        self.policy = ("per_module",)
        return self._layout([[i] for i in range(len(self.modules))])

    def group_explicit(self, groups: Sequence[Sequence[int]]) -> "BucketPlan":
        flat = sorted(mi for g in groups for mi in g)
        if flat != list(range(len(self.modules))):
            raise ValueError("groups must cover every registered module exactly once")
        self.policy = ("explicit", tuple(tuple(g) for g in groups))
        return self._layout(groups)

    # ------------------------------------------------------------------ layout
    def _layout(self, groups: Sequence[Sequence[int]]) -> "BucketPlan":
        groups = self._split_on_dtype(groups)
        self.buckets = []
        self.module_bucket = [-1] * len(self.modules)
        for bi, g in enumerate(groups):
            first = self.module_params[g[0]][0].param
            es = first.element_size()
            b = Bucket(index=bi, dtype=first.dtype, module_indices=list(g))
            palign = max(1, PARAM_ALIGN_BYTES // es)
            off = 0
            for mi in g:
                self.module_bucket[mi] = bi
                for s in self.module_params[mi]:
                    off = (off + palign - 1) // palign * palign
                    s.bucket = bi
                    s.index_in_bucket = len(b.slots)
                    s.start = off
                    off += s.numel
                    b.slots.append(s)
                    b.numel += s.numel
            quantum = self.world * max(1, SHARD_ALIGN_BYTES // es)
            b.padded_numel = max(quantum, (off + quantum - 1) // quantum * quantum)
            b.shard_numel = b.padded_numel // self.world
            self.buckets.append(b)
        return self

    # ------------------------------------------------------------------ helpers
    def describe(self) -> str:
        return "#Tensor fusion groups: %d\nBuffer sizes (MB): %s" % (
            len(self.buckets), ", ".join("%.2f" % b.size_mb for b in self.buckets))

    def signature(self):
        """Rank-independent fingerprint, used to assert all ranks built the same plan."""
        return tuple((b.dtype, b.padded_numel, tuple((s.name, s.start, s.numel) for s in b.slots))
                     for b in self.buckets)

    def hyper_segments(self, bucket: int, group_of: Dict[nn.Parameter, int]):
        """Contiguous element ranges of a bucket that share an optimizer param group.

        Returns ``[(end_element, group_index), ...]``; the gap after a parameter belongs to
        that parameter's segment, and the last segment extends to ``padded_numel``.
        """
        b = self.buckets[bucket]
        segs = []
        for i, s in enumerate(b.slots):
            gi = group_of[s.param]
            end = b.slots[i + 1].start if i + 1 < len(b.slots) else b.padded_numel
            if segs and segs[-1][1] == gi:
                segs[-1] = (end, gi)
            else:
                segs.append((end, gi))
        return segs
