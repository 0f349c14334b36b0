"""Checkpoint / resume for the sharded optimizer state.

The reference has no checkpointing at all (SURVEY.md §5.4); with momentum and fp32 master
weights sharded 1/P per rank (Kernel B) a checkpoint has to gather the shards, and a resume has
to scatter them — possibly into a *different* bucket layout or world size.  State is therefore
exchanged per parameter *name*, never per bucket.

``optimizer.state_dict()`` (collective) returns a dict in the layout of the wrapped ``torch.optim`` class, with the
full state under the names and step counts of its family (parallel/families.py), so a checkpoint written by DeAR loads
into stock PyTorch and vice versa.  State stored under another family's names is not read.
"""
from __future__ import annotations

import os
from typing import Dict

import torch
import torch.distributed as dist

from .. import runtime
from ..parallel.backends import SHARD_KINDS


@torch.no_grad()
def gather_sharded(shard: torch.Tensor, world: int) -> torch.Tensor:
    """All-gather a per-rank 1-D shard into the full flat tensor (collective)."""
    if world == 1:
        return shard.clone()
    out = torch.empty(world * shard.numel(), dtype=shard.dtype, device=shard.device)
    comm = runtime.communicator()
    if comm is not None:
        h = comm.allGather(shard.contiguous(), out)
        comm.syncStream(h)
    else:
        dist.all_gather_into_tensor(out, shard.contiguous(), group=runtime.group())
    return out


def _param_index(optimizer) -> Dict[torch.nn.Parameter, int]:
    idx = {}
    for g in optimizer.param_groups:
        for p in g["params"]:
            idx[p] = len(idx)
    return idx


@torch.no_grad()
def optimizer_state_dict(optimizer) -> dict:
    """Collective.  State dict in the layout of the wrapped torch.optim class, with full (un-sharded) state."""
    eng = optimizer._dear
    fam = eng.family
    eng.flush()
    carry = eng._gather_state()
    index = _param_index(optimizer)
    state = {}
    for s in eng.plan.slots:
        ent = {}
        names = fam.state_names(optimizer.param_groups[eng.group_of[s.param]])
        # torch.optim counts steps per parameter: updates this one sat out (no gradient) are not counted
        steps = carry["num_updates"] - eng._lag.get(s.param, 0)
        if s.name in carry[names[0][1]] and fam.has_entry(steps, carry["mom_init"] and s.param not in eng._virgin):
            if fam.counts_steps:
                ent["step"] = torch.tensor(float(steps))
            for name, kind in names:
                ent[name] = carry[kind][s.name].reshape(s.param.shape).clone()
        if s.name in carry["master"]:
            ent["master_param"] = carry["master"][s.name].reshape(s.param.shape).clone()
        if ent:
            state[index[s.param]] = ent
    groups = []
    for g in optimizer.param_groups:
        d = {k: v for k, v in g.items() if k != "params"}
        d["params"] = [index[p] for p in g["params"]]
        groups.append(d)
    return {"state": state, "param_groups": groups,
            "dear": {"num_steps": eng.num_steps, "num_updates": carry["num_updates"], "policy": eng.plan.policy,
                     "world": eng.world}}


@torch.no_grad()
def load_optimizer_state_dict(optimizer, sd: dict) -> None:
    """Collective.  Accepts a dict from ``optimizer_state_dict`` or from the stock ``torch.optim`` class."""
    eng = optimizer._dear
    fam = eng.family
    eng.flush()
    for g, saved in zip(optimizer.param_groups, sd["param_groups"]):
        for k, v in saved.items():
            if k != "params":
                g[k] = v
    index = _param_index(optimizer)
    meta = sd.get("dear") or {}
    carry = dict({kind: {} for kind in SHARD_KINDS}, mom_init=False,
                 num_updates=int(meta.get("num_updates", eng.num_updates)))
    steps = {}                             # per-parameter step counts of the families that keep them
    eng._virgin = {s.param for s in eng.plan.slots} if fam.tracks_first_gradient(optimizer.param_groups) else set()
    for s in eng.plan.slots:
        ent = sd["state"].get(index[s.param], sd["state"].get(str(index[s.param])))
        if not ent:
            continue
        names = fam.state_names(optimizer.param_groups[eng.group_of[s.param]])
        found = [(name, kind) for name, kind in names if ent.get(name) is not None]
        for name, kind in found:
            carry[kind][s.name] = ent[name].to(eng.device, torch.float32).reshape(-1)
        if found:
            carry["mom_init"] = True       # the next update is not this parameter's first
            eng._virgin.discard(s.param)
            if fam.counts_steps and ent.get("step") is not None:
                steps[s.param] = int(float(ent["step"]))
        mp = ent.get("master_param")
        if mp is not None:
            carry["master"][s.name] = mp.to(eng.device, torch.float32).reshape(-1)
    fam.restore_count(eng, carry, steps)
    eng._restore_state(carry)
    eng.set_step(eng.num_updates)
    eng._hyper_key = [None] * len(eng._hyper_key)
    eng.num_steps = int(meta.get("num_steps", eng.num_steps))


def save_checkpoint(path: str, model: torch.nn.Module, optimizer, extra: dict = None) -> None:
    """Collective: every rank participates in the gather; rank 0 writes ``path`` atomically."""
    osd = optimizer.state_dict()
    optimizer._dear.synchronize(host=True)
    if runtime.rank() == 0:
        msd = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
        osd_cpu = {"state": {i: {k: v.cpu() for k, v in e.items()} for i, e in osd["state"].items()},
                   "param_groups": osd["param_groups"], "dear": osd["dear"]}
        tmp = path + ".tmp.%d" % os.getpid()
        torch.save({"model": msd, "optimizer": osd_cpu, "extra": extra or {}}, tmp)
        os.replace(tmp, path)
    runtime.barrier()


def load_checkpoint(path: str, model: torch.nn.Module, optimizer, map_location="cpu") -> dict:
    """Collective: every rank reads ``path`` and restores the model and its shard of the state."""
    ckpt = torch.load(path, map_location=map_location, weights_only=False)
    optimizer._dear.synchronize(host=True)
    with torch.no_grad():
        own = model.state_dict()
        for k, v in ckpt["model"].items():
            own[k].copy_(v)          # in place: parameters stay views of the buckets
    optimizer._dear.backend.init_master_shards()
    optimizer.load_state_dict(ckpt["optimizer"])
    runtime.barrier()
    return ckpt.get("extra", {})
