"""The optimizer families of the fused update (SGD, Adam / AdamW, RMSprop): how each ``torch.optim`` class maps onto
the update kernels (``csrc/dear_common.h``).  A family validates its param groups, turns a group into a hyper-parameter
row, names the fp32 state shards a bucket needs (``mom``: momentum buffer / exp_avg, ``var``: exp_avg_sq / square_avg,
``gavg``: grad_avg) and their torch state names, owns the step-count rules, and runs the eager update of TorchBackend.
"""
from __future__ import annotations

import math
from typing import NamedTuple

import torch

OPT_SGD, OPT_ADAM, OPT_ADAMW, OPT_RMSPROP = 0, 1, 2, 3
HYPER_NESTEROV, HYPER_SKIP, HYPER_CENTERED = 1, 2, 4   # bits of HyperRow.flags (csrc/dear_common.h)


class HyperRow(NamedTuple):
    """One segment of a bucket's hyper-parameter table, in the order of ``BucketSet.set_hyper``'s arguments.  A param
    group's row has ``end`` 0; the engine sets it per segment."""
    end: int
    lr: float
    weight_decay: float
    momentum: float         # SGD / RMSprop momentum, Adam beta1
    dampening: float        # SGD dampening, RMSprop 1 - alpha
    flags: int              # HYPER_NESTEROV | HYPER_SKIP | HYPER_CENTERED
    opt: int                # OPT_*
    beta2: float            # Adam beta2, RMSprop alpha
    eps: float              # Adam / RMSprop


class _Family:
    counts_steps = False    # torch.optim counts ``step`` per parameter; the engine tracks updates sat out (``_lag``)
    folds_lag = False       # ... and folds that lag into the parameter's row (``lag_adjust``)

    def validate(self, groups):
        for g in groups:
            if g.get("amsgrad", False) or g.get("capturable", False) or g.get("differentiable", False):
                raise ValueError("amsgrad / capturable / differentiable Adam variants are not supported")
        for g in groups:
            if g.get("maximize", False):
                raise ValueError("maximize=True is not supported")

    def tracks_first_gradient(self, groups) -> bool:
        """Whether a parameter's first gradient needs its own row (``DearEngine._virgin``)."""
        return False

    def has_entry(self, steps: int, started: bool) -> bool:
        """Whether ``state_dict()`` has an entry for a parameter of a bucket with state, after ``steps`` updates of
        its own (``started``: one of them was applied).  Adam: always, with step 0 before the first gradient."""
        return True


class SGD(_Family):
    def row(self, g) -> HyperRow:
        return HyperRow(0, float(g["lr"]), float(g.get("weight_decay", 0.0)), float(g.get("momentum", 0.0)),
                        float(g.get("dampening", 0.0)), HYPER_NESTEROV if g.get("nesterov", False) else 0, OPT_SGD,
                        0.0, 0.0)

    def shard_kinds(self, rows):
        return ("mom",) if any(r.momentum > 0 for r in rows) else ()

    def state_names(self, g):
        """(torch state name, shard kind) of a parameter of group ``g``; the first one decides whether it has state."""
        return (("momentum_buffer", "mom"),)

    def tracks_first_gradient(self, groups):
        # torch initialises a parameter's momentum buffer with its first gradient (undampened); the kernels know one
        # global "first step", so a parameter that starts later gets dampening 0 in its row for that one update
        return any(g.get("momentum", 0) != 0 and g.get("dampening", 0) != 0 for g in groups)

    def has_entry(self, steps, started):
        return started      # torch.optim.SGD has no buffer yet for a parameter that never received a gradient

    def restore_count(self, eng, carry, steps):
        if carry["mom_init"]:
            # momentum buffers exist, so the next update is not the first one (torch.optim.SGD keeps no count)
            carry["num_updates"] = max(carry["num_updates"], 1)

    def update(self, row, p, d, shards, sl, first_step, t):
        """Eager update of one row's range ``p`` (gradient ``d``, state ``shards[kind][sl]``, ``t`` updates applied so
        far); returns the number of kernels launched."""
        if row.weight_decay != 0:
            d = d.add(p, alpha=row.weight_decay)
        if row.momentum > 0:
            buf = shards["mom"][sl]
            if first_step:
                buf.copy_(d)
            else:
                buf.mul_(row.momentum).add_(d, alpha=1 - row.dampening)
            d = d.add(buf, alpha=row.momentum) if row.flags & HYPER_NESTEROV else buf
        p.add_(d, alpha=-row.lr)
        return 3


class Adam(_Family):
    """torch.optim.Adam (``OPT_ADAM``, L2 in the gradient) and AdamW (``OPT_ADAMW``, decoupled decay)."""
    counts_steps = True
    folds_lag = True

    def __init__(self, opt: int):
        self.opt = opt

    def row(self, g) -> HyperRow:
        b1, b2 = g["betas"]
        return HyperRow(0, float(g["lr"]), float(g.get("weight_decay", 0.0)), float(b1), 0.0, 0, self.opt, float(b2),
                        float(g["eps"]))

    def shard_kinds(self, rows):
        return ("mom", "var")

    def state_names(self, g):
        return (("exp_avg", "mom"), ("exp_avg_sq", "var"))

    def restore_count(self, eng, carry, steps):
        if steps:
            # the kernels keep ONE step count (the largest); parameters behind it get their bias correction adjusted
            # through their hyper row (lag_adjust)
            t = carry["num_updates"] = max(steps.values())
            eng._lag = {p: t - v for p, v in steps.items() if v < t}

    def lag_adjust(self, row: HyperRow, t: int, lag: int) -> HyperRow:
        """The row that makes the kernel's update with the GLOBAL step count ``t`` equal to Adam's update with the
        parameter's own count ``s = t - lag`` (torch.optim counts steps per parameter and skips a parameter without
        gradient):   lr/bc1(s) * m / (sqrt(v)/sqrt(bc2(s)) + eps)  ==  lr'/bc1(t) * m / (sqrt(v)/sqrt(bc2(t)) + eps')
        with  r = sqrt(bc2(s)/bc2(t)),  eps' = eps r,  lr' = lr r bc1(t)/bc1(s);  AdamW's decoupled decay keeps
        lr' wd' = lr wd."""
        lr, b1, b2, s = row.lr, row.momentum, row.beta2, t - lag
        r = math.sqrt((1.0 - b2 ** s) / (1.0 - b2 ** t)) if b2 < 1.0 else 1.0
        lr2 = lr * r * ((1.0 - b1 ** t) / (1.0 - b1 ** s) if 0.0 < b1 < 1.0 else 1.0)
        wd2 = row.weight_decay * lr / lr2 if (row.opt == OPT_ADAMW and lr2 != 0.0) else row.weight_decay
        return row._replace(lr=lr2, weight_decay=wd2, eps=row.eps * r)

    def update(self, row, p, d, shards, sl, first_step, t):
        t, mom, beta2, lr, wd = t + 1, row.momentum, row.beta2, row.lr, row.weight_decay
        m, v = shards["mom"][sl], shards["var"][sl]
        if row.opt == OPT_ADAM and wd != 0:
            d = d.add(p, alpha=wd)
        m.mul_(mom).add_(d, alpha=1 - mom)
        v.mul_(beta2).addcmul_(d, d, value=1 - beta2)
        bc1, bc2 = 1 - mom ** t, 1 - beta2 ** t
        if row.opt == OPT_ADAMW:
            p.mul_(1 - lr * wd)
        p.addcdiv_(m, v.sqrt().div_(bc2 ** 0.5).add_(row.eps), value=-lr / bc1)
        return 6


class RMSprop(_Family):
    """torch.optim.RMSprop: ``dampening`` holds 1 - alpha, ``beta2`` alpha, ``flags`` HYPER_CENTERED.  The step count
    changes none of the math; it is counted per parameter for ``state_dict()`` only."""
    counts_steps = True

    def validate(self, groups):
        for g in groups:
            for k in ("maximize", "capturable", "differentiable"):
                if g.get(k, False):
                    raise ValueError("RMSprop with %s=True is not supported by the fused update" % k)
            if isinstance(g["lr"], torch.Tensor):
                raise ValueError("RMSprop with a tensor lr is not supported by the fused update (pass a float)")
        super().validate(groups)

    def row(self, g) -> HyperRow:
        alpha = float(g["alpha"])
        # 1 - alpha is formed in double and rounded once, like the Python scalar torch hands to its kernels
        return HyperRow(0, float(g["lr"]), float(g.get("weight_decay", 0.0)), float(g.get("momentum", 0.0)),
                        1.0 - alpha, HYPER_CENTERED if g.get("centered", False) else 0, OPT_RMSPROP, alpha,
                        float(g["eps"]))

    def shard_kinds(self, rows):
        return (("mom",) if any(r.momentum > 0 for r in rows) else ()) + ("var",) + \
            (("gavg",) if any(r.flags & HYPER_CENTERED for r in rows) else ())

    def state_names(self, g):
        return ((("square_avg", "var"),) + ((("momentum_buffer", "mom"),) if g["momentum"] > 0 else ())
                + ((("grad_avg", "gavg"),) if g["centered"] else ()))

    def has_entry(self, steps, started):
        return steps > 0    # no entry before a parameter's first gradient

    def restore_count(self, eng, carry, steps):
        # no stored state: nothing has been applied yet; a parameter without an entry has not had a gradient (its
        # state is zero, and so is its count)
        t = carry["num_updates"] = max(steps.values(), default=0)
        eng._lag = {s.param: t - steps.get(s.param, 0) for s in eng.plan.slots if steps.get(s.param, 0) < t}

    def update(self, row, p, d, shards, sl, first_step, t):
        # torch.optim.RMSprop (_single_tensor_rmsprop)
        if row.weight_decay != 0:
            d = d.add(p, alpha=row.weight_decay)
        sq = shards["var"][sl]
        sq.mul_(row.beta2).addcmul_(d, d, value=row.dampening)
        if row.flags & HYPER_CENTERED:
            ga = shards["gavg"][sl]
            ga.lerp_(d, row.dampening)
            avg = sq.addcmul(ga, ga, value=-1).sqrt_().add_(row.eps)
        else:
            avg = sq.sqrt().add_(row.eps)
        if row.momentum > 0:
            buf = shards["mom"][sl]
            buf.mul_(row.momentum).addcdiv_(d, avg)
            p.add_(buf, alpha=-row.lr)
        else:
            p.addcdiv_(d, avg, value=-row.lr)
        return 5


def family_of(optimizer: torch.optim.Optimizer) -> _Family:
    """The family of the wrapped optimizer (``DistributedOptimizer``'s class derives from the user's class)."""
    if isinstance(optimizer, torch.optim.AdamW):
        return Adam(OPT_ADAMW)
    if isinstance(optimizer, torch.optim.Adam):
        return Adam(OPT_ADAM)
    if isinstance(optimizer, torch.optim.RMSprop):
        return RMSprop()
    if isinstance(optimizer, torch.optim.SGD):
        return SGD()
    raise TypeError(
        "the decoupled all-reduce fuses the parameter update into the all-gather kernel; supported: "
        "torch.optim.SGD (the reference's only DeAR optimizer, dear/dear_dopt.py:310-336), Adam, AdamW and "
        "RMSprop; got %s. Use parallel.baselines for other optimizers." % type(optimizer).__mro__[1].__name__)
