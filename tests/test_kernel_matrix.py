"""Every instantiation of the fused reduce-scatter (Kernel A: ``rs_kernel``, ``rs_pipe_kernel``) and update (Kernel B:
``ag_kernel``) kernels against exact and float64 references, at bucket level through ``BucketSet``.

One worker body runs on the host emulation (CPU, always) and on the CUDA kernels (gpu marker); ranks share one GPU when
there is only one.  Each (backend, world, algorithm) is one ``run_ranks`` call that loops over a list of configurations
(parameter dtype and wire, epilogue, optimizer), building a fresh ``BucketSet`` for each.  ``test_matrix_reaches_every_
instantiation`` maps every configuration to the template arguments the dispatch picks (``launch_rs``, ``launch_rs_pipe``,
``launch_ag``) and fails if a reachable instantiation is not run; each worker checks ``rs_plan`` against that mapping.

Oracles:
* Kernel A's shard, bit for bit (NaN matches NaN): ``fl32(sum_q fl32(g_q as T)) * s`` with an fp32 accumulator that
  starts at 0, summed in the variant's order (rank order for one-shot; ``rank+1, ..., rank`` for the pipelined kernel)
  and ``s = fl32(grad_scale) / fl32(P)``, times ``fl32(1 / scale)`` under a dynamic loss scale.
* The overflow word, the scaler's decision and growth / backoff, and a skipped step leaving everything untouched.
* The clipping slots against a float64 sum of squares; ``total_norm`` as the documented fp32 combine of every rank's slots
  (slot order within a rank, then rank order); ``coef`` as ``clip_coef`` in fp32; both bit-identical on all ranks.
* Kernel B against torch.optim's SGD / Adam / AdamW formulas in float64, from the state before the step and the kernel's
  own (bit-checked) gradient shard and coefficient; exact invariants for HYPER_SKIP, 16-bit parameters (== master
  rounded), the parameter buffer (identical on every rank) and the count of applied updates.

A third part checks the general collectives (``gen_kernel``): reductions bit for bit, copies byte for byte."""
import collections
import hashlib

import numpy as np
import pytest
import torch

from _mp import run_ranks

ENV = {"DEAR_SPIN_TIMEOUT_S": "15"}
ALGO_ENV = {
    "oneshot": {"DEAR_RS_ALGO": "oneshot"},
    # 64 KiB stripe target: several stripes per bucket, and shards that are not a multiple of the 16 KiB pull chunk
    "pipe": {"DEAR_RS_ALGO": "pipe", "DEAR_PIPE_MIN_MB": "0", "DEAR_STRIPE_MB": "0.0625"},
    "nvls": {"DEAR_RS_ALGO": "nvls", "DEAR_PROVIDER": "vmm", "DEAR_MULTICAST": "1"},
}
DTS = ("f32", "bf16", "f16")
TORCH_DT = {"f32": torch.float32, "bf16": torch.bfloat16, "f16": torch.float16}
INT_VIEW = {"f32": torch.int32, "bf16": torch.int16, "f16": torch.int16}
CODE = {"f32": "DT_F32", "bf16": "DT_BF16", "f16": "DT_F16"}
ES = {"f32": 4, "bf16": 2, "f16": 2}
MANT = {"f32": 24, "bf16": 8, "f16": 11}          # significand bits of the wire type
HYPER_SKIP = 2                                     # HyperSeg::nesterov bit 1 (csrc/dear_common.h)
OPT_SGD, OPT_ADAM, OPT_ADAMW = 0, 1, 2
GROWTH_INTERVAL = 2
U = 2.0 ** -24                                     # fp32 unit roundoff; one ulp of x in [1, 2) is 2U

# Kernel B is checked against float64 with a bound of a few fp32 ulps of the magnitudes that enter each result (the
# sum of the absolute values of its terms).  Device and emulation differ here by design: nvcc contracts a*b+c into FMA
# (one rounding instead of two) and the Adam path has sqrt, two divisions and fp32 bias corrections, so neither is
# bit-exact against the other.  SGD's chain (coef, decay, momentum, nesterov, step) has at most 6 roundings; Adam's
# has about 10.  Adam's bias corrections 1 - beta^t are formed in fp32 with powf (a few ulps), which the cancellation
# amplifies by beta^t / (1 - beta^t); that factor is added on the update term explicitly.
ULPS_SGD = 4
ULPS_ADAM = 8

SGD_GROUPS = [dict(kind=OPT_SGD, lr=0.1, wd=1e-2, mu=0.9, damp=0.1, nest=0, b2=0.0, eps=0.0),
              dict(kind=OPT_SGD, lr=0.05, wd=5e-3, mu=0.8, damp=0.0, nest=1, b2=0.0, eps=0.0),
              dict(kind=OPT_SGD, lr=0.2, wd=1e-3, mu=0.0, damp=0.0, nest=0, b2=0.0, eps=0.0)]
ADAM_GROUPS = [dict(kind=OPT_ADAM, lr=1e-3, wd=1e-2, mu=0.9, damp=0.0, nest=0, b2=0.999, eps=1e-8),
               dict(kind=OPT_ADAMW, lr=2e-3, wd=5e-2, mu=0.8, damp=0.0, nest=0, b2=0.95, eps=1e-6)]
# non-finite values injected on AMP steps 3..6 (one per step, on one rank): where, value
INJECT = [("body", float("inf")), ("tail", float("nan")), ("tile_end", float("-inf")), ("last", float("nan"))]

Cfg = collections.namedtuple("Cfg", "pdt wire epi opt big")


def configs(world, algo):
    """The configurations one (world, algorithm) run loops over.  Per parameter dtype the (epilogue, optimizer) pairs
    reach Kernel A's AMP x CLIP and Kernel B's ADAM x CLIP; converting sets (fp32 parameters, 16-bit wire) add CVT."""
    pairs = [("none", "sgd"), ("static", "sgd_nobuf"), ("amp", "adam"), ("clip", "sgd"), ("ampclip", "adam")]
    out = [Cfg(p, p, e, o, p == "f32" and e == "clip") for p in DTS for e, o in pairs]
    if world > 1:
        cvt = [("none", "adam"), ("amp", "sgd"), ("clip", "adam"), ("ampclip", "sgd_nobuf")]
        if algo == "pipe":
            cvt = cvt[1:2]            # converting sets fall back to one-shot under pipe: one case checks the fallback
        out += [Cfg("f32", w, e, o, False) for w in ("bf16", "f16") for e, o in cvt]
    return out


def planned_algo(cfg, world, algo):
    """The Kernel A variant BucketSet picks (communicator.cpp: one rank and converting sets run one-shot under pipe)."""
    if world == 1:
        return "oneshot"
    if algo == "pipe" and cfg.wire != cfg.pdt:
        return "oneshot"
    return algo


def kernel_tuples(cfg, world, algo):
    """Template arguments of the kernels the dispatch launches for one configuration (kernels.cu: launch_rs, launch_ag;
    rs_pipe.cu: launch_rs_pipe).  W is the world for 1, 2, 4, 8 and 0 (the generic code) otherwise."""
    W = world if world in (1, 2, 4, 8) else 0
    amp, clip = cfg.epi in ("amp", "ampclip"), cfg.epi in ("clip", "ampclip")
    cvt, mc = cfg.wire != cfg.pdt, algo == "nvls"
    rs = planned_algo(cfg, world, algo)
    out = {("ag_kernel", cfg.pdt, W, mc, cfg.opt == "adam", clip)}
    if rs == "pipe":
        out.add(("rs_pipe_kernel", cfg.wire, amp, clip))
    else:
        out.add(("rs_kernel", cfg.wire, W, mc and rs == "nvls", amp, clip, cvt))
    return out


def reachable(worlds, mc=False):
    """Every instantiation a box running `worlds` can launch (MC: the NVLS multicast ones instead)."""
    Ws = {w if w in (1, 2, 4, 8) else 0 for w in worlds}
    out = set()
    for T in DTS:
        for W in Ws:
            if mc and W == 1:
                continue
            for a in (False, True):
                for c in (False, True):
                    out.add(("rs_kernel", T, W, mc, a, c, False))
                    out.add(("ag_kernel", T, W, mc, a, c))
                    if T != "f32" and W != 1:
                        out.add(("rs_kernel", T, W, mc, a, c, True))
                    if not mc and any(w > 1 for w in worlds):
                        out.add(("rs_pipe_kernel", T, a, c))
    return out


# ---------------------------------------------------------------------------------------------------- bucket layouts
def _round(x, q):
    return (x + q - 1) // q * q


def std_layout(es, world):
    """Segments (start, numel, kind) in elements of the bucket (wire) dtype, starts multiples of 64 elements: 1-, 3- and
    7-element vector tails, one 64 KiB tile exactly, one tile plus one element, one over three tiles, a segment absent
    on one rank (zero-filled over stale bucket bytes), a gap, a parameter absent on every rank (HYPER_SKIP) and a last
    segment that ends the bucket.  One hyper segment per parameter, so neighbours differ."""
    tile = 65536 // es
    spec = [(1001, "src"), (515, "src"), (263, "src"), (tile, "src"), (tile + 1, "src"), (3 * tile + 5, "src"),
            (777, "zero_stale"), (None, "gap"), (300, "absent"), (None, "last")]
    segs, off = [], 0
    for k, kind in spec:
        off = _round(off, 64)
        if kind == "gap":
            off += 128
            continue
        if kind == "last":
            n = _round(off + 1000, world * 64)
            segs.append((off, n - off, "src"))
            break
        segs.append((off, k, kind))
        off += k
    ends = [s for s, _, _ in segs[1:]] + [n]
    L = dict(n=n, segs=segs, tile=tile, hyper=[(e, i, segs[i][2]) for i, e in enumerate(ends)])
    sh = n // world
    assert world == 1 or any(s < q * sh < s + k for s, k, _ in segs for q in range(1, world)), "no shard boundary in a segment"
    return L


def wide_layout(world, npack, nhyper, staged):
    """`npack` packed segments (+1 staged in place) and `nhyper` hyper segments: past the shared-memory caches of Kernel
    A (384 PackSeg) and Kernel B (256 HyperSeg) at 385 / 257.  Neighbouring hyper segments alternate two groups."""
    nparam = npack + (1 if staged else 0)
    segs = [(64 * i, 5 + 4 * (i % 5), "staged" if staged and i == nparam // 2 else "src") for i in range(nparam)]
    n = _round(64 * nparam, world * 64)
    ends = [segs[(j * nparam) // nhyper][0] for j in range(1, nhyper)] + [n]
    return dict(n=n, segs=segs, tile=None, hyper=[(e, j, "src") for j, e in enumerate(ends)])


def big_layout(es, world):
    """16 MiB of gradient in one segment and one hyper segment: a multi-CTA Kernel A whose clip combine sums many
    CTA partials."""
    n = _round((16 << 20) // es, world * 64)
    return dict(n=n, segs=[(0, n, "src")], tile=None, hyper=[(n, 0, "src")])


def inject_pos(L, where):
    a, d = L["segs"][0], L["segs"][5]
    return {"body": a[0] + 500, "tail": a[0] + a[1] - 1, "tile_end": d[0] + L["tile"] - 1, "last": L["n"] - 1}[where]


def make_grad(L, seed, absent_here):
    """This rank's fp32 gradient of the whole bucket: magnitudes spread over 1e-3 ... 1e2, zeros where it has none."""
    g = torch.Generator().manual_seed(seed)
    n = L["n"]
    v = torch.randn(n, generator=g) * torch.pow(10.0, torch.rand(n, generator=g) * 5 - 3)
    mask = torch.zeros(n, dtype=torch.bool)
    for s, k, kind in L["segs"]:
        if kind in ("src", "staged") or (kind == "zero_stale" and not absent_here):
            mask[s:s + k] = True
    return torch.where(mask, v, torch.zeros(()))


def _f32(x):
    return float(np.float32(x))


def hyper_rows(L, groups, rank, absent_rank):
    """set_hyper rows and the HYPER_SKIP flags of this rank for this step."""
    ends, rows = [], []
    for end, j, kind in L["hyper"]:
        h = dict(groups[j % (3 if len(groups) == 3 and L["tile"] is not None else 2)])
        h["skip"] = kind == "absent" or (kind == "zero_stale" and rank == absent_rank)
        ends.append(end)
        rows.append(h)
    return ends, rows


def hyper_arrays(ends, rows, lo, hi):
    """Per-element float64 hyper-parameters (fp32-rounded, as the kernels see them) of elements [lo, hi)."""
    lens = torch.tensor(np.diff([0] + ends))
    out = {}
    for key in ("kind", "lr", "wd", "mu", "damp", "nest", "b2", "eps", "skip"):
        vals = torch.tensor([_f32(float(r[key])) for r in rows], dtype=torch.float64)
        out[key] = torch.repeat_interleave(vals, lens)[lo:hi]
    return out


def ref_step(p, g, m, v, H, coef, first, t, has_mom, adam):
    """One torch.optim step in float64 (SGD with torch's momentum / dampening / Nesterov / L2 decay; Adam with L2
    decay; AdamW), with the error bound of each result: (p1, m1, v1, bound_p, bound_m, bound_v)."""
    gc = g * coef
    if adam:
        l2 = (H["kind"] == OPT_ADAM).double()
        g1 = gc + l2 * H["wd"] * p
        Mg = gc.abs() + l2 * (H["wd"] * p).abs()
        b1, b2 = H["mu"], H["b2"]
        m1 = b1 * m + (1 - b1) * g1
        Mm = b1 * m.abs() + (1 - b1) * Mg
        v1 = b2 * v + (1 - b2) * g1 * g1
        Mv = b2 * v + (1 - b2) * Mg * Mg
        bc1, bc2 = 1 - b1 ** t, 1 - b2 ** t
        denom = v1.sqrt() / bc2.sqrt() + H["eps"]
        upd = H["lr"] / bc1 * (m1 / denom)
        Mu = H["lr"] / bc1 * (Mm / denom)
        pw = torch.where(H["kind"] == OPT_ADAMW, p * (1 - H["lr"] * H["wd"]), p)
        p1 = pw - upd
        rel_bc = 8 * U * b1 ** t / bc1 + 4 * U * b2 ** t / bc2
        k = ULPS_ADAM * 2 * U
        bp, bm, bv = k * (p.abs() + Mu) + rel_bc * Mu, k * Mm, k * Mv
    else:
        g1 = gc + H["wd"] * p
        Mg = gc.abs() + (H["wd"] * p).abs()
        mu, damp = H["mu"], H["damp"]
        use = (mu > 0) & bool(has_mom)
        buf = g1 if first else mu * m + (1 - damp) * g1
        Mb = Mg if first else mu * m.abs() + (1 - damp) * Mg
        nest = H["nest"] > 0
        d = torch.where(use, torch.where(nest, g1 + mu * buf, buf), g1)
        Md = torch.where(use, torch.where(nest, Mg + mu * Mb, Mb), Mg)
        m1 = torch.where(use, buf, m)
        p1 = p - H["lr"] * d
        k = ULPS_SGD * 2 * U
        v1, bp, bm, bv = v, k * (p.abs() + H["lr"] * Md), torch.where(use, k * Mb, torch.zeros(())), torch.zeros(())
    # HYPER_SKIP: no gradient on this rank and none reduced -> untouched, bit for bit
    skip = (H["skip"] > 0) & (g == 0)
    zero = torch.zeros(())
    return (torch.where(skip, p, p1), torch.where(skip, m, m1), torch.where(skip, v, v1),
            torch.where(skip, zero, bp), torch.where(skip, zero, bm), torch.where(skip, zero, bv))


def same_bits(a, b, what):
    """Bit for bit, except that every NaN matches every NaN."""
    na, nb = torch.isnan(a), torch.isnan(b)
    assert torch.equal(na, nb), "%s: NaN positions differ" % what
    bad = (a[~na].view(torch.int32) != b[~nb].view(torch.int32)).nonzero()
    assert bad.numel() == 0, "%s: %d elements differ, first at %d: %r != %r" % (
        what, bad.numel(), int(bad[0]), float(a[~na][bad[0]]), float(b[~nb][bad[0]]))


def _bits(t, dt):
    return t.contiguous().view(INT_VIEW[dt])


def _within(got, want, bound, what):
    err = (got - want).abs()
    bad = (err > bound).nonzero()
    assert bad.numel() == 0, "%s: %d elements off, first at %d: got %r want %r bound %r" % (
        what, bad.numel(), int(bad[0]), float(got[bad[0]]), float(want[bad[0]]), float(bound[bad[0]]))


# ---------------------------------------------------------------------------------------------------- the worker
def run_config(C, comm, dev, rank, world, algo, ci, cfg):
    tdt, wdt = TORCH_DT[cfg.pdt], TORCH_DT[cfg.wire]
    wes = ES[cfg.wire]
    cvt = cfg.wire != cfg.pdt
    amp, clip = cfg.epi in ("amp", "ampclip"), cfg.epi in ("clip", "ampclip")
    adam, has_mom = cfg.opt == "adam", cfg.opt != "sgd_nobuf"
    zero_grad = amp or cfg.opt == "sgd_nobuf"
    groups = ADAM_GROUPS if adam else SGD_GROUPS
    lays = [std_layout(wes, world), wide_layout(world, 384, 256, False), wide_layout(world, 385, 257, True)]
    if cfg.big:
        lays.append(big_layout(wes, world))
    nb = len(lays)
    bs = C.BucketSet(comm, [L["n"] for L in lays], getattr(C, CODE[cfg.pdt]), True,
                     getattr(C, CODE[cfg.wire]) if cvt else None)
    want_algo = planned_algo(cfg, world, algo)
    for b in range(nb):
        plan = bs.rs_plan(b)
        assert plan.split(":")[0] == want_algo and (":wire=" in plan) == cvt, (cfg, plan)
    g0 = torch.Generator().manual_seed(1000 + ci)
    st = []
    for b, L in enumerate(lays):
        n = L["n"]
        sh = n // world
        init = torch.zeros(n)
        for s, k, _ in L["segs"]:
            init[s:s + k] = torch.randn(k, generator=g0)
        pbuf = bs.param_buffer(b)
        pbuf.copy_(init.to(tdt))
        S = dict(L=L, pbuf=pbuf, gbuf=bs.grad_buffer(b), lo=rank * sh, sh=sh, gs=torch.zeros(sh, device=dev),
                 mom=torch.zeros(sh, device=dev) if has_mom else None, var=torch.zeros(sh, device=dev) if adam else None,
                 master=pbuf[rank * sh:(rank + 1) * sh].float().clone() if cfg.pdt != "f32" else None)
        bs.set_shards(b, S["gs"], S["mom"], S["master"], S["var"])
        bs.set_step(b, 0)
        st.append(S)
    scale, tracker, applied = 1024.0, 0, 0
    if amp:
        ampst = torch.zeros(9, dtype=torch.int32, device=dev)
        ampst.view(torch.float32)[2] = scale
        ampst.view(torch.float32)[5] = 2.0
        ampst.view(torch.float32)[6] = 0.5
        ampst[7] = GROWTH_INTERVAL
        bs.set_amp(ampst)
    slots = [nb - b for b in range(nb)]           # engine-wide numbering, not local order; slot 0 belongs to nobody here
    max_norm = 1.0 if cfg.epi == "clip" else 1e4
    if clip:
        clipst = torch.zeros(C.clip_state_floats(nb + 1), dtype=torch.float32, device=dev)
        clipst[0] = max_norm
        clipst.view(torch.int32)[3] = nb + 1
        bs.set_clip(clipst, slots)
    gscale = 1.0
    if cfg.epi == "static":
        gscale = 1.0 / 96
        bs.set_grad_scale(gscale)

    recs = []
    for step in range(3 + (len(INJECT) if amp else 0)):
        inj = INJECT[step - 3] if step >= 3 else None
        absent_rank = step % world
        allg = []
        for b, S in enumerate(st):
            L = S["L"]
            seed = ((ci * 16 + step) * 16 + b) * 16
            gq = [make_grad(L, seed + q, q == absent_rank).to(tdt) for q in range(world)]
            if inj is not None and b == 0:
                pos = inject_pos(L, inj[0])
                gq[(step + 1) % world][pos] = inj[1]
                S["inj"] = pos
            allg.append(gq)
            mine = gq[rank].to(dev)
            S["keep"] = mine
            src, off, nby, fl = [], [], [], []
            for s, k, kind in L["segs"]:
                off.append(s * wes)
                nby.append(k * wes)
                if kind == "staged":
                    S["gbuf"][s:s + k].copy_(mine[s:s + k])       # torch rounds a converting set's gradient
                    src.append(0); fl.append(0)
                elif kind == "absent" or (kind == "zero_stale" and rank == absent_rank):
                    S["gbuf"][s:s + k].fill_(7.0)                  # stale bytes the zero fill must clear
                    src.append(0); fl.append(C.SEG_ZERO_FILL)
                else:
                    src.append(mine.data_ptr() + s * mine.element_size()); fl.append(0)
            bs.set_pack(b, src, off, nby, fl)
            ends, rows = hyper_rows(L, groups, rank, absent_rank)
            bs.set_hyper(b, ends, [r["lr"] for r in rows], [r["wd"] for r in rows], [r["mu"] for r in rows],
                         [r["damp"] for r in rows], [r["nest"] | (HYPER_SKIP if r["skip"] else 0) for r in rows],
                         opt=[r["kind"] for r in rows], beta2=[r["b2"] for r in rows], eps=[r["eps"] for r in rows])
            S["H"] = hyper_arrays(ends, rows, S["lo"], S["lo"] + S["sh"])
            S["p0"] = S["pbuf"].clone()
            S["m0"] = S["mom"].clone() if has_mom else None
            S["v0"] = S["var"].clone() if adam else None
            S["w0"] = S["master"].clone() if S["master"] is not None else None
        # ---- Kernel A
        for b in range(nb):
            bs.reduce_scatter(b, True)
        bs.synchronize()
        s = torch.tensor(gscale, dtype=torch.float32) / torch.tensor(float(world), dtype=torch.float32)
        if amp:
            s = s * (torch.tensor(1.0, dtype=torch.float32) / torch.tensor(scale, dtype=torch.float32))
        any_bad = False
        cst = clipst.cpu() if clip else None
        for b, S in enumerate(st):
            lo, sh = S["lo"], S["sh"]
            order = [(rank + 1 + j) % world for j in range(world)] if want_algo == "pipe" else range(world)
            acc = torch.zeros(sh)
            for q in order:
                x = allg[b][q][lo:lo + sh]
                acc = acc + (x.to(wdt).float() if cvt else x.float())
            want = acc * s
            got = S["gs"].cpu()
            what = "%s step %d bucket %d shard" % (cfg, step, b)
            ex = sum((allg[b][q][lo:lo + sh].to(wdt) if cvt else allg[b][q][lo:lo + sh]).double() for q in range(world))
            mag = sum((allg[b][q][lo:lo + sh].to(wdt) if cvt else allg[b][q][lo:lo + sh]).double().abs()
                      for q in range(world)) * float(s)
            fin = torch.isfinite(want)
            if algo == "nvls":
                # the switch sums in its own order and returns the wire type: one rounding of the wire per addition
                _within(got.double()[fin], want.double()[fin], (world * 2.0 ** -MANT[cfg.wire] * mag)[fin], what)
                assert torch.equal(fin, torch.isfinite(got)), what
            elif world == 1:
                # one rank: the device's direct pack writes g * s with no accumulator, so a gradient of -0 (an fp16
                # underflow) stays -0 where the accumulator gives +0; the sign of a zero is the only freedom here
                same_bits(got + 0.0, want + 0.0, what)
            else:
                same_bits(got, want, what)
            # sanity: the float64 sum, within the fp32 roundings of P additions and one multiplication
            _within(got.double()[fin], (ex * float(s))[fin], ((world + 2) * U * mag)[fin], what + " vs float64")
            any_bad |= not bool(fin.all())
            S["got"] = got
            if clip:
                ref = float((got.double() ** 2).sum())
                val = float(cst[4 + slots[b]])
                # the device sums per thread, then over warps and CTAs: relative 1e-5.  The emulation adds the squares
                # one after the other in fp32, whose worst-case error grows with the count (sh * U)
                rel = 1e-5 if comm.is_cuda() else max(1e-5, sh * U)
                if np.isfinite(ref):
                    assert abs(val - ref) <= rel * ref + 1e-30, (what, "clip slot", val, ref)
        ov = None
        if amp:
            ov = int(ampst[0])
            assert ov == int(any_bad), (cfg, step, "overflow word", ov)
        # ---- Kernel B
        first = applied == 0
        for b in range(nb):
            bs.allgather_update(b, True, first, True, zero_grad, b == 0 and (amp or clip))
        bs.synchronize()
        skipped = inj is not None
        if amp:
            a = ampst.cpu()
            if skipped:
                scale, tracker = scale * 0.5, 0
            else:
                tracker += 1
                if tracker == GROWTH_INTERVAL:
                    scale, tracker = scale * 2.0, 0
            assert (int(a[0]), int(a[1]), float(a.view(torch.float32)[2]), int(a[3]), int(a[4])) == (
                0, int(skipped), scale, tracker, applied + (0 if skipped else 1)), (cfg, step, a.tolist())
        t = applied + 1
        if not skipped:
            applied += 1
        cst = clipst.cpu() if clip else None
        coef = float(cst[2]) if clip else 1.0
        hashes = []
        for b, S in enumerate(st):
            lo, sh = S["lo"], S["sh"]
            what = "%s step %d bucket %d" % (cfg, step, b)
            pb = S["pbuf"].cpu()
            master = S["master"].cpu() if S["master"] is not None else pb[lo:lo + sh].float()
            mom = S["mom"].cpu() if has_mom else torch.zeros(sh)
            var = S["var"].cpu() if adam else torch.zeros(sh)
            if skipped:
                assert torch.equal(_bits(pb, cfg.pdt), _bits(S["p0"].cpu(), cfg.pdt)), what + ": parameters moved"
                if S["w0"] is not None:
                    assert torch.equal(_bits(master, "f32"), _bits(S["w0"].cpu(), "f32")), what + ": master moved"
                if has_mom:
                    assert torch.equal(_bits(mom, "f32"), _bits(S["m0"].cpu(), "f32")), what + ": momentum moved"
                if adam:
                    assert torch.equal(_bits(var, "f32"), _bits(S["v0"].cpu(), "f32")), what + ": exp_avg_sq moved"
            else:
                p0 = (S["w0"].cpu() if S["w0"] is not None else S["p0"].cpu()[lo:lo + sh].float()).double()
                m0 = S["m0"].cpu().double() if has_mom else torch.zeros(sh, dtype=torch.float64)
                v0 = S["v0"].cpu().double() if adam else torch.zeros(sh, dtype=torch.float64)
                p1, m1, v1, bp, bm, bv = ref_step(p0, S["got"].double(), m0, v0, S["H"], coef, first, t, has_mom, adam)
                _within(master.double(), p1, bp, what + " parameters vs float64")
                if has_mom:
                    _within(mom.double(), m1, bm, what + " momentum / exp_avg vs float64")
                if adam:
                    _within(var.double(), v1, bv, what + " exp_avg_sq vs float64")
            if S["master"] is not None:
                assert torch.equal(_bits(pb[lo:lo + sh], cfg.pdt), _bits(master.to(tdt), cfg.pdt)), \
                    what + ": 16-bit parameters are not the master rounded"
            if zero_grad:
                assert not S["gbuf"].cpu().any(), what + ": gradient bucket not zeroed"
            hashes.append(hashlib.sha1(pb.view(torch.uint8).numpy().tobytes()).hexdigest())
        rec = dict(cfg=tuple(cfg), step=step, hashes=hashes, ov=ov, clip=clip, amp=amp, max_norm=max_norm,
                   inj_rank=(st[0]["inj"] // st[0]["sh"]) if inj is not None else None)
        if clip:
            rec.update(slots=[float(x) for x in cst[4:4 + nb + 1]], total=float(cst[1]), coef=float(cst[2]))
        recs.append(rec)
    del bs
    return recs


def matrix_worker(rank, world, algo):
    import dear_pytorch_b200 as dear
    from dear_pytorch_b200 import ops
    C = ops.require_native()
    comm = dear.communicator()
    dev = dear.device()
    if algo == "nvls":
        probe = C.BucketSet(comm, [world * 4096], C.DT_F32, True)
        ok = probe.has_multicast()
        del probe
        if not ok:
            return "no-multicast"
    recs = []
    for ci, cfg in enumerate(configs(world, algo)):
        recs += run_config(C, comm, dev, rank, world, algo, ci, cfg)
    comm.check_status()
    return recs


def _f(x):
    return np.float32(x)


def check_ranks(outs, world):
    """What needs every rank: identical parameters, the documented norm combine, and the overflow bit on exactly the
    rank whose shard holds the injected value."""
    assert all(len(o) == len(outs[0]) for o in outs)
    for recs in zip(*outs):
        r0 = recs[0]
        what = "%s step %d" % (r0["cfg"], r0["step"])
        assert all(r["hashes"] == r0["hashes"] for r in recs), what + ": parameter buffers differ between ranks"
        if r0["clip"]:
            with np.errstate(all="ignore"):
                total = _f(0)
                for r in recs:                       # rank order of each rank's slot-order partial
                    part = _f(0)
                    for x in r["slots"]:
                        part = _f(part + _f(x))
                    total = _f(total + part)
                total = np.sqrt(total, dtype=np.float32)
                coef = _f(_f(r0["max_norm"]) / _f(total + _f(1e-6)))
                coef = _f(1) if coef > 1 else coef
            for r in recs:
                same_bits(torch.tensor([r["total"], r["coef"]]), torch.tensor([float(total), float(coef)]),
                          what + " total_norm / coef")
        if r0["amp"]:
            want = [int(q == r0["inj_rank"]) for q in range(world)]
            assert [r["ov"] for r in recs] == want, (what, "overflow words", [r["ov"] for r in recs], want)


RUNS = [(1, "oneshot"), (2, "oneshot"), (3, "oneshot"), (4, "oneshot"), (8, "oneshot"), (2, "pipe"), (3, "pipe"),
        (4, "pipe")]


def test_matrix_reaches_every_instantiation():
    """The configurations of RUNS launch every instantiation of rs_kernel, rs_pipe_kernel and ag_kernel that a box
    with one H100 (ranks sharing it, worlds 1-4) can reach, and W = 8 with eight GPUs.  The MC (NVLS) ones are
    checked by the multicast test.  Each worker asserts that rs_plan agrees with planned_algo."""
    ngpu = torch.cuda.device_count() if torch.cuda.is_available() else 0
    worlds = [1, 2, 3, 4] + ([8] if ngpu >= 8 else [])
    covered = set()
    for world, algo in RUNS:
        if world in worlds:
            for cfg in configs(world, algo):
                covered |= kernel_tuples(cfg, world, algo)
    missing = reachable(worlds) - covered
    assert not missing, sorted(missing)
    counts = collections.Counter(t[0] for t in covered)
    assert counts == {"rs_kernel": 72 + (24 if 8 in worlds else 0), "ag_kernel": 48 + (12 if 8 in worlds else 0),
                      "rs_pipe_kernel": 12}, counts


def _gpu_world_ok(world):
    n = torch.cuda.device_count()
    if world == 8:
        return n >= 8
    return n == 1 or n >= world or world % n == 0


@pytest.mark.parametrize("world,algo", [r for r in RUNS if r[0] != 8])
def test_emulated_matrix(world, algo):
    """Host emulation: the same oracles, bit-exact where the kernels are.  At P >= 3 the pipelined order differs from
    rank order, so the emulation must follow the kernel's rotation."""
    check_ranks(run_ranks(matrix_worker, world=world, backend="emu", args=(algo,), extra_env=dict(ENV, **ALGO_ENV[algo]),
                          timeout=900), world)


@pytest.mark.gpu
@pytest.mark.parametrize("world,algo", RUNS)
def test_cuda_matrix(world, algo):
    if not _gpu_world_ok(world):
        pytest.skip("W = 8 needs eight GPUs" if world == 8 else "ranks cannot share the GPUs evenly")
    outs = run_ranks(matrix_worker, world=world, backend="b200", args=(algo,), extra_env=dict(ENV, **ALGO_ENV[algo]),
                     timeout=900)
    check_ranks(outs, world)


@pytest.mark.gpu
@pytest.mark.multigpu
def test_cuda_matrix_nvls():
    """The MC instantiations: multimem.ld_reduce in Kernel A (one wire rounding per addition) and multimem.st in
    Kernel B.  Needs an NVSwitch that can bind a multicast object."""
    world = min(torch.cuda.device_count(), 8)
    covered = set()
    for cfg in configs(world, "nvls"):
        covered |= kernel_tuples(cfg, world, "nvls")
    missing = reachable([world], mc=True) - covered
    assert not missing, sorted(missing)
    outs = run_ranks(matrix_worker, world=world, backend="b200", args=("nvls",), extra_env=dict(ENV, **ALGO_ENV["nvls"]),
                     timeout=900)
    if outs[0] == "no-multicast":
        pytest.skip("this box cannot create an NVLS multicast object")
    check_ranks(outs, world)


# ---------------------------------------------------------------------------------------------------- general ops
GEN_LENGTHS = [1, 15, 16, 17, 1_000_003]
COPY_LENGTHS = [1, 17, 2_500_001]


def _view(n, dt, off, dev, fill=None):
    """A contiguous tensor of n elements that starts `off` elements into its allocation (off = 1: not 16-byte aligned)."""
    base = torch.zeros(n + off + 16, dtype=dt, device=dev)
    t = base[off:off + n]
    if fill is not None:
        t.copy_(fill)
    return t


def _rank_vals(seed, n, dt):
    g = torch.Generator().manual_seed(seed)
    if dt in (torch.uint8, torch.int64):
        hi = 256 if dt == torch.uint8 else 1 << 62
        return torch.randint(0, hi, (n,), generator=g, dtype=torch.int64).to(dt)
    return (torch.randn(n, generator=g) * torch.pow(10.0, torch.rand(n, generator=g) * 4 - 2)).to(dt)


def gen_worker(rank, world):
    import dear_pytorch_b200 as dear
    comm = dear.communicator()
    dev = dear.device()
    scale = 1.0 / 3
    sc = torch.tensor(scale, dtype=torch.float32)
    root = world - 1
    for dn in DTS:
        dt = TORCH_DT[dn]
        for n in GEN_LENGTHS:
            for off in (0, 1):
                what = "%s n=%d off=%d" % (dn, n, off)
                vals = [_rank_vals(7 * n + 31 * q + off, n, dt) for q in range(world)]
                acc = torch.zeros(n)
                for q in range(world):
                    acc = acc + vals[q].float()
                want = (acc * sc).to(dt)
                t = _view(n, dt, off, dev, vals[rank])
                comm.allReduce(t, scale)
                comm.synchronize()
                same_bits(t.cpu().float(), want.float(), "allReduce " + what)
                t = _view(n, dt, off, dev, vals[rank])
                comm.reduce(t, root, scale)
                comm.synchronize()
                same_bits(t.cpu().float(), (want if rank == root else vals[rank]).float(), "reduce " + what)
                # reduceScatter: rank q's send holds world rows of n; row r goes to rank r
                sends = [_rank_vals(11 * n + 37 * q + off, world * n, dt) for q in range(world)]
                acc = torch.zeros(n)
                for q in range(world):
                    acc = acc + sends[q][rank * n:(rank + 1) * n].float()
                send = _view(world * n, dt, off, dev, sends[rank])
                recv = _view(n, dt, off, dev)
                comm.reduceScatter(send, recv, scale)
                comm.synchronize()
                same_bits(recv.cpu().float(), (acc * sc).to(dt).float(), "reduceScatter " + what)
    for dt, offs in ((torch.uint8, (1, 4)), (torch.int64, (0, 1))):
        for n in COPY_LENGTHS:
            for off in offs:
                what = "%s n=%d off=%d" % (dt, n, off)
                vals = [_rank_vals(5 * n + 13 * q + off, n, dt) for q in range(world)]
                send = _view(n, dt, off, dev, vals[rank])
                recv = _view(world * n, dt, off, dev)
                comm.allGather(send, recv)
                comm.synchronize()
                assert torch.equal(recv.cpu(), torch.cat(vals)), "allGather " + what
                t = _view(n, dt, off, dev, vals[rank])
                comm.bcast(t, root)
                comm.synchronize()
                assert torch.equal(t.cpu(), vals[root]), "bcast " + what
                peer = (rank + 1) % world
                recv = _view(n, dt, off, dev)
                comm.sendrecv(send, recv, peer)
                comm.synchronize()
                assert torch.equal(recv.cpu(), vals[peer]), "sendrecv " + what
    comm.check_status()
    return True


# 1 MiB of staging: the long cases run in several chunks (communicator.cpp: gen_chunked, reduce_scatter)
GEN_ENV = {"DEAR_STAGING_MB": "1"}


@pytest.mark.parametrize("world", [2, 3])
def test_emulated_general_ops(world):
    assert all(run_ranks(gen_worker, world=world, backend="emu", extra_env=dict(ENV, **GEN_ENV), timeout=600))


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_cuda_general_ops(world):
    if not _gpu_world_ok(world):
        pytest.skip("ranks cannot share the GPUs evenly")
    assert all(run_ranks(gen_worker, world=world, backend="b200", extra_env=dict(ENV, **GEN_ENV), timeout=600))
