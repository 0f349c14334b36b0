"""The fused BatchNorm (``csrc/bn_act.cu``) and dropout-add-LayerNorm / bias-GELU (``csrc/ln_fused.cu``) kernels against
exact and float64 references, at the launch geometries the benchmarks reach.

Host-side mirrors of ``make_geo``, ``grid_for`` and ``bg_grid`` take the SM count as an argument.  The table tests (CPU
with 132 SMs, GPU with the device's own count) fail if the case lists miss a geometry regime, and the coverage test
fails if a template instantiation is not exercised.  The GPU tests call the native ops directly, so each stage is checked
from the kernel's own intermediate outputs (``s``, ``mean``, ``rstd``, ``scale``, ``shift``, ``y``, ``dz``), and the
launch counters confirm that the fused kernels ran.

Bounds.  References are float64, on the device, from the exact values the kernel reads.  ``U = 2^-24`` is the fp32 unit
roundoff.  A sequential fp32 sum of n terms is within ``n U sum|t|`` (first order); a tree is bounded by its depth, the
longest chain of additions any term takes (per-thread loop + shared-memory chain + partial loop + shuffle levels).  A
result stored in T from an fp32 value within ``e`` of the reference is within ``e + ulp_T(|ref| + e) / 2``.  CUDA's
documented errors: ``rsqrtf`` and ``erff`` 2 ulp, ``__expf(x)`` ``2 + floor(|1.173 x|)`` ulp; one fp32 ulp is at most
``2U`` relative.  Second-order terms (products of two ``U`` terms) are left out.  The float64 references' own rounding
(``~n 2^-53``) is unmeasured and negligible against these bounds."""
import math
import zlib

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

U = 2.0 ** -24
F32, BF16 = torch.float32, torch.bfloat16
DTS = (F32, BF16)
TNAME = {F32: "float", BF16: "bf16"}
VEC = {F32: 4, BF16: 8}                 # elements per 128-bit vector
PBITS = {F32: 24, BF16: 8}              # significand bits
CPU_SMS = 132                           # H100 SXM
# row counts that depend on the SM count: the forward grid (2 CTAs of 8 warps per SM) covers 2 * sms * 8 rows per pass
ROWS_ONE_PASS, ROWS_ONE_PASS_PLUS_1 = "2*sms*8", "2*sms*8+1"


# ------------------------------------------------------------------------------------------- geometry mirrors
def bn_geo(M, C, dt, sms):
    """bn_act.cu ``make_geo``; None where the kernel does not apply."""
    vec = VEC[dt]
    if C % vec:
        return None
    cv = C // vec
    txv = 1
    while txv < 64 and cv % (txv * 2) == 0:
        txv *= 2
    if txv < 4:
        return None
    ty = 256 // txv
    ch_groups = cv // txv
    want = -(-M // (ty * 8))
    cap = max(1, (sms * 8) // ch_groups)
    rb = max(1, min(want, cap))
    rpb = -(-M // rb)                                  # rows per stats block (contiguous chunks)
    last = M - (rb - 1) * rpb                          # rows of the last block; <= 0: trailing blocks are empty
    return dict(txv=txv, ty=ty, ch_groups=ch_groups, row_blocks=rb, cap_bound=want > cap, rpb=rpb,
                min_rows=min(rpb, last), vec=vec)


def ln_grid(rows, ctas_per_sm, sms):
    """ln_fused.cu ``grid_for``: CTAs of 8 warps, one row per warp per pass."""
    return max(1, min(-(-rows // 8), sms * ctas_per_sm))


def bg_grid(rows, N, dt, sms):
    """ln_fused.cu ``bg_grid``: (column blocks of 64 vectors, row groups of 4)."""
    gx = (N // VEC[dt] + 63) // 64
    gy = max(1, min((rows + 3) // 4, max(1, 2 * sms // gx)))
    return gx, gy


# ---------------------------------------------------------------------------------------------------- cases
# BatchNorm: (shape, relu, residual).  Small shapes run every (relu, residual) pair; the real ResNet-50 shapes at 64
# images run the pair the network uses there.
BN_PAIRS = [(True, False), (True, True), (False, False), (False, True)]
BN_SMALL = [
    (2, 64, 1, 1),        # M = 2
    (3, 96, 1, 5),        # M = 15 (odd), C = 96: txv 8 (fp32) / 4 (bf16), three channel groups
    (1, 48, 3, 3),        # fp32 only: txv 4, three channel groups (bf16 has 6 vectors: composite)
    (8, 64, 14, 14),      # 2..31 row blocks
    (2, 128, 7, 9),       # txv 32 (fp32) / 16 (bf16)
    (3, 160, 5, 5),       # DenseNet width 64 + 32k
    (4, 64, 90, 93),      # > 128 row blocks, not a multiple of 32
    (5, 256, 3, 5),       # txv 64 with one channel group
]
BN_REAL = [((64, 64, 112, 112), True, False),      # stem: cap-bound
           ((64, 256, 56, 56), True, True),        # bottleneck end: cap-bound, empty trailing stats blocks
           ((64, 2048, 7, 7), True, True)]         # last stage: 32..128 row blocks, several channel groups


def bn_cases():
    out = []
    for dt in DTS:
        for shape in BN_SMALL:
            if bn_geo(shape[0] * shape[2] * shape[3], shape[1], dt, CPU_SMS) is None:
                continue
            out += [(dt, shape, relu, res) for relu, res in BN_PAIRS]
        out += [(dt, shape, relu, res) for shape, relu, res in BN_REAL]
    return out


# LayerNorm: (rows, H); each runs without and with dropout, without and with the branch bias.
def ln_cases(dt):
    idle = 1016 if dt == BF16 else 1020          # last vector slot leaves one lane idle
    return [(1, 8), (7, 64), (100, idle), (2048, 1024), (ROWS_ONE_PASS, 768), (ROWS_ONE_PASS_PLUS_1, 136),
            (4096, 1024), (ROWS_ONE_PASS_PLUS_1, idle)]


def ln_rows(rows, sms):
    return {ROWS_ONE_PASS: 2 * sms * 8, ROWS_ONE_PASS_PLUS_1: 2 * sms * 8 + 1}.get(rows, rows)


LN_VARIANTS = [(0.0, False), (0.0, True), (0.1, False), (0.1, True)]     # (p, branch bias)

# bias-GELU: (rows, N)
BG_CASES = [(1, 520), (3, 4096), (130, 520), (2048, 4096), (4099, 520), (4096, 72)]


# --------------------------------------------------------------------------------------- regimes and coverage
def bn_regimes(dt, shape, sms):
    N, C, H, W = shape
    g = bn_geo(N * H * W, C, dt, sms)
    rb = g["row_blocks"]
    r = {("txv", TNAME[dt], g["txv"]), ("ch_groups", "1" if g["ch_groups"] == 1 else ">1")}
    if rb == 1:
        r.add(("rb", "1"))
    elif rb < 32:
        r.add(("rb", "2-31"))
    elif rb <= 128:
        r.add(("rb", "32-128"))
    elif rb % 32:
        r.add(("rb", ">128, not a multiple of 32"))
    if g["cap_bound"]:
        r.add(("rb", "cap-bound"))
    if g["min_rows"] < g["ty"]:
        r.add(("block", "fewer rows than ty"))
    M = N * H * W
    if M == 2:
        r.add(("M", "2"))
    if M % 2:
        r.add(("M", "odd"))
    return r


BN_REQUIRED = ({("txv", TNAME[dt], t) for dt in DTS for t in (4, 8, 16, 32, 64)}
               | {("ch_groups", "1"), ("ch_groups", ">1")}
               | {("rb", k) for k in ("1", "2-31", "32-128", ">128, not a multiple of 32", "cap-bound")}
               | {("block", "fewer rows than ty"), ("M", "2"), ("M", "odd")})


def ln_regimes(dt, rows, H, sms):
    n = ln_rows(rows, sms)
    r = {("H", H if H not in (1016, 1020) else "idle lanes")}
    r.add(("rows", {1: "1", 7: "7", 2048: "2048", 4096: "4096", 2 * sms * 8: "2*sms*8",
                    2 * sms * 8 + 1: "2*sms*8+1"}.get(n, "other")))
    parts = ln_grid(n, 1, sms)
    r.add(("colsum partials", "<16" if parts < 16 else (">16" if parts > 16 else "16")))
    return r


LN_REQUIRED = ({("H", h) for h in (8, 64, 136, 768, 1024, "idle lanes")}
               | {("rows", k) for k in ("1", "7", "2048", "2*sms*8", "2*sms*8+1", "4096")}
               | {("colsum partials", "<16"), ("colsum partials", ">16")})


def bg_regimes(dt, rows, N, sms):
    gx, gy = bg_grid(rows, N, dt, sms)
    r = set()
    if (N // VEC[dt]) % 64:
        r.add(("N/vec", "not a multiple of 64"))
    if N == 4096:
        r.add(("N", 4096))
    r.add(("rows", {1: "1", 3: "3", 2048: "2048"}.get(rows, ">=4096" if rows >= 4096 else "other")))
    r.add(("gy", "row-bound" if gy == (rows + 3) // 4 and gy < 2 * sms // gx else "SM-bound"))
    return r


BG_REQUIRED = {("N/vec", "not a multiple of 64"), ("N", 4096), ("rows", "1"), ("rows", "3"), ("rows", "2048"),
               ("rows", ">=4096"), ("gy", "row-bound"), ("gy", "SM-bound")}


def instantiations():
    """Template arguments every case dispatches to (bn_act.cu fwd_impl / bwd_impl, ln_fused.cu fwd_launch / bwd_launch /
    bias_gelu_*)."""
    got = set()
    for dt, shape, relu, res in bn_cases():
        t, a = TNAME[dt], "%s,%d,%d" % (TNAME[dt], relu, res)
        got |= {"bn_stats_kernel<%s>" % t, "train:bn_apply_kernel<%s>" % a, "eval:bn_apply_kernel<%s>" % a,
                "bn_bwd_reduce_kernel<%s>" % a, "bn_bwd_apply_kernel<%s>" % a}
    for dt in DTS:
        t = TNAME[dt]
        for _ in ln_cases(dt):
            for p, bias in LN_VARIANTS:
                got |= {"ln_fwd_kernel<%s,%d>" % (t, p > 0), "ln_bwd_kernel<%s,%d,%d>" % (t, p > 0, bias),
                        "colsum_finalize<%s>" % t}
        for _ in BG_CASES:
            got |= {"bias_gelu_fwd_kernel<%s>" % t, "bias_gelu_bwd_kernel<%s>" % t, "colsum_finalize<%s>" % t}
    return got


def required_instantiations():
    req = set()
    for dt in DTS:
        t = TNAME[dt]
        req.add("bn_stats_kernel<%s>" % t)
        for relu in (0, 1):
            for res in (0, 1):
                a = "%s,%d,%d" % (t, relu, res)
                req |= {"train:bn_apply_kernel<%s>" % a, "eval:bn_apply_kernel<%s>" % a,
                        "bn_bwd_reduce_kernel<%s>" % a, "bn_bwd_apply_kernel<%s>" % a}
        for drop in (0, 1):
            req.add("ln_fwd_kernel<%s,%d>" % (t, drop))
            for dbias in (0, 1):
                req.add("ln_bwd_kernel<%s,%d,%d>" % (t, drop, dbias))
        req |= {"colsum_finalize<%s>" % t, "bias_gelu_fwd_kernel<%s>" % t, "bias_gelu_bwd_kernel<%s>" % t}
    return req


def check_tables(sms):
    bn = set().union(*(bn_regimes(dt, shape, sms) for dt, shape, _, _ in bn_cases()))
    assert BN_REQUIRED <= bn, sorted(BN_REQUIRED - bn, key=str)
    ln = set().union(*(ln_regimes(dt, rows, H, sms) for dt in DTS for rows, H in ln_cases(dt)))
    assert LN_REQUIRED <= ln, sorted(LN_REQUIRED - ln, key=str)
    for dt in DTS:                                 # every LN regime in each dtype
        ln_dt = set().union(*(ln_regimes(dt, rows, H, sms) for rows, H in ln_cases(dt)))
        assert LN_REQUIRED <= ln_dt, (dt, sorted(LN_REQUIRED - ln_dt, key=str))
        bg = set().union(*(bg_regimes(dt, rows, N, sms) for rows, N in BG_CASES))
        assert BG_REQUIRED <= bg, (dt, sorted(BG_REQUIRED - bg, key=str))
    # the real ResNet-50 shapes are cap-bound where the partial-merge loop takes several passes
    stem = bn_geo(64 * 112 * 112, 64, F32, sms)
    assert stem["cap_bound"] and stem["row_blocks"] > 128


def test_geometry_mirrors_agree_with_the_documented_launches():
    # launch geometry of the benchmark shapes on a 132-SM H100 (ResNet-50 at 64 images, BERT at 2048 tokens)
    assert bn_geo(64 * 112 * 112, 64, F32, CPU_SMS)["row_blocks"] == 1056
    assert bn_geo(64 * 112 * 112, 64, BF16, CPU_SMS)["row_blocks"] == 1056
    assert bn_geo(64 * 56 * 56, 256, F32, CPU_SMS)["min_rows"] <= 0          # trailing empty stats blocks
    assert bn_geo(8 * 14 * 14, 64, F32, CPU_SMS)["row_blocks"] == 13
    assert bn_geo(2 * 6 * 6, 24, F32, CPU_SMS) is None                        # 6 vectors: txv 2 < 4
    assert ln_grid(2048, 2, CPU_SMS) == 256 and ln_grid(2113, 2, CPU_SMS) == 264
    assert bg_grid(2048, 4096, F32, CPU_SMS) == (16, 16) and bg_grid(3, 4096, BF16, CPU_SMS) == (8, 1)


def test_case_tables_reach_every_regime_at_132_sms():
    check_tables(CPU_SMS)


def test_cases_reach_every_instantiation():
    missing = required_instantiations() - instantiations()
    assert not missing, sorted(missing)


@pytest.mark.gpu
def test_case_tables_reach_every_regime_on_this_device():
    check_tables(torch.cuda.get_device_properties(0).multi_processor_count)


# ----------------------------------------------------------------------------------------------------- helpers
def _native():
    from dear_pytorch_b200 import ops
    return ops.require_native()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def ulp(v, dt):
    """ulp in dtype dt of the float64 magnitudes v (normal range)."""
    _, e = torch.frexp(v.abs().clamp_min(2.0 ** -126))
    return torch.ldexp(torch.ones_like(v), e - PBITS[dt])


def stored(e, ref, dt):
    """Bound on a value stored in dt from an fp32 value within e of ref."""
    return e + 0.5 * ulp(ref.abs() + e, dt)


def assert_within(got, ref, bound, what):
    err = (got.double() - ref).abs()
    bad = ~(err <= bound)                               # NaN fails
    if bool(bad.any()):
        i = int(bad.flatten().nonzero()[0])
        raise AssertionError("%s: %d of %d elements outside the bound; first at flat index %d: got %r ref %r bound %r"
                             % (what, int(bad.sum()), bad.numel(), i, got.flatten()[i].item(), ref.flatten()[i].item(),
                                bound.flatten()[i].item() if torch.is_tensor(bound) and bound.numel() > 1 else bound))


def bits(t):
    return t.view(torch.int32) if t.dtype == F32 else t.view(torch.int16)


def _gen(seed):
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    return g


def _randn(shape, g, scale=1.0, shift=0.0):
    return torch.randn(shape, device="cuda", generator=g) * scale + shift


# ---------------------------------------------------------------------------------------------------- BatchNorm
def _bn_ids():
    return ["%s-%s-relu%d-res%d" % (TNAME[dt], "x".join(map(str, s)), relu, res) for dt, s, relu, res in bn_cases()]


@pytest.mark.gpu
@pytest.mark.parametrize("case", bn_cases(), ids=_bn_ids())
def test_batchnorm_against_float64(case):
    dt, shape, relu, res = case
    C_ = _native()
    N, C, H, W = shape
    M = N * H * W
    g = bn_geo(M, C, dt, _sms())
    cl = torch.channels_last
    gen = _gen(zlib.crc32(repr((TNAME[dt], shape, relu, res)).encode()))
    x = _randn(shape, gen, 2.0, 0.5).to(dt).contiguous(memory_format=cl)
    z = _randn(shape, gen).to(dt).contiguous(memory_format=cl) if res else None
    w = torch.rand(C, device="cuda", generator=gen) + 0.5
    b = _randn(C, gen)
    rm0, rv0 = _randn(C, gen, 0.1), torch.rand(C, device="cuda", generator=gen) + 0.5
    rm, rv = rm0.clone(), rv0.clone()
    assert C_.bn_act_supported(x, z)
    mom, eps = 0.1, 1e-5
    m32 = float(torch.tensor(mom, dtype=F32))
    n0 = C_.bn_act_launches()

    def rows(t):                                        # [N, C, H, W] channels-last -> [M, C] view, no copy
        return t.permute(0, 2, 3, 1).reshape(M, C)

    # float64 temporaries are made per chunk of about 4M elements (32 MB), so the real ResNet shapes (51M elements)
    # need tens of MB beyond their inputs and outputs
    step = max(1, (1 << 22) // C)
    chunks = [slice(i, min(M, i + step)) for i in range(0, M, step)]
    xr = rows(x)
    zr = rows(z) if res else None

    def pre_and_ref(sl, sc64, sh64):
        pre = xr[sl].double() * sc64 + sh64             # x * scale is exact in float64
        return pre, (pre + zr[sl].double() if res else pre)

    # ---- forward (training) ----
    y, mean, invstd, scale, shift = C_.bn_act_forward(x, z, w, b, rm, rv, True, mom, eps, relu)
    assert C_.bn_act_launches() == n0 + 3
    yr = rows(y)
    mu64 = sum(xr[sl].double().sum(0) for sl in chunks) / M
    var64 = sum(((xr[sl].double() - mu64) ** 2).sum(0) for sl in chunks) / M
    xmax = torch.stack([xr[sl].double().abs().amax(0) for sl in chunks]).amax(0)
    # Welford over n_t rows per thread, then Chan merges: ty in the block, ceil(rb/32) per lane, 5 shuffle levels.
    # Each update/merge rounds the mean by ~3U of |x| and |mean| (4U taken) and M2 by ~4U relative (8U taken) times the
    # conditioning 1 + mean^2/var of the updating algorithm.
    steps = -(-g["rpb"] // g["ty"]) + g["ty"] + -(-g["row_blocks"] // 32) + 5
    e_mean = 4 * U * steps * xmax
    var_rel = 8 * U * steps * (1 + mu64 ** 2 / var64)
    assert_within(mean, mu64, e_mean, "save_mean")
    # invstd = rsqrtf(fl(fl(m2 / n) + eps)): var_rel / 2, plus 2 ulp (4U) for rsqrtf and U for each rounding
    ist64 = (var64 + eps).rsqrt()
    assert_within(invstd, ist64, ist64 * (0.5 * var_rel * var64 / (var64 + eps) + 6 * U), "save_invstd")
    rm64 = (1 - m32) * rm0.double() + m32 * mu64
    assert_within(rm, rm64, m32 * e_mean + 4 * U * ((1 - m32) * rm0.double().abs() + m32 * mu64.abs()), "running_mean")
    unb64 = var64 * M / (M - 1)
    assert_within(rv, (1 - m32) * rv0.double() + m32 * unb64,
                  m32 * unb64 * (var_rel + 3 * U) + 4 * U * ((1 - m32) * rv0.double() + m32 * unb64), "running_var")
    # y = T(act(fmaf(x, scale, shift) [+ z])) from the kernel's own scale / shift: one fp32 rounding of the fma, then
    # the add and the store together stay within one ulp of T.  The backward's ReLU mask is y > 0 with a residual, else
    # the sign of fmaf(x, scale, shift), which is the sign of the float64 pre-activation.
    sc64, sh64 = scale.double(), shift.double()
    mask = torch.ones((M, C), dtype=torch.bool, device="cuda")
    for sl in chunks:
        pre, ref = pre_and_ref(sl, sc64, sh64)
        e = U * pre.abs()
        bnd = e + ulp(ref.abs() + e, dt)
        y64 = yr[sl].double()
        assert_within(y64, ref.clamp_min(0) if relu else ref, bnd, "y")
        if relu:
            assert bool((y64[ref < -bnd] == 0).all()), "ReLU left a clearly negative pre-activation nonzero"
            mask[sl] = (y64 > 0) if res else (pre > 0)
        del pre, ref, e, bnd, y64

    # ---- backward: random dy against the float64 BN backward from the kernel's own statistics and mask ----
    dy = _randn(shape, gen).to(dt).contiguous(memory_format=cl)
    dx, dz, dgamma, dbeta = C_.bn_act_backward(dy, x, y if (res and relu) else None, mean, invstd, scale, shift, relu, res)
    assert C_.bn_act_launches() == n0 + 6
    dyr, dxr = rows(dy), rows(dx)
    if res:                                             # dz is the masked dy, bit for bit
        assert torch.equal(bits(dz), bits(torch.where(mask.view(N, H, W, C).permute(0, 3, 1, 2), dy,
                                                      torch.zeros((), dtype=dt, device="cuda"))))
    mu_k, is_k = mean.double(), invstd.double()

    def g_xh(sl):
        g64 = torch.where(mask[sl], dyr[sl].double(), torch.zeros((), dtype=torch.float64, device="cuda"))
        return g64, (xr[sl].double() - mu_k) * is_k

    s1 = s2 = a1 = a2 = 0
    for sl in chunks:
        g64, xh64 = g_xh(sl)
        s1, s2 = s1 + g64.sum(0), s2 + (g64 * xh64).sum(0)
        a1, a2 = a1 + g64.abs().sum(0), a2 + (g64 * xh64).abs().sum(0)
        del g64, xh64
    # partial sums: n_b rows per thread (grid-stride), ty in shared memory, 4 per lane per pass, 5 shuffle levels
    depth = -(-M // (g["row_blocks"] * g["ty"])) + g["ty"] + 4 * -(-g["row_blocks"] // 128) + 5
    e_s1 = depth * U * a1
    e_s2 = (depth + 3) * U * a2                         # + fl(x - mean), * invstd, in the fma
    assert_within(dbeta, s1, e_s1, "dbeta")
    assert_within(dgamma, s2, e_s2, "dgamma")
    c1, c2 = s1 / M, s2 / M
    e_c1, e_c2 = e_s1 / M + 2 * U * c1.abs(), e_s2 / M + 2 * U * c2.abs()
    for sl in chunks:
        g64, xh64 = g_xh(sl)
        dx64 = sc64 * (g64 - c1 - xh64 * c2)
        e = sc64.abs() * (e_c1 + xh64.abs() * e_c2 + 5 * U * (g64.abs() + c1.abs() + (xh64 * c2).abs()))
        assert_within(dxr[sl], dx64, stored(e, dx64, dt), "dx")
        del g64, xh64, dx64, e
    del dx, dz, dxr

    # ---- backward with dy == 1: dbeta is an integer count, exact in fp32 below 2^24 (every partial merged once) ----
    ones = torch.ones_like(dy)
    _, dz1, _, dbeta1 = C_.bn_act_backward(ones, x, y if (res and relu) else None, mean, invstd, scale, shift, relu, res)
    assert C_.bn_act_launches() == n0 + 9
    assert torch.equal(dbeta1, mask.sum(0).float()), "dbeta with dy = 1 is not the exact count of unmasked rows"
    if res:
        assert torch.equal(bits(dz1), bits(torch.where(mask.view(N, H, W, C).permute(0, 3, 1, 2), ones,
                                                       torch.zeros((), dtype=dt, device="cuda"))))
    del mask, dz1, ones

    # ---- inference: bn_fold_kernel's scale / shift from the running statistics, then the same apply check ----
    ye, _, _, sce, she = C_.bn_act_forward(x, z, w, b, rm, rv, False, mom, eps, relu)
    assert C_.bn_act_launches() == n0 + 11
    ist = (rv.double() + eps).rsqrt()
    sc_ref = w.double() * ist
    e_sc = 7 * U * sc_ref.abs()                          # rsqrtf 2 ulp, + eps, * gamma
    assert_within(sce, sc_ref, e_sc, "eval scale")
    sh_ref = b.double() - rm.double() * sc_ref
    assert_within(she, sh_ref, rm.double().abs() * e_sc + 2 * U * (b.double().abs() + (rm.double() * sc_ref).abs()),
                  "eval shift")
    yer = rows(ye)
    for sl in chunks:
        pre, ref = pre_and_ref(sl, sce.double(), she.double())
        e = U * pre.abs()
        assert_within(yer[sl], ref.clamp_min(0) if relu else ref, e + ulp(ref.abs() + e, dt), "eval y")
        del pre, ref, e


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTS, ids=TNAME.get)
def test_batchnorm_one_value_per_channel_raises_like_pytorch(dt):
    C_ = _native()
    x = torch.randn(1, 64, 1, 1, device="cuda").to(dt).contiguous(memory_format=torch.channels_last)
    m = _fused_bn_module(64)
    with pytest.raises(ValueError, match="more than 1 value per channel"):
        nn.BatchNorm2d(64).cuda()(x.float())
    with pytest.raises(ValueError, match="more than 1 value per channel"):
        m(x)
    with pytest.raises(RuntimeError, match="more than 1 value per channel"):
        C_.bn_act_forward(x, None, m.weight, m.bias, m.running_mean, m.running_var, True, 0.1, 1e-5, True)
    assert torch.equal(m.running_var, torch.ones(64, device="cuda"))      # nothing was updated
    # inference with one value per channel is well defined, and fused
    m.eval()
    n0 = C_.bn_act_launches()
    with torch.no_grad():
        got = m(x)
    assert C_.bn_act_launches() == n0 + 2
    ref = F.relu(F.batch_norm(x.float(), m.running_mean, m.running_var, m.weight, m.bias, False, 0.1, 1e-5))
    torch.testing.assert_close(got.float(), ref.to(dt).float(), rtol=0, atol=float(ulp(ref.double().abs().max(), dt)))


def _fused_bn_module(c):
    from dear_pytorch_b200.ops.fused_bn import FusedBatchNormAct2d
    return FusedBatchNormAct2d(c).cuda()


# ---------------------------------------------------------------------------------------------------- LayerNorm
def _ln_params():
    return [(dt, rows, H) for dt in DTS for rows, H in ln_cases(dt)]


@pytest.mark.gpu
@pytest.mark.parametrize("dt,rows,H", _ln_params(), ids=["%s-%s-%d" % (TNAME[d], r, h) for d, r, h in _ln_params()])
def test_layernorm_against_float64(dt, rows, H):
    C_ = _native()
    sms = _sms()
    R = ln_rows(rows, sms)
    n_lane = -(-H // (32 * VEC[dt])) * VEC[dt]          # elements one lane sums sequentially
    nblocks = ln_grid(R, 1, sms)                        # backward CTAs = partial rows of colsum_finalize
    col_depth = -(-R // (nblocks * 8)) + 8 + -(-nblocks // 16) + 16
    eps = 1e-5
    for vi, (p, with_bias) in enumerate(LN_VARIANTS):
        # fresh inputs for every call: rows a kernel failed to write would hold some other call's values, never these
        gen = _gen(7000 + 97 * vi + R * 3 + H + (1 if dt == BF16 else 0))
        a = _randn((R, H), gen).to(dt)
        r = _randn((R, H), gen).to(dt)
        w = (1.0 + 0.1 * _randn(H, gen)).to(dt)
        b = (0.1 * _randn(H, gen)).to(dt)
        bb = _randn(H, gen).to(dt) if with_bias else None
        assert C_.ln_supported(a, r, w, b, bb)
        n0 = C_.ln_launches()
        torch.manual_seed(11 + vi)
        y, s, mean, rstd, mask = C_.ln_forward(a, r, w, b, p, True, eps, bb)
        assert C_.ln_launches() == n0 + 1
        a_eff = (a.float() + bb.float()).to(dt) if with_bias else a          # the kernel rounds a + bias to T
        # ---- s ----
        if p == 0:
            assert mask.numel() == 0
            assert torch.equal(bits(s), bits((a_eff.float() + r.float()).to(dt))), "s is not T(a + r)"
        else:
            keep = mask.bool()
            assert bool(((mask == 0) | (mask == 1)).all())
            sc32 = torch.tensor(1.0, dtype=F32) / (torch.tensor(1.0, dtype=F32) - torch.tensor(p, dtype=F32))
            sc = float(sc32)
            # a * scale is exact in float64; the one float64 rounding of the sum can differ from the fma's single
            # rounding only where it lands exactly on an fp32 midpoint
            two = torch.where(keep, a_eff.float() * sc32.item() + r.float(), r.float() + 0.0).to(dt)
            fma = torch.where(keep, (a_eff.double() * sc + r.double()).float(), r.float() + 0.0).to(dt)
            ok = (bits(s) == bits(two)) | (bits(s) == bits(fma))
            assert bool(ok.all()), "s differs from both roundings of a * scale + r at %d elements" % int((~ok).sum())
        # ---- mean / rstd from the stored s ----
        s64 = s.double()
        mu64 = s64.mean(1)
        assert_within(mean, mu64, (n_lane + 7) * U * s64.abs().mean(1), "mean")
        var_k = ((s64 - mean.double()[:, None]) ** 2).mean(1)             # around the kernel's mean, as it sums
        rs64 = (var_k + eps).rsqrt()
        assert_within(rstd, rs64, rs64 * ((n_lane + 11) * U / 2 + 4 * U), "rstd")
        # ---- y from the kernel's own s, mean and rstd ----
        xh = (s64 - mean.double()[:, None]) * rstd.double()[:, None]
        y64 = xh * w.double() + b.double()
        assert_within(y, y64, stored(4 * U * ((xh * w.double()).abs() + b.double().abs()), y64, dt), "y")
        del y64
        # ---- backward ----
        dy = _randn((R, H), gen).to(dt)
        d_res, d_a, dgamma, dbeta, dbias = C_.ln_backward(dy, s, mean, rstd, w, mask, p, with_bias)
        assert C_.ln_launches() == n0 + 3
        dy64, gm = dy.double(), w.double()
        gy = dy64 * gm
        c1, c2 = gy.mean(1, keepdim=True), (gy * xh).mean(1, keepdim=True)
        e_c1 = (n_lane + 7) * U * gy.abs().mean(1, keepdim=True)
        e_c2 = (n_lane + 9) * U * (gy * xh).abs().mean(1, keepdim=True)
        rs = rstd.double()[:, None]
        ds64 = rs * (gy - c1 - xh * c2)
        e_ds = rs * (e_c1 + xh.abs() * e_c2 + 5 * U * (gy.abs() + c1.abs() + (xh * c2).abs()))
        assert_within(d_res, ds64, stored(e_ds, ds64, dt), "d_residual")
        del ds64, e_ds, gy
        if p > 0:
            want = torch.where(keep, d_res.float() * sc, torch.zeros((), device="cuda"))
            if dt == F32:                               # d_a = fl32(d_res * scale) where kept, bit for bit
                assert torch.equal(bits(d_a), bits(want)), "d_a is not fl32(d_residual * scale) under the mask"
            else:                                       # scaled before d_res was rounded to T: half an ulp of
                assert bool((d_a[~keep] == 0).all())    # d_res times scale, the product, then the store
                w64 = want.double()
                e = 0.5 * sc * ulp(d_res.double(), dt) * keep + U * w64.abs()
                assert_within(d_a, w64, stored(e, w64, dt), "d_a")
        else:
            assert d_a.data_ptr() == d_res.data_ptr()
        # ---- column sums: warp loop, 8 warps, colsum_finalize's per-thread loop and 16-row chain ----
        prod = dy64 * xh
        assert_within(dgamma, prod.sum(0), stored((col_depth + 3) * U * prod.abs().sum(0), prod.sum(0), dt), "dgamma")
        assert_within(dbeta, dy64.sum(0), stored(col_depth * U * dy64.abs().sum(0), dy64.sum(0), dt), "dbeta")
        if with_bias:
            # the kernel sums d_a before it is rounded to T: half an ulp of T per row on top of the fp32 sum
            da64 = d_a.double()
            e = col_depth * U * da64.abs().sum(0)
            if dt == BF16:
                e = e + (0.5 * ulp(da64, dt) * (da64 != 0)).sum(0)
            assert_within(dbias, da64.sum(0), stored(e, da64.sum(0), dt), "dbias")
        else:
            assert dbias.numel() == 0
        del prod, xh, s64, dy64
        # ---- dy == 1: dbeta is the row count, exact in fp32, then rounded to T once ----
        d1 = C_.ln_backward(torch.ones_like(dy), s, mean, rstd, w, mask, p, False)
        assert torch.equal(bits(d1[3]), bits(torch.full((H,), float(R), device="cuda").to(dt))), "dbeta != rows"
        assert C_.ln_launches() == n0 + 5


@pytest.mark.gpu
@pytest.mark.parametrize("with_bias", [False, True])
def test_dropout_mask_is_keyed_by_element_index(with_bias):
    """fp32 (4 lanes per vector) and bf16 (8 lanes per vector) draw the same mask from the same generator state."""
    C_ = _native()
    R, H = 2 * _sms() * 8 + 1, 1016
    gen = _gen(31 + with_bias)
    a, r = _randn((R, H), gen), _randn((R, H), gen)
    w, b = torch.ones(H, device="cuda"), torch.zeros(H, device="cuda")
    bb = _randn(H, gen) if with_bias else None
    masks = {}
    for p in (0.1, 0.5):
        for dt in DTS:
            torch.manual_seed(1234)
            masks[p, dt] = C_.ln_forward(a.to(dt), r.to(dt), w.to(dt), b.to(dt), p, True, 1e-5,
                                         None if bb is None else bb.to(dt))[4]
        assert torch.equal(masks[p, F32], masks[p, BF16]), "fp32 and bf16 masks differ for p = %g" % p
        # keep ~ Binomial(n, 1 - p): 6 standard deviations (false alarm ~2e-9)
        n = masks[p, F32].numel()
        frac = masks[p, F32].double().mean().item()
        assert abs(frac - (1 - p)) <= 6 * math.sqrt(p * (1 - p) / n), (p, frac)
    for dt in DTS:
        assert C_.ln_forward(a.to(dt), r.to(dt), w.to(dt), b.to(dt), 0.5, False, 1e-5)[4].numel() == 0   # eval
        assert C_.ln_forward(a.to(dt), r.to(dt), w.to(dt), b.to(dt), 0.0, True, 1e-5)[4].numel() == 0    # p = 0


# ---------------------------------------------------------------------------------------------------- bias-GELU
def _bg_params():
    return [(dt, rows, N) for dt in DTS for rows, N in BG_CASES]


@pytest.mark.gpu
@pytest.mark.parametrize("dt,rows,N", _bg_params(), ids=["%s-%d-%d" % (TNAME[d], r, n) for d, r, n in _bg_params()])
def test_bias_gelu_against_float64(dt, rows, N):
    C_ = _native()
    _, gy = bg_grid(rows, N, dt, _sms())
    gen = _gen(500 + rows + N + (1 if dt == BF16 else 0))
    z = _randn((rows, N), gen, 2.0).to(dt)
    bias = _randn(N, gen).to(dt)
    dh = _randn((rows, N), gen).to(dt)
    assert C_.bias_gelu_supported(z, bias)
    n0 = C_.ln_launches()
    h = C_.bias_gelu_forward(z, bias)
    dz, dbias = C_.bias_gelu_backward(dh, z, bias)
    assert C_.ln_launches() == n0 + 3
    t = (z.float() + bias.float()).to(dt).double()       # the kernel rounds z + b to T
    at = t.abs()
    erf = torch.special.erf(t / math.sqrt(2.0))
    h64 = 0.5 * t * (1 + erf)
    # fl(t * fl(1/sqrt2)): 2U|t|/sqrt2 in the argument, times erf' <= 2/sqrt(pi): 1.6U|t|; erff 2 ulp: 4U; 1 + erf: 2U;
    # the product: U|h|
    e_erf = 1.6 * U * at + 6 * U
    e_h = 0.5 * at * e_erf + U * h64.abs()
    assert_within(h, h64, stored(e_h, h64, dt), "h")
    # gelu'(t) = (1 + erf) / 2 + t phi(t);  q = -t^2/2 rounded (U|q|), __expf: 2 + floor(1.173|q|) ulp, then three
    # roundings for t * fl(1/sqrt(2 pi)) * exp and U for the final sum
    q = 0.5 * t * t
    tphi = t * torch.exp(-q) / math.sqrt(2 * math.pi)
    d64 = 0.5 * (1 + erf) + tphi
    e_exp = U * q + 2 * U * (2 + torch.floor(1.173 * q))
    e_d = 0.5 * e_erf + tphi.abs() * (e_exp + 3 * U) + U * d64.abs()
    dh64 = dh.double()
    dz64 = dh64 * d64
    assert_within(dz, dz64, stored(dh64.abs() * e_d + U * dz64.abs(), dz64, dt), "dz")
    # dbias sums exactly the stored dz: per-thread rows, the 4 row groups, colsum_finalize's loop and 16-row chain
    depth = -(-rows // (4 * gy)) + 3 + -(-gy // 16) + 15
    own = dz.double()
    ref = own.sum(0)
    assert_within(dbias, ref, stored(depth * U * own.abs().sum(0), ref, dt), "dbias")


# ----------------------------------------------------------------------------------------------------- alignment
def _misaligned(shape, dt, channels_last=False):
    """A contiguous (or channels-last) view one element past a 16-byte boundary.  Only its pointer is used: nothing
    reads or writes through it, so no kernel runs on misaligned memory."""
    n = math.prod(shape)
    base = torch.empty(n + 8, device="cuda", dtype=dt)
    if channels_last:
        N, C, H, W = shape
        t = base[1:1 + n].view(N, H, W, C).permute(0, 3, 1, 2)
        assert t.is_contiguous(memory_format=torch.channels_last)
    else:
        t = base[1:1 + n].view(shape)
        assert t.is_contiguous()
    assert t.data_ptr() % 16
    return t


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTS, ids=TNAME.get)
def test_misaligned_operands_are_not_supported(dt):
    """Every operand the kernels move as 128-bit vectors must be 16-byte aligned; a contiguous view at an odd storage
    offset makes the predicates (and so the wrappers' choice of path) reject the fused kernels."""
    from dear_pytorch_b200.ops.fused_ln import fused_ln_applicable
    C_ = _native()
    cl = torch.channels_last
    shape = (2, 64, 5, 5)
    x = torch.empty(shape, device="cuda", dtype=dt).contiguous(memory_format=cl)
    assert C_.bn_act_supported(x) and C_.bn_act_supported(x, torch.empty_like(x))
    assert not C_.bn_act_supported(_misaligned(shape, dt, True))
    assert not C_.bn_act_supported(x, _misaligned(shape, dt, True))
    R, H = 33, 64
    ok = [torch.empty(R, H, device="cuda", dtype=dt), torch.empty(R, H, device="cuda", dtype=dt)] + \
         [torch.empty(H, device="cuda", dtype=dt) for _ in range(3)]          # a, residual, weight, bias, branch bias
    assert C_.ln_supported(*ok) and fused_ln_applicable(*ok)
    for k in range(5):
        args = list(ok)
        args[k] = _misaligned(tuple(ok[k].shape), dt)
        assert not C_.ln_supported(*args), k
        assert not fused_ln_applicable(*args), k
    z, b = torch.empty(R, 72, device="cuda", dtype=dt), torch.empty(72, device="cuda", dtype=dt)
    assert C_.bias_gelu_supported(z, b)
    assert not C_.bias_gelu_supported(_misaligned((R, 72), dt), b)
    assert not C_.bias_gelu_supported(z, _misaligned((72,), dt))


def _misaligned_copy(src):
    """The values of ``src`` in a view one element past a 16-byte boundary, in the same memory format, filled by a flat
    same-dtype copy.  None of the fused kernels may read it."""
    n = src.numel()
    base = torch.empty(n + 8, device="cuda", dtype=src.dtype)
    if src.dim() == 4:                                  # channels-last: [N, H, W, C] in memory
        N, C, H, W = src.shape
        base[1:1 + n].copy_(src.permute(0, 2, 3, 1).reshape(-1))
        t = base[1:1 + n].view(N, H, W, C).permute(0, 3, 1, 2)
        assert t.is_contiguous(memory_format=torch.channels_last)
    else:
        base[1:1 + n].copy_(src.reshape(-1))
        t = base[1:1 + n].view(src.shape)
    assert t.data_ptr() % 16
    return t


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTS, ids=TNAME.get)
def test_misaligned_views_take_the_composite(dt):
    """Each public wrapper, given a misaligned view of real data, launches none of the fused kernels and returns what
    the composite returns on aligned copies of the same values."""
    from dear_pytorch_b200.ops.bias_gelu import bias_gelu
    from dear_pytorch_b200.ops.fused_bn import bn_act
    from dear_pytorch_b200.ops.fused_ln import dropout_add_layer_norm
    C_ = _native()
    tol = dict(rtol=1e-5, atol=1e-5) if dt == F32 else {}
    # BatchNorm + residual + ReLU: x, then the residual
    shape = (4, 64, 6, 5)
    x = torch.randn(shape, device="cuda").to(dt).contiguous(memory_format=torch.channels_last)
    z = torch.randn(shape, device="cuda").to(dt).contiguous(memory_format=torch.channels_last)
    w, b = torch.rand(64, device="cuda") + 0.5, torch.randn(64, device="cuda")
    for xi, zi in ((_misaligned_copy(x), z), (x, _misaligned_copy(z))):
        assert not C_.bn_act_supported(xi, zi)
        rm, rv = torch.zeros(64, device="cuda"), torch.ones(64, device="cuda")
        n0 = C_.bn_act_launches()
        got = bn_act(xi, w, b, rm, rv, True, 0.1, 1e-5, relu=True, residual=zi)
        assert C_.bn_act_launches() == n0
        rm2, rv2 = torch.zeros(64, device="cuda"), torch.ones(64, device="cuda")
        torch.testing.assert_close(got, F.relu(F.batch_norm(x, rm2, rv2, w, b, True, 0.1, 1e-5) + z), **tol)
        torch.testing.assert_close((rm, rv), (rm2, rv2), **tol)
    # dropout + add + LayerNorm: the branch a, the residual, the branch bias
    R, H = 33, 64
    a, r, bb = (torch.randn(R, H, device="cuda").to(dt), torch.randn(R, H, device="cuda").to(dt),
                torch.randn(H, device="cuda").to(dt))
    lw, lb = (1 + 0.1 * torch.randn(H, device="cuda")).to(dt), (0.1 * torch.randn(H, device="cuda")).to(dt)
    for ai, ri, bbi in ((_misaligned_copy(a), r, None), (a, _misaligned_copy(r), bb), (a, r, _misaligned_copy(bb))):
        n0 = C_.ln_launches()
        got = dropout_add_layer_norm(ai, ri, lw, lb, 0.0, False, 1e-5, branch_bias=bbi)
        assert C_.ln_launches() == n0
        ref = F.layer_norm(r + (a if bbi is None else a + bb), (H,), lw, lb, 1e-5)
        torch.testing.assert_close(got, ref, **tol)
    # bias + GELU: z, then the bias
    zg, bg = torch.randn(R, 72, device="cuda").to(dt), torch.randn(72, device="cuda").to(dt)
    for zi, bi in ((_misaligned_copy(zg), bg), (zg, _misaligned_copy(bg))):
        n0 = C_.ln_launches()
        got = bias_gelu(zi, bi)
        assert C_.ln_launches() == n0
        torch.testing.assert_close(got, F.gelu(zg + bg), **tol)
