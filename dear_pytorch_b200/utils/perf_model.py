"""Analytical performance models.

(1) The reference's alpha-beta tables and cost models (``*/utils.py:62-158``,
    ``dear/hv_distributed_optimizer.py:44-61``), kept as data for the MG-WFBP baselines.
(2) The roofline used to judge the fused kernels: time >= max(HBM bytes / HBM bandwidth, NVLink bytes /
    per-direction link bandwidth).
"""
from __future__ import annotations

import json
import os

import numpy as np

# ---- (1) reference network models --------------------------------------------------------------
# all-reduce alpha (s) / beta (s per byte) measured by the reference's authors
GbE_multi_p_ab_small = {2: (1.6e-3, 1.0e-8), 4: (2.7e-3, 1.3e-8), 8: (4.0e-3, 1.5e-8), 16: (1.1e-2, 1.7e-8)}
GbE_multi_p_ab_large = {2: (4.4e-3, 5.8e-9), 4: (5.6e-3, 7.4e-9), 8: (7.68e-3, 8.2e-9), 16: (2.1e-2, 1.7e-8)}
tenGbE_multi_p_ab = {2: (1.5e-5, 5.7e-11), 4: (3.6e-5, 1.1e-10), 8: (8.5e-5, 1.4e-10), 16: (1.4e-4, 2.1e-10)}
# tables used by the MG-WFBP optimizer (dear/hv_distributed_optimizer.py:44-61)
ALPHA_BETA_56GbIB = {64: (0.00080632079996292579, 5.8899804e-10), 32: (0.00040632079996292579, 4.9e-10),
                     16: (0.00023583677659915685, 4.4571353e-10), 8: (9.75367204301171e-05, 3.0568387e-10),
                     4: (4.204298980348825e-05, 2.0589653e-10), 2: (2.554691138304671e-06, 9.837389e-11)}
ALPHA_BETA_10GbE = {64: (0.0070436, 9.6432e-10), 32: (0.0023476, 8.218e-10), 16: (0.0009080981007148093, 7.395651e-10),
                    8: (0.0005230272768511732, 8.570746e-10), 4: (4.204298980348825e-05, 2.0589653e-10),
                    2: (2.554691138304671e-06, 9.837389e-11)}

TOPK_S = 2.18896957e-10      # P102-100 top-k cost constant (dear/utils.py:62)


def topk_perf_model(x, s=TOPK_S):
    """t = s * x * log2(x) for selecting top-k out of x parameters."""
    return 0.0 if x == 0 else s * x * np.log2(x)


def allgather_perf_model(x, P, density=0.001, eth="GbE"):
    if x == 0:
        return 0.0
    size = x * P * 4 * density
    a, b = (GbE_multi_p_ab_large if size >= 1024 * 1024 else GbE_multi_p_ab_small)[P]
    return (a + b * size) * 2


def predict_density_with_size_and_computation(m, comp_time, P):
    return 0.001


def predict_allreduce_time_with_size(alpha, beta, size, P=None):
    return 0.0 if size == 0 else alpha + beta * size


def gen_threshold_from_normal_distribution(p_value, mu, sigma):
    from scipy import stats
    z = stats.norm.ppf((1 - p_value) / 2)
    return mu + z * sigma, mu - z * sigma


def check_unique(items):
    seen = set()
    for k in items:
        if k in seen:
            return False
        seen.add(k)
    return True


# ---- (2) roofline -------------------------------------------------------------------------------
def measured_peaks(path: str = None) -> dict:
    """HBM / NVLink denominators: MEASURED_PEAKS.json if present, else the H100 SXM data-sheet figures (never reached
    in practice: a bound computed from them is a lower bound on time)."""
    root = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    path = path or os.path.join(root, "MEASURED_PEAKS.json")
    peaks = {"hbm_gbs": 3350.0, "bf16_tflops": 989.0, "source": "H100 SXM data sheet"}
    try:
        with open(path) as f:
            d = json.load(f)
        peaks.update(hbm_gbs=float(d["hbm_gbs"]), bf16_tflops=float(d["bf16_tflops"]), source="measured")
    except Exception:
        pass
    peaks["nvlink_gbs_per_dir"] = 450.0      # H100 SXM NVLink 4: 900 GB/s in both directions together (data sheet)
    return peaks


def rs_roofline_us(bucket_bytes: int, world: int, elem_bytes: int = 4, peaks: dict = None,
                   src_elem_bytes: int = None) -> dict:
    """Kernel A lower bound for one bucket on one GPU.

    HBM: pack reads the local gradients and writes the local bucket, the local shard is read, the fp32 shard is written;
    NVLink: (P-1)/P of the bucket is pulled from peers (per direction).  ``bucket_bytes`` / ``elem_bytes`` describe the
    bucket as it travels; ``src_elem_bytes`` (default ``elem_bytes``) is the gradient element the pack reads — 4 for
    fp32 gradients sent at 16 bits (grad_comm_dtype).
    """
    pk = peaks or measured_peaks()
    shard = bucket_bytes / world
    src_bytes = bucket_bytes / elem_bytes * (src_elem_bytes or elem_bytes)
    if world == 1 and elem_bytes == 4:
        hbm = 2 * bucket_bytes          # single GPU: the pack writes the fp32 shard directly
    else:
        hbm = src_bytes + bucket_bytes + shard + (shard / elem_bytes) * 4
    link = bucket_bytes * (world - 1) / world
    t_hbm = hbm / (pk["hbm_gbs"] * 1e3)
    t_link = link / (pk["nvlink_gbs_per_dir"] * 1e3)
    return {"hbm_us": t_hbm, "nvlink_us": t_link, "bound_us": max(t_hbm, t_link), "hbm_bytes": hbm, "link_bytes": link}


def ag_roofline_us(bucket_bytes: int, world: int, elem_bytes: int = 4, momentum: bool = True, peaks: dict = None) -> dict:
    """Kernel B lower bound: shard-sized reads of grad/momentum/param + momentum write locally,
    (P-1)/P of the bucket pushed over NVLink, and P shards landing in local HBM."""
    pk = peaks or measured_peaks()
    shard_elems = bucket_bytes / elem_bytes / world
    hbm = shard_elems * 4 * (2 + (2 if momentum else 0)) + bucket_bytes
    link = bucket_bytes * (world - 1) / world
    t_hbm = hbm / (pk["hbm_gbs"] * 1e3)
    t_link = link / (pk["nvlink_gbs_per_dir"] * 1e3)
    return {"hbm_us": t_hbm, "nvlink_us": t_link, "bound_us": max(t_hbm, t_link)}


# ---- (3) alpha-beta model of the fused kernels, fitted to the measured sweep -----------------------
def fit_alpha_beta(rows, key: str):
    """Least-squares ``time = alpha + beta * bytes`` over a ``tools/kernel_bench.py`` sweep (alpha in s, beta in s/byte)."""
    xs = [r["bucket_mb"] * 2 ** 20 for r in rows if key in r]
    ys = [r[key] * 1e-6 for r in rows if key in r]
    n = len(xs)
    if n < 2:
        raise ValueError("need at least two bucket sizes to fit alpha and beta")
    mx, my = sum(xs) / n, sum(ys) / n
    beta = sum((x - mx) * (y - my) for x, y in zip(xs, ys)) / sum((x - mx) ** 2 for x in xs)
    return max(my - beta * mx, 0.0), beta


def fused_kernel_model(path: str) -> dict:
    """alpha-beta of Kernel A / Kernel B and of NCCL's reduce-scatter / all-gather on one machine, from a sweep written by
    ``tools/kernel_bench.py`` — the counterpart of the reference's hard-coded per-cluster tables
    (``dear/utils.py:62-104``), which MG-WFBP style planners (baselines/wfbp.py: mgwfbp_groups) consume."""
    with open(path) as f:
        rows = json.load(f)["rows"]
    out = {"world": rows[0].get("world"), "source": os.path.basename(path)}
    for name, key in (("reduce_scatter", "rs_us"), ("reduce_scatter_in_place", "rs_nopack_us"), ("allgather_update", "ag_sgd_us"),
                      ("nccl_reduce_scatter", "nccl_rs_us"), ("nccl_all_gather", "nccl_ag_us"),
                      ("nccl_copy_reduce_scatter_div", "nccl_copy_rs_div_us")):
        try:
            out[name] = fit_alpha_beta(rows, key)
        except (ValueError, ZeroDivisionError):
            pass
    return out
