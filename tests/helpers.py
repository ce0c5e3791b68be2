"""Shared helpers for the parity tests: synthetic binned data + tree comparison with the near-tie rule
of SURVEY.md §8d (if two candidate splits are closer than the stated tolerance either choice is valid and
the comparison stops at the divergence point)."""
from __future__ import annotations

import math

import numpy as np


def synth_identity(n, f, seed, informative=8, num_bin=255):
    """bins drawn uniformly; stored value == bin (SURVEY.md §8c(ii)); L2 gradients at score 0."""
    rng = np.random.default_rng(seed)
    bins = rng.integers(0, num_bin, (n, f), dtype=np.uint8)
    k = min(informative, f)
    w = rng.normal(size=k)
    y = ((bins[:, :k] / (num_bin / 2.0) - 1) @ w + 0.5 * rng.normal(size=n)).astype(np.float32)
    grad = (0.0 - y).astype(np.float32)
    hess = np.ones(n, np.float32)
    return bins, y, grad, hess


def logistic_grad(y01, score=0.0):
    p = 1.0 / (1.0 + np.exp(-score))
    g = (p - y01).astype(np.float32)
    h = np.full(len(y01), p * (1 - p), np.float32) if np.isscalar(p) else (p * (1 - p)).astype(np.float32)
    return g, h


MARGIN_TOL = 1e-5      # stated tolerance of the split-sequence comparison (DESIGN.md §2)
DIVERGENCES = []       # (test-visible) log of accepted near-tie divergences: (split index, relative margin)
STRICT_TOL = 1e-12     # exact-input tier: margin and field tolerance of compare_trees(strict=True) (DESIGN.md §2)
ESCAPES = []           # log of strict-mode divergences: (split index, relative margin); the exact-input tests want none


def _gain_scale(b):
    """Magnitude of the terms a split gain is the difference of: sum_g^2 / sum_h of both children.  A gain much smaller
    than its terms carries their fp64 rounding, so the strict tier measures gain errors against this scale."""
    s = abs(float(b["gain"]))
    for side in ("left", "right"):
        sh = float(b[side + "_sum_hessian"])
        if sh > 0:
            s += float(b[side + "_sum_gradient"]) ** 2 / sh
    return s


def compare_trees(gpu, orc, rtol=1e-5, min_prefix=None, strict=False):
    """gpu: lightgbm_b200.Tree, orc: oracle_py.OracleTree.  Returns (#splits that matched exactly, diverged?).

    Every split must match the oracle's: structural fields exactly, float fields within rtol*10.  The ONLY tolerated
    divergence is the margin rule of SURVEY.md §8d: at the first differing split the ORACLE's own best-vs-runner-up
    margin (gain - second_gain, recorded by oracle/lgbm_oracle.c for every split) must be below MARGIN_TOL relative,
    i.e. the reference's choice was itself a numerical coin flip; the comparison then stops (the trees legitimately
    differ from there on) and the divergence is logged in DIVERGENCES.  A mismatch at a split whose margin is larger
    fails the test.

    strict=True is the exact-input tier (inputs whose fixed point and fp64 sums are exact, so the GPU and the oracle
    add the same numbers): a structural mismatch is accepted only where the oracle's margin is <= STRICT_TOL relative
    (then only the fp64 order of the kEpsilon additions and FMA contraction can differ) and is logged in ESCAPES;
    gains (against the scale of their terms), sums and leaf values must agree within STRICT_TOL.  An exact tie has
    margin 0, so tests of this tier assert that the comparison did not diverge at all."""
    tol = STRICT_TOL if strict else rtol * 10
    ns = min(gpu.num_leaves, orc.num_leaves) - 1
    matched = 0
    for i in range(ns):
        a, b = gpu.splits[i], orc.splits[i]
        same = (a["leaf"] == b["leaf"] and a["feature"] == b["feature"] and a["threshold"] == b["threshold"]
                and a["default_left"] == b["default_left"])
        if not same:
            names = b.dtype.names or ()
            second = float(b["second_gain"]) if "second_gain" in names else float("-inf")
            margin = (float(b["gain"]) - second) / max(abs(float(b["gain"])), 1e-300)
            if strict:
                assert margin <= STRICT_TOL, (f"split {i}: structural mismatch where the oracle's margin is {margin:.3e} "
                                              f"(> {STRICT_TOL}): gpu={a} oracle={b}")
                ESCAPES.append((i, margin))
                print(f"[compare_trees] strict: divergence at split {i}/{ns}, oracle margin {margin:.3e}")
                return matched, True
            assert margin < MARGIN_TOL, (f"split {i}: structural mismatch where the oracle's margin is {margin:.3e} "
                                         f"(>= {MARGIN_TOL}): gpu={a} oracle={b}")
            rel = abs(a["gain"] - b["gain"]) / max(abs(b["gain"]), 1e-300)
            assert rel < rtol * 10, f"split {i}: near-tie divergence but the gains differ by {rel:.3e}: gpu={a} oracle={b}"
            DIVERGENCES.append((i, margin))
            print(f"[compare_trees] accepted near-tie divergence at split {i}/{ns}: oracle margin {margin:.3e}")
            if min_prefix is not None:
                assert matched >= min_prefix
            return matched, True
        assert a["left_count"] == b["left_count"] and a["right_count"] == b["right_count"], f"split {i} counts {a} {b}"
        for k in ("gain", "left_sum_gradient", "left_sum_hessian", "right_sum_gradient", "right_sum_hessian",
                  "left_output", "right_output"):
            scale = max(abs(b[k]), 1e-12)
            if strict:
                scale = _gain_scale(b) if k == "gain" else abs(b[k])
                assert abs(a[k] - b[k]) <= tol * scale, f"split {i} field {k}: gpu={a[k]!r} oracle={b[k]!r} (strict)"
                continue
            if k.endswith("gradient"):
                # gradient sums can cancel: compare against the magnitude of the leaf's hessian-weighted scale
                scale = max(scale, 1e-6 * max(abs(b["left_sum_hessian"]), abs(b["right_sum_hessian"])))
            assert abs(a[k] - b[k]) <= tol * scale + 1e-9, f"split {i} field {k}: gpu={a[k]!r} oracle={b[k]!r}"
        matched += 1
    if min_prefix is not None:
        assert matched >= min_prefix
    assert gpu.num_leaves == orc.num_leaves, f"num_leaves gpu={gpu.num_leaves} oracle={orc.num_leaves}"
    np.testing.assert_array_equal(gpu.leaf_count, orc.leaf_count)
    if strict:
        np.testing.assert_allclose(gpu.leaf_value, orc.leaf_value, rtol=tol, atol=0)
    else:
        np.testing.assert_allclose(gpu.leaf_value, orc.leaf_value, rtol=tol, atol=1e-9)
    return matched, False


# ---- exact fixed-point reference of the histogram path (DESIGN.md §4.1) -------------------------------------------
# Per tree every row's gradient (hessian) becomes q = rint(value * 2^k) with 2^k the largest power of two such that
# max|value| * 2^k < 2^30, max over ALL rows of the dataset even when a bag or a row subset is histogrammed
# (partition_kernel.cuh pow2_scale / k_quant_rows); a histogram cell is the exact integer sum of its rows' q, and the
# learner reports it as sum * 2^-k (a float64 that holds the integer exactly).

def pow2_exponent(bound) -> int:
    """k with 2^k == pow2_scale(bound): the largest power of two with bound * 2^k < 2^30 (1 when bound is 0)."""
    bound = float(bound)
    if not bound > 0.0:
        return 0
    _, e = math.frexp(bound)            # bound < 2^e
    return max(-1000, min(1000, 30 - e))


def fixed_point_rows(values, k) -> np.ndarray:
    """q = rint(value * 2^k), round half to even (__double2int_rn); the product by a power of two is exact."""
    return np.rint(np.ldexp(np.asarray(values, np.float32).astype(np.float64), k)).astype(np.int64)


def cell_counts(bins, rows=None) -> np.ndarray:
    """int64 [C, 256]: rows per (column, stored value) over `rows` (None = all rows)."""
    b = np.ascontiguousarray((bins if rows is None else bins[rows]).T)
    out = np.zeros((b.shape[0], 256), np.int64)
    for c in range(b.shape[0]):
        out[c] = np.bincount(b[c], minlength=256)
    return out


def cell_sums(bins, rows, q) -> np.ndarray:
    """Exact int64 [C, 256] sums of the per-row integers q (indexed by row id) over `rows` (None = all rows).
    Like the kernel, q is split into hi = q >> 16 and lo = q & 0xffff; each half is bincounted on its own, and its
    float64 partial sums stay integers below 2^53 (|half| < 2^16, fewer than 2^31 rows), so nothing is rounded."""
    q = np.asarray(q, np.int64)
    if rows is not None:
        q = q[rows]
    b = np.ascontiguousarray((bins if rows is None else bins[rows]).T)
    hi, lo = (q >> 16).astype(np.float64), (q & 0xffff).astype(np.float64)
    out = np.zeros((b.shape[0], 256), np.int64)
    for c in range(b.shape[0]):
        sh = np.bincount(b[c], weights=hi, minlength=256)
        sl = np.bincount(b[c], weights=lo, minlength=256)
        out[c] = sh.astype(np.int64) * 65536 + sl.astype(np.int64)
    return out


def fixed_point_hist(bins, rows, g, h, const_hess=False):
    """The histogram the learner computes for the rows `rows` (None = all) of the row-major uint8 matrix `bins`, for
    fp32 gradients g / hessians h over ALL rows.  Returns (sums, values, (kg, kh)): int64 [C, 256, 2] cell sums of the
    fixed-point rows, their float64 values sums * 2^-k (what the learner's pool read-back returns, exactly) and the
    exponents.  const_hess: the count-and-scale kernel, hessian cell = count * llrint(h[0] * 2^kh)."""
    g = np.asarray(g, np.float32)
    h = np.asarray(h, np.float32)
    kg = pow2_exponent(np.max(np.abs(g)) if len(g) else 0.0)
    kh = pow2_exponent(np.max(np.abs(h)) if len(h) else 0.0)
    C = bins.shape[1]
    sums = np.empty((C, 256, 2), np.int64)
    sums[..., 0] = cell_sums(bins, rows, fixed_point_rows(g, kg))
    if const_hess:
        hq = int(np.rint(np.ldexp(float(h[0]), kh)))
        sums[..., 1] = cell_counts(bins, rows) * hq
    else:
        sums[..., 1] = cell_sums(bins, rows, fixed_point_rows(h, kh))
    values = np.empty(sums.shape, np.float64)
    values[..., 0] = np.ldexp(sums[..., 0].astype(np.float64), -kg)
    values[..., 1] = np.ldexp(sums[..., 1].astype(np.float64), -kh)
    return sums, values, (kg, kh)


def int_hist(bins, rows, qg, qh) -> np.ndarray:
    """Quantized training: the pool holds the raw integer sums of the discretized (g, h) (scale 1) -> float64."""
    out = np.empty((bins.shape[1], 256, 2), np.float64)
    out[..., 0] = cell_sums(bins, rows, qg)
    out[..., 1] = cell_sums(bins, rows, qh)
    return out


def assert_hist_equal(got, want, what=""):
    """Bit-for-bit equality of two [C, 256, 2] histograms, with a readable report of the first differing cells."""
    got = np.asarray(got)
    want = np.asarray(want)
    if np.array_equal(got, want):
        return
    bad = np.argwhere(got != want)
    lines = [f"col {c} value {v} {'gh'[k]}: got {got[c, v, k]!r} want {want[c, v, k]!r}" for c, v, k in bad[:8]]
    raise AssertionError(f"{what}: {len(bad)} histogram cells differ\n  " + "\n  ".join(lines))


# ---- exact-input generators: the fixed point loses nothing and the oracle's fp64 sums are exact -------------------

def exact_grad(values, bits=10, bound_log2=6):
    """Round `values` to multiples of 2^-bits and clip to |g| < 2^bound_log2 (fp32 holds them exactly)."""
    lim = 2.0 ** bound_log2 - 2.0 ** -bits
    return np.clip(np.round(np.asarray(values, np.float64) * 2 ** bits) / 2 ** bits, -lim, lim).astype(np.float32)


def exact_hess(rng, n):
    """Multiples of 2^-6 in [2^-3, 4]."""
    return (rng.integers(8, 257, n) * 2.0 ** -6).astype(np.float32)
