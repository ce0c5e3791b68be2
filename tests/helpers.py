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


# ---- plain restatements of the rows either side of the path (DESIGN.md §4.8, §4.9) ---------------------------------
# The value -> bin pass and the predictor claim bit identity with LGBM_DatasetCreateFromMat and LGBM_BoosterPredictForMat.
# These restate both in float64 numpy, and the generators below build inputs that sit on and next to every bin bound and
# every threshold, where a `<` for a `<=` or a missing float rounding step would show.

K_ZERO = float(np.float32(1e-35))            # kZeroThreshold (meta.h:56): the float literal, widened
MISSING_NONE, MISSING_ZERO, MISSING_NAN = 0, 1, 2
FLT_MAX = float(np.finfo(np.float32).max)


def value_to_bin_reference(X, meta, upper_bounds):
    """The uint8 [rows, num_columns] matrix LGBM_DatasetCreateFromMat stores for the float matrix X under a fitted layout
    (`Binner.layout_meta()` keys) and its bin upper bounds.  A feature's bin is BinMapper::ValueToBin (bin.h:612-637):
    the count of searchable bounds below (double)x, with num_bin - 1 searchable bounds, one fewer when the last bin is the
    NaN bin; NaN goes to that bin, or is read as 0.0 under the other missing types.  FeatureGroup::PushData stores nothing
    at the most frequent bin and lo + bin - (mfb == 0) elsewhere; a later sub-feature of a bundle overwrites an earlier one."""
    X = np.asarray(X)
    out = np.zeros((X.shape[0], int(meta["num_columns"])), np.uint8)
    for f in range(int(meta["num_features"])):
        nb, mt, mfb = int(meta["feat_num_bin"][f]), int(meta["feat_missing_type"][f]), int(meta["feat_most_freq_bin"][f])
        x = X[:, int(meta["feat_real_index"][f])].astype(np.float64)
        nan = np.isnan(x)
        searchable = nb - 1 - (1 if mt == MISSING_NAN else 0)
        b = np.searchsorted(np.asarray(upper_bounds[f], np.float64)[:searchable], np.where(nan, 0.0, x), side="left")
        if mt == MISSING_NAN:
            b[nan] = nb - 1
        keep = b != mfb
        out[keep, int(meta["feat_column"][f])] = (int(meta["feat_lo"][f]) + b[keep] - (1 if mfb == 0 else 0)).astype(np.uint8)
    return out


def predict_raw_reference(model, X):
    """LGBM_BoosterPredictForMat raw scores of a numerical model (lightgbm_b200.Model) for the float matrix X.  The rows are
    read through RowPairFunctionFromDenseMatrix, which drops every value with |x| <= kZeroThreshold (c_api.cpp:2864), so
    the trees see 0.0 there; each node decides as NumericalDecision does (tree.h:337-355); the leaf values are added in
    float64, one tree at a time in model order, starting from 0 (GBDT::PredictRaw)."""
    X = np.asarray(X).astype(np.float64)
    X = np.where(np.abs(X) <= K_ZERO, 0.0, X)                 # NaN compares false and stays
    n = X.shape[0]
    out = np.zeros(n, np.float64)
    for t in model.trees:
        if t.num_leaves <= 1:
            out += t.leaf_value[0]
            continue
        node = np.zeros(n, np.int64)
        live = np.arange(n)
        while live.size:
            nd = node[live]
            v = X[live, t.split_feature[nd]]
            dt = t.decision_type[nd].astype(np.int64)
            mt = (dt >> 2) & 3
            nan = np.isnan(v)
            v = np.where(nan & (mt != MISSING_NAN), 0.0, v)
            to_default = ((mt == MISSING_ZERO) & (v >= -K_ZERO) & (v <= K_ZERO)) | ((mt == MISSING_NAN) & nan)
            left = np.where(to_default, (dt & 2) != 0, v <= t.threshold[nd])
            node[live] = np.where(left, t.left_child[nd], t.right_child[nd])
            live = live[node[live] >= 0]
        out += t.leaf_value[~node]
    return out


# ---- adversarial inputs: values on and next to bounds and thresholds ------------------------------------------------

def f32_floor(t: float) -> float:
    """The largest float32 <= the double t (what the device compares a float against)."""
    with np.errstate(over="ignore"):
        f = np.float32(t)
    if float(f) > t:
        f = np.nextafter(f, np.float32(-np.inf))
    return float(f)


def _f32_next(v: float, toward: float) -> float:
    with np.errstate(over="ignore"):
        return float(np.nextafter(np.float32(v), np.float32(toward)))


def edge_values(float64: bool) -> list:
    """Values that probe the zero band, the denormals and the ends of the range whatever the bounds are."""
    v = [0.0, -0.0, np.nan, np.inf, -np.inf, FLT_MAX, -FLT_MAX]
    for s in (1.0, -1.0):
        v += [s * K_ZERO, s * _f32_next(K_ZERO, np.inf), s * _f32_next(K_ZERO, 0.0),
              s * float(np.nextafter(K_ZERO, np.inf)), s * float(np.nextafter(K_ZERO, 0.0)), s * 5e-36,
              s * float(np.float32(2.0 ** -149)), s * float(np.float32(1e-40)), s * float(np.float32(1e-38))]
        if float64:
            v += [s * 1e-320, s * 1e-310, s * 1e300]
    return v


def boundary_values(bounds, float64: bool) -> np.ndarray:
    """Per-feature adversarial values for the finite bounds (or thresholds) `bounds`: each bound t, its float64
    neighbours, the largest float <= t and the float above that, values below the first and above the last, and
    edge_values().  Distinct by bit pattern, so +0.0 and -0.0 both stay."""
    b = np.asarray([x for x in np.asarray(bounds, np.float64) if np.isfinite(x)])
    v = list(edge_values(float64))
    for t in b:
        lo = f32_floor(t)
        v += [t, float(np.nextafter(t, np.inf)), float(np.nextafter(t, -np.inf)), lo, _f32_next(lo, np.inf)]
    if len(b):
        v += [b.min() - 1.0 - abs(b.min()), b.max() + 1.0 + abs(b.max())]
    a = np.asarray(v, np.float64)
    return a[np.unique(a.view(np.int64), return_index=True)[1]]


def boundary_matrix(columns, rows, rng, dtype) -> np.ndarray:
    """[max(rows, longest column), len(columns)] matrix of `dtype`: column j lists every value of columns[j] once (in a
    random order), then random repeats of them."""
    n = max([rows] + [len(c) for c in columns])
    X = np.empty((n, len(columns)), np.float64)
    for j, c in enumerate(columns):
        c = np.asarray(c, np.float64)
        X[:, j] = np.concatenate([rng.permutation(c), rng.choice(c, n - len(c))])
    with np.errstate(over="ignore", under="ignore"):
        return np.ascontiguousarray(X.astype(dtype))


def threshold_pool(rng, k=16) -> np.ndarray:
    """Split thresholds: exact floats, doubles no float equals (midpoints of adjacent floats), the zero band (+-kZ, 0,
    values inside it, the double below -kZ), +-1e300 and +-FLT_MAX."""
    f = (rng.normal(size=k) * 10.0 ** rng.integers(-3, 4, k)).astype(np.float32)
    mids = (f.astype(np.float64) + np.nextafter(f, np.float32(np.inf)).astype(np.float64)) / 2.0
    band = [K_ZERO, -K_ZERO, 0.0, -0.0, 5e-36, -5e-36, float(np.nextafter(-K_ZERO, -np.inf)), float(np.nextafter(K_ZERO, 0.0)),
            float(np.nextafter(-K_ZERO, 0.0))]
    return np.concatenate([f.astype(np.float64), mids, band, [1e300, -1e300, FLT_MAX, -FLT_MAX]])


def _tree_links(pick_leaf, L):
    """Child arrays of a tree grown as Tree::Split grows one (tree.h:543-585): split `node` turns leaf pick_leaf(node)
    into an internal node whose left child keeps that leaf id and whose right child is the new leaf node + 1."""
    n = L - 1
    lc, rc = np.zeros(n, np.int32), np.zeros(n, np.int32)
    parent = np.full(L, -1, np.int64)
    for node in range(n):
        leaf = pick_leaf(node)
        p = parent[leaf]
        if p >= 0:
            if lc[p] == ~leaf:
                lc[p] = node
            else:
                rc[p] = node
        lc[node], rc[node] = ~leaf, ~(node + 1)
        parent[leaf] = parent[node + 1] = node
    return lc, rc


def synthetic_tree(rng, shape, features, pool, decision_types=None):
    """A ModelTree of `shape`: "random" (2..64 leaves), "chain" (255 leaves, 254 deep, zig-zag), "balanced" (2..128
    leaves, full levels) or "leaf" (a single leaf).  Split features from `features`, thresholds from `pool`, decision
    types from `decision_types` (default: all six numerical ones).  Leaf values span 16 decades, so the order in which
    they are added changes the sum."""
    from lightgbm_b200.model import ModelTree
    if shape == "leaf":
        L, lc, rc = 1, np.zeros(0, np.int32), np.zeros(0, np.int32)
    elif shape == "random":
        L = int(rng.integers(2, 65))
        lc, rc = _tree_links(lambda node: int(rng.integers(0, node + 1)), L)
    elif shape == "balanced":
        depth = int(rng.integers(1, 8))
        L = 1 << depth
        order = [j for d in range(depth) for j in range(1 << d)]
        lc, rc = _tree_links(lambda node: order[node], L)
    else:
        L = 255
        last = [0]

        def pick(node):                          # one of the two children of the previous split
            if node > 0 and rng.random() < 0.5:
                last[0] = node
            return last[0]
        lc, rc = _tree_links(pick, L)
    n = L - 1
    dts = np.asarray(decision_types if decision_types is not None else [m << 2 | d for m in range(3) for d in (0, 2)], np.int8)
    return ModelTree(L, rng.choice(np.asarray(features, np.int32), n).astype(np.int32), np.ones(n, np.float32),
                     rng.choice(np.asarray(pool, np.float64), n), rng.choice(dts, n).astype(np.int8), lc, rc,
                     rng.normal(size=L) * 10.0 ** rng.integers(-8, 8, L), np.ones(L), np.ones(L, np.int32),
                     np.zeros(n), np.zeros(n), np.zeros(n, np.int32))


def text_model(trees, ncol):
    """Write the trees as model text and read it back (Model.to_string / Model.from_string), as a user's model arrives."""
    from lightgbm_b200.model import Model
    return Model.from_string(Model(trees=list(trees), max_feature_idx=ncol - 1).to_string())


def synthetic_model(rng, num_trees, ncol, features=None, pool=None, shapes=("random", "chain", "balanced", "leaf")):
    features = list(range(ncol)) if features is None else features
    pool = threshold_pool(rng) if pool is None else pool
    return text_model([synthetic_tree(rng, shapes[i % len(shapes)], features, pool) for i in range(num_trees)], ncol)


def stump_grid_model(pool, ncol):
    """One single-split tree per (threshold, decision type) pair, round-robin over the columns: with every column holding
    every adversarial value, each value meets each threshold under each missing type and default direction."""
    from lightgbm_b200.model import ModelTree
    trees = []
    dts = [m << 2 | d for m in range(3) for d in (0, 2)]
    for i, (t, dt) in enumerate((t, dt) for t in pool for dt in dts):
        trees.append(ModelTree(2, np.array([i % ncol], np.int32), np.ones(1, np.float32), np.array([t]), np.array([dt], np.int8),
                               np.array([-1], np.int32), np.array([-2], np.int32), np.array([2.0 ** -(i % 40), -(3.0 ** (i % 23))]),
                               np.ones(2), np.ones(2, np.int32), np.zeros(1), np.zeros(1), np.zeros(1, np.int32)))
    return text_model(trees, ncol)


def model_columns(model, ncol, float64):
    """boundary_values() of every column from the thresholds the model splits it on."""
    th = [[] for _ in range(ncol)]
    for t in model.trees:
        for f, v in zip(t.split_feature[:t.num_leaves - 1], t.threshold[:t.num_leaves - 1]):
            th[int(f)].append(float(v))
    return [boundary_values(c, float64) for c in th]


# Binner features whose searchable bound counts hit every depth edge of search_bounds_smem (binning.cuh)
BOUND_COUNTS = (0, 1, 2, 3, 4, 7, 8, 15, 16, 31, 32, 63, 64, 127, 128, 254)


def binner_fit_matrix(rng, n=2000, dtype=np.float32):
    """A float matrix to fit with min_data_in_bin=1 and feature_pre_filter=false.  k distinct positive values give k
    searchable bounds (kZeroThreshold, then the k - 1 midpoints); a zero + NaN column gives a NaN-bin feature with none
    searchable, a constant + NaN column one; mixed-sign columns put -kZ and kZ among the bounds; a continuous column
    takes the equal-count branch of the bin finder."""
    cols = []

    def spread(vals):
        vals = np.asarray(vals, np.float64)
        return rng.permutation(np.concatenate([vals, rng.choice(vals, n - len(vals))]))
    for r in BOUND_COUNTS[1:]:
        cols.append(spread(np.unique(rng.uniform(0.5, 1000.0, 4 * r).astype(np.float32))[:r]))
    cols.append(np.where(rng.random(n) < 0.5, 0.0, np.nan))                         # zero + NaN: no searchable bound
    cols.append(np.where(rng.random(n) < 0.3, np.nan, 3.25))                        # constant + NaN: one
    cols.append(spread(np.arange(-3.0, 4.0)))                                       # -3 .. 3: -kZ and kZ are bounds
    cols.append(spread(np.concatenate([-np.unique(rng.uniform(1e-3, 50, 40).astype(np.float32)), [0.0]])))
    c = rng.normal(size=n); c[rng.random(n) < 0.1] = np.nan; cols.append(c)          # continuous with NaN
    c = rng.normal(size=n) * 1e-30; c[rng.random(n) < 0.3] = 0.0; cols.append(c)     # values near the zero band
    return np.ascontiguousarray(np.stack(cols, axis=1).astype(dtype))


def binner_sparse_matrix(rng, n=3000, c=24, dtype=np.float32):
    """Mostly exclusive sparse columns (each row has one non-zero column), which feature bundling packs into shared
    stored columns, next to two dense ones."""
    X = np.zeros((n, c), np.float64)
    owner = rng.permutation(np.concatenate([np.arange(c - 2), rng.integers(0, c - 2, n - (c - 2))]))     # every column used
    X[np.arange(n), owner] = rng.choice(np.array([-2.5, -1.0, 0.5, 1.0, 2.0, 7.0]), n) * (1 + owner % 3)
    X[:, c - 2] = rng.normal(size=n)
    X[:, c - 1] = np.round(rng.normal(size=n) * 3)
    return np.ascontiguousarray(X.astype(dtype))


def binner_columns(meta, ub, ncol, float64):
    """boundary_values() of every real column from its fitted searchable bounds (edge values alone for unused columns)."""
    cols = [boundary_values([], float64) for _ in range(ncol)]
    for f in range(int(meta["num_features"])):
        nb, mt = int(meta["feat_num_bin"][f]), int(meta["feat_missing_type"][f])
        cols[int(meta["feat_real_index"][f])] = boundary_values(ub[f][:nb - 1 - (1 if mt == MISSING_NAN else 0)], float64)
    return cols
