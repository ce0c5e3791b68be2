"""Exact-input tree parity.  Gradients are multiples of 2^-10 with |g| < 2^6 and hessians 1 or multiples of 2^-6 in
[2^-3, 4]: the 30-bit fixed point of the histogram path loses nothing and the oracle's fp64 sums are exact, so the GPU
and the oracle add the same numbers.  The whole split sequence must then match (compare_trees(strict=True)): a
divergence is accepted only where the oracle's own margin is <= 1e-12 (fp64 order of the kEpsilon additions, FMA
contraction) and none of the cases below may have one — in particular not at an exact tie, where the reference's
tie-breaks (lower real feature index, then lower leaf index, then earlier threshold in scan order) decide.

Also metamorphic checks that need no oracle: scaling the gradients by 2^+-40, permuting columns across the 32- and
64-column group boundaries, appending or masking inert columns."""
import numpy as np
import pytest

from helpers import ESCAPES, assert_hist_equal, compare_trees, exact_grad, exact_hess

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def mods(built_lib):
    import lightgbm_b200 as lgb
    from oracle import oracle_py
    return lgb, oracle_py


def _strict(lgb, orc, lay, g, h, const_hess=False, bag=None, mask=None, min_splits=1, **cfg):
    """Train on the GPU and in the oracle and require the identical tree (no escape)."""
    L = lgb.B200TreeLearner(lgb.Config(**cfg))
    L.init(lay, is_constant_hessian=const_hess)
    if bag is not None:
        L.set_bagging_data(bag)
    if mask is not None:
        L.set_feature_mask(mask)
    t = L.train(g, h)
    o = orc.train_tree(lay, g, h, bag_indices=bag, feature_used=mask, **cfg)
    n_esc = len(ESCAPES)
    matched, diverged = compare_trees(t, o, strict=True)
    assert not diverged and len(ESCAPES) == n_esc, f"strict comparison escaped at split {matched}: {ESCAPES[n_esc:]}"
    assert matched == o.num_leaves - 1 >= min_splits, (matched, o.num_leaves)
    return L, t, o


def skewed_identity(n, c, seed):
    """90-99.9 % of the rows at stored value 0, two-valued and constant columns, exact L2-like gradients."""
    rng = np.random.default_rng(seed)
    bins = np.zeros((n, c), np.uint8)
    zero_frac = np.linspace(0.9, 0.999, c)
    for j in range(c):
        on = rng.random(n) >= zero_frac[j]
        bins[on, j] = rng.integers(1, 255, int(on.sum()))
    bins[:, 3] = np.where(rng.random(n) < 0.5, 0, 7)            # two-valued
    bins[:, 4] = 0                                               # constant
    bins[:, c - 1] = 42                                          # constant, not at 0
    y = (bins[:, 3] == 7) * 1.5 + (bins[:, 5] > 0) * 2.0 - (bins[:, 6] > 100) * 3.0 + (bins[:, 0] > 0) * 1.0
    g = exact_grad(-y + rng.normal(size=n))
    return bins, g, rng


@pytest.mark.parametrize("n,c,leaves,hess", [(300_000, 96, 31, "exact"), (300_000, 96, 31, "const"),
                                             (1_200_000, 256, 15, "exact")])
def test_skewed_identity_layouts(mods, n, c, leaves, hess):
    """1.2M x 256 with general hessians: the root pass gives each CTA ~73k rows of one set on 132 SMs (crosses a
    flush); the non-root passes are gathered over many CTAs.  "const" selects the count-and-scale kernel."""
    lgb, orc = mods
    bins, g, rng = skewed_identity(n, c, seed=n + c)
    h = np.ones(n, np.float32) if hess == "const" else exact_hess(rng, n)
    _strict(lgb, orc, lgb.Layout.identity(bins), g, h, const_hess=hess == "const", min_splits=leaves - 1,
            num_leaves=leaves)


def _binner_matrix(n, seed):
    """Raw floats: NaN, zeros, few distinct values, exclusive sparse blocks (EFB) — the patterns of binning_cases."""
    rng = np.random.default_rng(seed)
    X = np.zeros((n, 100), np.float32)
    X[:, :30] = rng.normal(size=(n, 30))
    dense = X[:, :30]                                             # a view
    dense[rng.random((n, 30)) < 0.05] = np.nan
    X[:, 30:50] = np.where(rng.random((n, 20)) < 0.8, 0.0, rng.normal(size=(n, 20)))
    X[:, 50:60] = rng.integers(0, 5, (n, 10))
    for b in range(10):                                           # 10 blocks of 4 mutually exclusive sparse features
        which = rng.integers(0, 4, n)
        on = rng.random(n) < 0.1
        vals = rng.integers(1, 64, n).astype(np.float32)
        for k in range(4):
            m = on & (which == k)
            X[m, 60 + 4 * b + k] = vals[m]
    Xn = np.nan_to_num(X)
    y = Xn[:, 0] - 0.5 * Xn[:, 1] + np.isnan(X[:, 2]) * 1.5 + (Xn[:, 31] > 0) + 0.3 * Xn[:, 52] + (Xn[:, 61] > 10)
    return X, y + 0.5 * rng.normal(size=n), rng


@pytest.mark.parametrize("zero_as_missing", ["false", "true"])
def test_binner_layouts(mods, zero_as_missing):
    """Layouts the Binner makes at 200k x 100: most-frequent-bin elision (mfb > 0), NaN and Zero missing types, small
    num_bin and EFB bundles, at scale."""
    lgb, orc = mods
    from binning_cases import BASE
    X, y, rng = _binner_matrix(200_000, seed=77)
    b = lgb.Binner(dict(BASE, zero_as_missing=zero_as_missing)).fit(X)
    bins, _ = b.transform(X, to_device=False)
    lay = b.layout(bins)
    assert lay.num_columns < lay.num_features                     # bundles formed
    assert (lay.feat_mfb > 0).any() and set(np.unique(lay.feat_missing)) >= {2 if zero_as_missing == "false" else 1}
    g = exact_grad(-y)
    _strict(lgb, orc, lay, g, exact_hess(rng, len(g)), min_splits=30, num_leaves=63)


def test_exact_ties_across_features(mods):
    """Columns 20..39 duplicate 0..19 and the real feature indices are permuted: every winning split has an exact
    twin, and the one with the lower REAL index must win (SplitInfo::operator>)."""
    lgb, orc = mods
    n = 200_000
    bins, g, rng = skewed_identity(n, 20, seed=9)
    bins[:, 4] = rng.integers(0, 255, n)                         # no constant column here
    dup = np.concatenate([bins, bins[:, rng.permutation(20)]], axis=1)
    lay = lgb.Layout.identity(dup)
    lay.feat_real_index = rng.permutation(40).astype(np.int32)
    _, t, _ = _strict(lgb, orc, lay, g, exact_hess(rng, n), min_splits=20, num_leaves=31)
    # ties were really there: every split's feature has a twin column with identical bins
    assert len(set(t.splits["feature"])) >= 3


def test_exact_ties_across_leaves(mods):
    """Two copies of the rows, feature 0 = 0 in the first and 1 in the second, gradients negated (+ an offset that
    makes feature 0 the first split) in the second: the two children have mirror histograms, so every candidate of
    one has a twin of equal gain in the other and k_select's leaf tie-break (lower leaf index) decides."""
    lgb, orc = mods
    n = 100_000
    bins, g, rng = skewed_identity(n, 24, seed=11)
    h = exact_hess(rng, n)
    # the second copy also reverses the stored values of the other features (v -> 254 - v): with the same values its
    # rows would cancel the first copy's in every root cell, no feature but 0 would be splittable at the root, and
    # is_splittable_ inheritance would stop the tree after one split.  Reversed, every threshold of one child has a
    # twin in the other with the same two row sets, sides swapped.
    b2 = np.concatenate([bins, (254 - bins).astype(np.uint8)])
    b2[:n, 0], b2[n:, 0] = 0, 1
    g1 = exact_grad(g.astype(np.float64) + 3.0)
    g2 = np.concatenate([g1, -g1])
    h2 = np.concatenate([h, h])
    _, t, _ = _strict(lgb, orc, lgb.Layout.identity(b2), g2, h2, min_splits=20, num_leaves=31)
    s = t.splits
    assert s[0]["feature"] == 0 and s[0]["left_count"] == s[0]["right_count"] == n
    # twins were grown on both sides: the same feature split in both children with gains equal to 1e-12
    twins = [(i, j) for i in range(1, len(s)) for j in range(i + 1, len(s))
             if s[i]["feature"] == s[j]["feature"] and s[i]["threshold"] + s[j]["threshold"] == 253
             and abs(s[i]["gain"] - s[j]["gain"]) <= 1e-12 * abs(s[i]["gain"])]
    assert twins, s[["leaf", "feature", "threshold", "gain"]]


def test_gates_that_bind_exactly(mods):
    """min_data_in_leaf and min_sum_hessian_in_leaf equal to the right-side count / hessian of the best root split,
    max_depth, and min_data_in_leaf = min_sum_hessian_in_leaf = 0 (empty children allowed)."""
    lgb, orc = mods
    n = 200_000
    bins, _, rng = skewed_identity(n, 32, seed=13)
    bins[:, 1] = rng.integers(0, 255, n)
    h = exact_hess(rng, n)
    g = exact_grad(np.where(bins[:, 1] > 250, -20.0, 1.0) + rng.normal(size=n) * 0.1)
    lay = lgb.Layout.identity(bins)
    _, t0, _ = _strict(lgb, orc, lay, g, h, num_leaves=15)
    root = t0.splits[0]
    right = bins[:, root["feature"]] > root["threshold"]          # the root split's right side (no missing values)
    m = int(right.sum())
    assert root["feature"] == 1 and m == root["right_count"] and m < n // 2
    # the root's winning candidate sits exactly at the limit and must still win (rejecting it changes the tree).  The
    # scan estimates counts from hessians (count = h * num_data / sum_h, rounded), so the count gate binds exactly
    # only with constant hessians.
    ones = np.ones(n, np.float32)
    _, t, _ = _strict(lgb, orc, lay, g, ones, num_leaves=15, min_data_in_leaf=m)
    assert t.splits[0]["feature"] == 1 and t.splits[0]["threshold"] == root["threshold"] and t.splits[0]["right_count"] == m
    hs = float(h[right].astype(np.float64).sum())
    _, t, _ = _strict(lgb, orc, lay, g, h, num_leaves=15, min_sum_hessian_in_leaf=hs)
    assert t.splits[0]["feature"] == 1 and t.splits[0]["threshold"] == root["threshold"]
    _strict(lgb, orc, lay, g, h, num_leaves=31, max_depth=3, min_splits=7)
    _strict(lgb, orc, lay, g, h, num_leaves=31, min_data_in_leaf=0, min_sum_hessian_in_leaf=0.0)


def test_all_zero_gradients(mods):
    lgb, orc = mods
    n = 50_000
    bins, _, rng = skewed_identity(n, 16, seed=17)
    g = np.zeros(n, np.float32)
    h = exact_hess(rng, n)
    L = lgb.B200TreeLearner(lgb.Config(num_leaves=15))
    L.init(lgb.Layout.identity(bins))
    t = L.train(g, h)
    o = orc.train_tree(lgb.Layout.identity(bins), g, h, num_leaves=15)
    assert t.num_leaves == o.num_leaves == 1
    assert np.isfinite(t.leaf_value).all() and t.leaf_value[0] == o.leaf_value[0] == 0.0


# ------------------------------------------------------------------------------------------- metamorphic checks

def _train(lgb, lay, g, h, mask=None, **cfg):
    L = lgb.B200TreeLearner(lgb.Config(**cfg))
    L.init(lay)
    if mask is not None:
        L.set_feature_mask(mask)
    return L, L.train(g, h)


STRUCT = ["leaf", "feature", "threshold", "default_left", "left_count", "right_count"]


@pytest.mark.parametrize("e", [40, -40])
def test_gradient_scaling_is_exact(mods, e):
    """g * 2^e: the fixed-point exponent moves by -e, the integers stay, so the histograms, every gain comparison and
    the splits are the same, and leaf values are 2^e times the original, bit for bit (default regularisation)."""
    lgb, _ = mods
    n = 200_000
    bins, g, rng = skewed_identity(n, 40, seed=19)
    h = exact_hess(rng, n)
    lay = lgb.Layout.identity(bins)
    gs = np.ldexp(g, e).astype(np.float32)
    L0, t0 = _train(lgb, lay, g, h, num_leaves=31)
    L1, t1 = _train(lgb, lay, gs, h, num_leaves=31)
    assert t0.num_leaves == t1.num_leaves == 31
    assert np.array_equal(t0.splits[STRUCT], t1.splits[STRUCT])
    assert np.array_equal(np.ldexp(t0.leaf_value, e), t1.leaf_value)
    assert np.array_equal(np.ldexp(t0.splits["gain"], 2 * e), t1.splits["gain"])
    h0, _ = L0.construct_histogram(g, h)
    h1, _ = L1.construct_histogram(gs, h)
    assert_hist_equal(h1[..., 0], np.ldexp(h0[..., 0], e), "scaled gradient histogram")
    assert_hist_equal(h1[..., 1], h0[..., 1], "hessian histogram")


def test_column_permutation_c129(mods):
    """C = 129 (a partial third 64-column group): permuting the columns together with their real indices relabels the
    tree's features and moves every histogram column, nothing else."""
    lgb, _ = mods
    n, c = 150_000, 129
    bins, g, rng = skewed_identity(n, c, seed=23)
    h = exact_hess(rng, n)
    perm = rng.permutation(c)
    lay = lgb.Layout.identity(bins)
    lay_p = lgb.Layout.identity(bins[:, perm])
    lay_p.feat_real_index = perm.astype(np.int32)                 # new feature j is old feature perm[j]
    L0, t0 = _train(lgb, lay, g, h, num_leaves=31)
    L1, t1 = _train(lgb, lay_p, g, h, num_leaves=31)
    assert t0.num_leaves == t1.num_leaves == 31
    assert np.array_equal(perm[t1.splits["feature"]], t0.splits["feature"])
    rest = [k for k in STRUCT if k != "feature"]
    assert np.array_equal(t0.splits[rest], t1.splits[rest]) and np.array_equal(t0.leaf_value, t1.leaf_value)
    h0, _ = L0.construct_histogram(g, h)
    h1, _ = L1.construct_histogram(g, h)
    assert_hist_equal(h1, h0[perm], "permuted columns")


def test_inert_columns(mods):
    """Appending constant columns, or appending them and masking them out, leaves the tree unchanged."""
    lgb, _ = mods
    n, c = 150_000, 40
    bins, g, rng = skewed_identity(n, c, seed=29)
    h = exact_hess(rng, n)
    wide = np.concatenate([bins, np.zeros((n, 30), np.uint8), np.full((n, 1), 200, np.uint8)], axis=1)
    _, t0 = _train(lgb, lgb.Layout.identity(bins), g, h, num_leaves=31)
    _, t1 = _train(lgb, lgb.Layout.identity(wide), g, h, num_leaves=31)
    mask = np.r_[np.ones(c, np.uint8), np.zeros(31, np.uint8)]
    _, t2 = _train(lgb, lgb.Layout.identity(wide), g, h, mask=mask, num_leaves=31)
    for t in (t1, t2):
        assert np.array_equal(t0.splits, t.splits) and np.array_equal(t0.leaf_value, t.leaf_value)
