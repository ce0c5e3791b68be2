"""One boosting iteration, bit for bit: everything B200Booster.update drives between one tree and the next must equal the
plain restatements of tests/helpers.py (pinned on the CPU by tests/test_boosting_reference.py).

  * GOSS (k_goss_begin / hist / pick / mark / scatter): the bag and the rescaled gradients equal goss_reference at sizes
    around the warp, block and radix-pass limits, on keys with ties, zeros, denormals and one-bucket radix passes, and at
    the rate edges; rows 2k and 2k + 1 are drawn independently;
  * stochastic rounding (k_quantize): every histogram slot after trees 1, 2 and 3 holds the integer sums of the oracle's
    discretization with the counter_uniform draws, and the trees equal the oracle's;
  * the objective's gradients (k_l2_gradients byte for byte, k_binary_gradients within one float ulp);
  * the score update (k_add_score, k_leaf_index 8- and 32-bit with the host add, k_route_rows) on trees of 2 .. 1025 leaves;
  * the booster loop and lightgbm_b200.train end to end: scores equal the model's predictions byte for byte, and the
    booster's handling of trees that cannot split, of the zero band and of tiny init scores equals the reference's."""
import math

import numpy as np
import pytest

import helpers as H
from test_gpu_hist_exact import check_leaf_histograms

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lgb(built_lib):
    import lightgbm_b200
    return lightgbm_b200


def _ulps(a, b):
    """float32 ulp distance (same sign assumed; +-0 count as equal)."""
    ia = np.asarray(a, np.float32).view(np.int32).astype(np.int64)
    ib = np.asarray(b, np.float32).view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = np.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    return np.abs(ia - ib)


# ---------------------------------------------------------------------------------------------------- GOSS
_LEARNERS = {}


def _goss_learner(lgb, n):
    if n not in _LEARNERS:
        L = lgb.B200TreeLearner(lgb.Config(num_leaves=4, min_data_in_leaf=1))
        L.init(lgb.Layout.identity(np.zeros((n, 1), np.uint8), num_bin=2))
        _LEARNERS.clear()
        _LEARNERS[n] = L
    return _LEARNERS[n]


def _keys(kind, n, rng):
    h = np.ones(n, np.float32)
    if kind == "distinct":
        g = rng.normal(size=n).astype(np.float32)
        h = (0.05 + rng.random(n)).astype(np.float32)
    elif kind == "ties":                        # a handful of values: the threshold has many equal keys
        g = rng.choice(np.float32([-3.0, -1.0, 0.5, 1.0, 2.0]), n).astype(np.float32)
    elif kind == "equal":
        g = np.full(n, 0.75, np.float32)
    elif kind == "zeros":                       # key 0 becomes the threshold
        g = np.where(rng.random(n) < 0.9, 0.0, rng.normal(size=n)).astype(np.float32)
    elif kind == "low_byte":                    # keys differ only in the low byte: three passes see one bucket
        g = (np.uint32(0x3F800000) + rng.integers(0, 256, n).astype(np.uint32)).view(np.float32)
    elif kind == "denormal":                    # products in the denormal range, some flushed to 0 by the rounding
        g = (rng.normal(size=n) * 1e-20).astype(np.float32)
        h = (rng.random(n) * 1e-20).astype(np.float32)
    else:                                       # full exponent range
        g = (np.ldexp(1.0 + rng.random(n), rng.integers(-126, 127, n)) * rng.choice([-1.0, 1.0], n)).astype(np.float32)
    return np.ascontiguousarray(g), np.ascontiguousarray(h)


def _goss_check(lgb, g, h, top, other, seed=7, it=11):
    from lightgbm_b200.tree_learner import DeviceArray
    n = len(g)
    L = _goss_learner(lgb, n)
    dg, dh = DeviceArray(n * 4).upload(g), DeviceArray(n * 4).upload(h)
    cnt = L.goss_sample(dg, dh, top, other, seed=seed, iteration=it)
    bag, g2, h2 = H.goss_reference(g, h, top, other, seed, it)
    got = L.get_bagging_data(cnt)
    assert cnt == len(bag) and got.tobytes() == bag.tobytes(), f"bag: {cnt} rows, want {len(bag)}"
    assert dg.download(np.float32, n).tobytes() == g2.tobytes()
    assert dh.download(np.float32, n).tobytes() == h2.tobytes()
    return bag


# part_blocks_ = 2 * SMs: on a 132-SM H100 (264 blocks of 256-row multiples), 65 537 rows leave blocks 257 .. 263 empty,
# 200 001 rows blocks 261 .. 263, and 134 657 rows leave the last block a single row
GOSS_SIZES = (1, 2, 31, 32, 33, 255, 256, 257, 65_537, 134_657, 200_001)


@pytest.mark.parametrize("n", GOSS_SIZES)
def test_goss_sizes(lgb, n):
    g, h = _keys("distinct", n, np.random.default_rng(n))
    _goss_check(lgb, g, h, 0.2, 0.1)


@pytest.mark.parametrize("kind", ["ties", "equal", "zeros", "low_byte", "denormal", "full_range"])
@pytest.mark.parametrize("n", [257, 65_537])
def test_goss_keys(lgb, kind, n):
    g, h = _keys(kind, n, np.random.default_rng(3))
    _goss_check(lgb, g, h, 0.2, 0.1)


@pytest.mark.parametrize("top,other", [(1e-9, 0.1), (0.2, 0.5 / 65_537), (0.3, 0.7), (0.05, 0.95)])
def test_goss_rates(lgb, top, other):
    """top_k floored to 1; other_k = 0 (nothing drawn, multiplier 0 unused); top + other = 1."""
    g, h = _keys("distinct", 65_537, np.random.default_rng(4))
    _goss_check(lgb, g, h, top, other)


def test_goss_draws_rows_independently(lgb):
    """Rows 2k and 2k + 1 are both drawn at rate p^2 (a draw shared by the pair gives p)."""
    n = 200_001
    rng = np.random.default_rng(5)
    g, h = _keys("distinct", n, rng)
    top, other = 0.01, 0.49
    bag = _goss_check(lgb, g, h, top, other)
    key = np.abs(g * h)
    kth = np.sort(key)[n - max(1, int(n * top))]
    small = key < kth
    drawn = np.zeros(n, bool); drawn[bag] = True; drawn &= small
    pairs = small[0:n - 1:2] & small[1::2]
    both = int(np.sum(drawn[0:n - 1:2][pairs] & drawn[1::2][pairs]))
    m, p = int(pairs.sum()), other / (1 - top)
    assert abs(both - m * p * p) <= 6 * np.sqrt(m * p * p * (1 - p * p)) + 1, (both, m * p * p, m * p)


# --------------------------------------------------------------------------------------------- stochastic rounding
@pytest.mark.parametrize("bins_q", [4, 16])
@pytest.mark.parametrize("const_hess,bagging", [(False, False), (True, False), (False, True)])
def test_stochastic_rounding_histograms_and_trees(lgb, bins_q, const_hess, bagging):
    from exact_worker import leaf_data
    from oracle import oracle_py
    bins, g, h, bag, _, cfg, _ = leaf_data("bagging" if bagging else "plain", n=60_000)
    if const_hess:
        h = np.ones_like(h)
    cfg = dict(cfg, use_quantized_grad=True, num_grad_quant_bins=bins_q, stochastic_rounding=True, seed=12345)
    lay = lgb.Layout.identity(bins)
    L = lgb.B200TreeLearner(lgb.Config(**cfg))
    L.init(lay, is_constant_hessian=const_hess)
    if bag is not None:
        L.set_bagging_data(bag)
    rows = np.arange(len(g))
    rng = np.random.default_rng(9)
    for t in (1, 2, 3):
        gt = (g * np.float32(1 + 0.25 * (t - 1)) + rng.normal(size=len(g)).astype(np.float32) * np.float32(0.01)).astype(np.float32)
        rg = H.counter_uniform(cfg["seed"], t, rows, H.QUANT_G_STREAM)
        rh = H.counter_uniform(cfg["seed"], t, rows, H.QUANT_H_STREAM)
        tree = L.train(gt, h)
        part = L.get_partition(tree.num_leaves)
        hists = np.stack([L.get_leaf_histogram(i) for i in range(tree.num_leaves)])
        qg, qh, _, _ = oracle_py.discretize(gt, h, bins_q, const_hess, random_g=rg, random_h=rh)
        want = lambda r: H.int_hist(bins, r, qg.astype(np.int64), qh.astype(np.int64))   # noqa: E731
        assert tree.num_leaves == cfg["num_leaves"]
        checked = check_leaf_histograms(bins, tree, part, hists, want, cfg)
        assert checked >= 10, checked
        o = oracle_py.train_tree_quant(lay, gt, h, bins_q, const_hess, bag_indices=bag, random_g=rg, random_h=rh,
                                       **{k: cfg[k] for k in ("num_leaves", "min_data_in_leaf", "min_sum_hessian_in_leaf")})
        matched, diverged = H.compare_trees(tree, o, strict=True)
        assert not diverged and matched == o.num_leaves - 1, (t, matched)


# ---------------------------------------------------------------------------------------------------- gradients
SCORE_EDGES = np.array([0.0, -0.0, 1e-300, -1e-300, 30.0, -30.0, 800.0, -800.0, 1.0, -1.0, 36.7, -36.7, 1e-8, -745.2, 710.0])


def _scores_labels(n, rng):
    s = np.concatenate([np.repeat(SCORE_EDGES, 2), rng.normal(size=n) * 10.0 ** rng.integers(-6, 3, n)])
    y = np.concatenate([np.tile(np.float32([0.0, 1.0]), len(SCORE_EDGES)), (rng.random(n) < 0.5).astype(np.float32)])
    return np.ascontiguousarray(s), np.ascontiguousarray(y)


def _device_gradients(lgb, kind, s, y, sigmoid=1.0):
    from lightgbm_b200.tree_learner import DeviceArray
    n = len(s)
    L = _goss_learner(lgb, n)
    ds, dy, dg, dh = DeviceArray(n * 8).upload(s), DeviceArray(n * 4).upload(y), DeviceArray(n * 4), DeviceArray(n * 4)
    if kind == "l2":
        L.l2_gradients(ds, dy, dg, dh, n)
    else:
        L.binary_gradients(ds, dy, dg, dh, n, sigmoid)
    return dg.download(np.float32, n), dh.download(np.float32, n)


def test_l2_gradients_bytes(lgb):
    rng = np.random.default_rng(1)
    s, _ = _scores_labels(20_000, rng)
    y = (rng.normal(size=len(s)) * 10.0 ** rng.integers(-8, 8, len(s))).astype(np.float32)
    s = s + np.where(rng.random(len(s)) < 0.3, y.astype(np.float64) * (1 + 2.0 ** -40), 0.0)   # near-cancelling pairs
    g, h = _device_gradients(lgb, "l2", s, y)
    wg, wh = H.l2_gradients_reference(s, y)
    assert g.tobytes() == wg.tobytes() and h.tobytes() == wh.tobytes()


@pytest.mark.parametrize("sigmoid", [0.5, 1.0, 2.7])
def test_binary_gradients_within_one_ulp(lgb, sigmoid):
    """CUDA's double exp and libm's may differ by an ulp of the double, which can move a float rounding by one: every
    value is within 1 float ulp of the restatement; the count that differs is printed."""
    s, y = _scores_labels(20_000, np.random.default_rng(2))
    g, h = _device_gradients(lgb, "binary", s, y, sigmoid)
    wg, wh = H.binary_gradients_reference(s, y, sigmoid)
    assert np.array_equal(np.signbit(g), np.signbit(wg))
    dg, dh = _ulps(g, wg), _ulps(h, wh)
    print(f"[binary sigmoid={sigmoid}] {int((dg > 0).sum())} gradients and {int((dh > 0).sum())} hessians of {len(s)} differ by 1 ulp")
    assert dg.max() <= 1 and dh.max() <= 1
    # where exp is exact (1e-300, 0) or overflows / underflows (+-800) the bytes agree
    edge = np.zeros(len(s), bool)
    edge[:2 * len(SCORE_EDGES)] = np.isin(np.abs(s[:2 * len(SCORE_EDGES)]), [0.0, 1e-300, 800.0])
    assert g[edge].tobytes() == wg[edge].tobytes() and h[edge].tobytes() == wh[edge].tobytes()


# ---------------------------------------------------------------------------------------------------- score update
LEAF_COUNTS = (2, 255, 256, 946, 947, 1025)


def _layout(lgb, kind, n, rng):
    if kind == "identity":
        bins = rng.integers(0, 255, (n, 12), dtype=np.uint8)
        bins[rng.random((n, 12)) < 0.3] = 0
        return lgb.Layout.identity(bins)
    if kind == "binner":               # NaN and zero missing types, mfb > 0, values near the zero band
        X = H.binner_fit_matrix(rng, n=n)
        params = dict(max_bin=255, min_data_in_bin=1, min_data_in_leaf=1, feature_pre_filter="false", enable_bundle="false")
    else:                              # EFB bundles
        X = H.binner_sparse_matrix(rng, n=n)
        params = dict(max_bin=63, min_data_in_bin=1, min_data_in_leaf=1, feature_pre_filter="false", enable_bundle="true")
    b = lgb.Binner(params).fit(X)
    bins, _ = b.transform(X, to_device=False)
    return b.layout(bins)


_LAYOUTS = {}


@pytest.mark.parametrize("bagging", ["none", "sorted", "goss"])
@pytest.mark.parametrize("layout", ["identity", "binner", "bundled"])
@pytest.mark.parametrize("leaves", LEAF_COUNTS)
def test_score_update_paths(lgb, leaves, layout, bagging):
    from lightgbm_b200.tree_learner import DeviceArray
    n = 24_000
    rng = np.random.default_rng(leaves)
    if layout not in _LAYOUTS:
        _LAYOUTS[layout] = _layout(lgb, layout, n, np.random.default_rng(17))
    lay = _LAYOUTS[layout]
    if layout == "bundled":
        assert len(set(lay.feat_column.tolist())) < lay.num_features
    g = rng.normal(size=n).astype(np.float32)
    h = (0.5 + rng.random(n)).astype(np.float32)
    L = lgb.B200TreeLearner(lgb.Config(num_leaves=leaves, min_data_in_leaf=1, min_sum_hessian_in_leaf=1e-6))
    L.init(lay)
    dg, dh = DeviceArray(n * 4).upload(g), DeviceArray(n * 4).upload(h)
    bag = None
    if bagging == "sorted":
        bag = np.sort(rng.choice(n, n * 3 // 4, replace=False)).astype(np.int32)
        L.set_bagging_data(bag)
    elif bagging == "goss":
        cnt = L.goss_sample(dg, dh, 0.3, 0.4, seed=2, iteration=3)
        bag = L.get_bagging_data(cnt)
    t = L.train(dg, dh)
    assert t.num_leaves == leaves
    leaf_bag = H.route_rows_reference(lay, t.splits, bag)
    leaf_all = H.route_rows_reference(lay, t.splits)
    lb, lc, idx = L.get_partition(leaves)
    part = np.full(n, -1, np.int32)
    for l in range(leaves):
        part[idx[lb[l]:lb[l] + lc[l]]] = l
    assert np.array_equal(part, leaf_bag), "partition leaf != the replayed split rule"
    t.leaf_value = rng.normal(size=leaves) * 10.0 ** rng.integers(-3, 3, leaves)
    s0 = rng.normal(size=n)
    # device score: the partition's rows only
    ds = DeviceArray(n * 8).upload(s0)
    L.add_prediction_to_score(t, ds)
    assert ds.download(np.float64, n).tobytes() == H.boost_step_reference(s0, t.leaf_value, leaf_bag).tobytes()
    # host score: leaf ids shipped as uint8 (0xFF outside the bag) up to 255 leaves, else int32
    hs = s0.copy()
    L.add_prediction_to_score(t, hs)
    assert hs.tobytes() == H.boost_step_reference(s0, t.leaf_value, leaf_bag).tobytes()
    if leaves <= 255:
        lo, hi = 37, n - 5
        out = np.zeros(hi - lo, np.uint8)
        L.get_leaf_index_range8(lo, hi, out)
        assert out.tobytes() == np.where(leaf_bag < 0, 255, leaf_bag)[lo:hi].astype(np.uint8).tobytes()
    # every row through the tree (out-of-bag rows too)
    ds.upload(s0)
    L.add_prediction_all_rows(t, ds)
    assert ds.download(np.float64, n).tobytes() == H.boost_step_reference(s0, t.leaf_value, leaf_all).tobytes()


# ---------------------------------------------------------------------------------------------------- zero hessians
def test_zero_hessian_rows_keep_their_gradients(lgb):
    """Rows whose hessian is 0 (a saturated logistic: |response| = 1 in float) still carry their gradient.  A cell
    holding only such rows has a hessian sum of 0 and a gradient sum that is not 0; the scan must add that gradient to
    its side like any other.  Exact inputs: the oracle's fp64 sums and the fixed point agree, so the trees must match
    strictly."""
    from oracle import oracle_py
    rng = np.random.default_rng(21)
    n = 6000
    bins = rng.integers(0, 16, (n, 4), dtype=np.uint8)
    g = H.exact_grad(rng.normal(size=n) * 0.1)
    h = H.exact_hess(rng, n)
    sat = np.isin(bins[:, 0], [3, 11])
    g[sat], h[sat] = np.float32(-1.0), np.float32(0.0)
    lay = lgb.Layout.identity(bins, num_bin=16)
    kw = dict(num_leaves=15, min_data_in_leaf=5)
    L = lgb.B200TreeLearner(lgb.Config(**kw))
    L.init(lay)
    t = L.train(g, h)
    o = oracle_py.train_tree(lay, g, h, **kw)
    matched, diverged = H.compare_trees(t, o, strict=True)
    assert not diverged and matched == o.num_leaves - 1, matched


# ---------------------------------------------------------------------------------------------------- booster loop
class _Recorder:
    """Records the raw tree each Train returns and the leaf values each score update adds."""

    def __init__(self, learner):
        self.raw, self.added = [], []
        for name in ("train", "add_prediction_to_score", "add_prediction_all_rows"):
            fn = getattr(learner, name)
            setattr(learner, name, self._wrap(name, fn))

    def _wrap(self, name, fn):
        import copy

        def w(*a, **k):
            out = fn(*a, **k)
            if name == "train":
                self.raw.append(copy.deepcopy(out))
            else:
                self.added.append((name, np.array(a[0].leaf_value)))
            return out
        return w


LOOP_CASES = {
    "l2_const_hess": dict(objective="regression", learning_rate=0.1),
    # lr 0.1 as in the bench configs: at 0.3 the logistic saturates within six trees, and gains computed from hessian sums
    # near 0 then magnify the fixed point's rounding (n * 2^-(k+1) per sum, DESIGN.md §4.1) past this tier's 1e-4;
    # test_zero_hessian_rows_keep_their_gradients holds the saturated case exactly
    "binary": dict(objective="binary", learning_rate=0.1),
    "goss": dict(objective="regression", learning_rate=0.5, data_sample_strategy="goss", top_rate=0.2, other_rate=0.3),
    "quantized": dict(objective="regression", learning_rate=0.2, quant=True),
}


@pytest.mark.parametrize("case", list(LOOP_CASES))
def test_booster_handover_loop(lgb, case):
    from oracle import oracle_py
    from lightgbm_b200.tree_learner import round_to_zero
    p = dict(LOOP_CASES[case])
    quant = p.pop("quant", False)
    n, nl = 30_000, 31
    rng = np.random.default_rng(6)
    bins = rng.integers(0, 64, (n, 10), dtype=np.uint8)
    z = bins[:, :4].astype(np.float64) @ rng.normal(size=4) / 30 + 0.3 * rng.normal(size=n)
    y = (z > 0).astype(np.float32) if p["objective"] == "binary" else z.astype(np.float32)
    lay = lgb.Layout.identity(bins, num_bin=64)
    cfg = lgb.Config(num_leaves=nl, min_data_in_leaf=5, use_quantized_grad=quant, num_grad_quant_bins=8,
                     stochastic_rounding=True, seed=77)
    B = lgb.B200Booster(lay, y, cfg, **p)
    rec = _Recorder(B.learner)
    lr = p["learning_rate"]
    for it in range(6):
        s0 = B.scores()
        t = B.update()
        assert not B.finished and t.num_leaves > 1
        raw = rec.raw[-1]
        if p["objective"] == "binary":
            wg, wh = H.binary_gradients_reference(s0, y, 1.0)
        else:
            wg, wh = H.l2_gradients_reference(s0, y)
        dg, dh = B.d_grad.download(np.float32, n), B.d_hess.download(np.float32, n)
        bag = None
        sampled = B.goss and it >= int(1.0 / lr)
        if sampled:
            bag, wg, wh = H.goss_reference(wg, wh, p["top_rate"], p["other_rate"], B.bagging_seed, it)
            assert B.learner.get_bagging_data(len(bag)).tobytes() == bag.tobytes()
        if p["objective"] == "binary":
            assert _ulps(dg, wg).max() <= 1 and _ulps(dh, wh).max() <= 1
        else:
            assert dg.tobytes() == wg.tobytes() and dh.tobytes() == wh.tobytes(), f"iteration {it}: gradients"
        # the tree on the device's own gradients
        kw = dict(num_leaves=nl, min_data_in_leaf=5)
        if quant:
            rows = np.arange(n)
            const = p["objective"] == "regression" and not B.goss
            o = oracle_py.train_tree_quant(lay, dg, dh, 8, const, bag_indices=bag,
                                           random_g=H.counter_uniform(77, it + 1, rows, H.QUANT_G_STREAM),
                                           random_h=H.counter_uniform(77, it + 1, rows, H.QUANT_H_STREAM), **kw)
            matched, diverged = H.compare_trees(raw, o, strict=True)
            assert not diverged and matched == o.num_leaves - 1
        else:
            o = oracle_py.train_tree(lay, dg, dh, bag_indices=bag, **kw)
            matched, diverged = H.compare_trees(raw, o, 1e-5)
            assert diverged or matched == o.num_leaves - 1
        # the score update adds the shrunk leaf values, rounded to zero, at every row's leaf
        name, added = rec.added[-1]
        assert name == ("add_prediction_all_rows" if sampled else "add_prediction_to_score")
        assert added.tobytes() == round_to_zero(raw.leaf_value * lr).tobytes()
        leaf = H.route_rows_reference(lay, raw.splits)
        assert B.scores().tobytes() == H.boost_step_reference(s0, added, leaf).tobytes(), f"iteration {it}: scores"


# ---------------------------------------------------------------------------------------------------- end to end
def _raw_matrix(rng, n):
    X = rng.normal(size=(n, 14)).astype(np.float32)
    X[rng.random((n, 14)) < 0.05] = np.nan
    X[:, 3] = np.where(rng.random(n) < 0.6, 0.0, X[:, 3])
    # values strictly inside the zero band: binned with 0 and read as 0 by the predictor.  +-kZeroThreshold itself is a
    # bin bound: the reference's Dataset bins -kZ below it and its predictor reads it as 0, so its training scores and
    # its own predictions disagree there, and so do this booster's (DESIGN.md §9)
    X[:, 4] = np.where(rng.random(n) < 0.3, rng.choice(np.float32([1e-36, -1e-36, 5e-36, -9e-36]), n), X[:, 4])
    sp = H.binner_sparse_matrix(rng, n=n, c=8)            # exclusive sparse columns: bundled
    X = np.ascontiguousarray(np.concatenate([X, sp], axis=1))
    s = np.nan_to_num(X[:, 0]) - 2 * np.nan_to_num(X[:, 4]) * 1e35 + np.nan_to_num(X[:, 5]) + 0.3 * sp[:, 0]
    return X, s


@pytest.mark.parametrize("objective", ["regression", "binary"])
@pytest.mark.parametrize("goss", [False, True])
def test_train_scores_equal_model_predictions(lgb, objective, goss):
    from oracle import refapi
    rng = np.random.default_rng(8)
    n = 20_000
    X, s = _raw_matrix(rng, n)
    y = (s + 0.2 * rng.normal(size=n)).astype(np.float32) if objective == "regression" else (s > 0).astype(np.float32)
    params = dict(objective=objective, num_leaves=31, learning_rate=0.25, min_data_in_leaf=10, min_data_in_bin=1)
    if goss:
        params.update(data_sample_strategy="goss", top_rate=0.2, other_rate=0.2)
    bst = lgb.train(params, lgb.Dataset(X, label=y), num_boost_round=9)
    assert len(bst.trees) == 9
    model = bst.to_model()
    text = model.to_string()
    scores = bst.scores()
    assert model.predict_raw(X).tobytes() == scores.tobytes()
    assert H.predict_raw_reference(lgb.Model.from_string(text), X).tobytes() == scores.tobytes()
    if refapi.available():
        loaded = refapi.RefLoadedBooster(text)
        assert loaded.predict(X, raw_score=True).tobytes() == scores.tobytes()
        loaded.free()


# ---------------------------------------------------------------------------------------------------- TrainOneIter
def _ref_run(X, y, params, rounds):
    from oracle import refapi
    p = dict(params, verbosity=-1, num_threads=1, deterministic="true")
    ds = refapi.RefDataset(X, y, p)
    b = refapi.RefBooster(ds, p)
    for _ in range(rounds):
        if b.update():
            break
    out = (b.trees(), b.inner_predict())
    b.free(); ds.free()
    return out


def _semantics_case(name, rng):
    n = 400
    x = (np.arange(n) % 4).astype(np.float32)
    X = np.ascontiguousarray(np.stack([x, rng.normal(size=n).astype(np.float32)], axis=1))
    base = dict(objective="regression", num_leaves=4, min_data_in_leaf=5, min_data_in_bin=1, learning_rate=0.1,
                feature_pre_filter="false")
    if name == "first_tree_no_split":
        return X, rng.normal(size=n).astype(np.float32), dict(base, min_data_in_leaf=300)
    if name == "first_tree_no_split_no_average":
        return X, rng.normal(size=n).astype(np.float32), dict(base, min_data_in_leaf=300, boost_from_average="false")
    if name == "later_tree_no_split":       # one step fits the labels: what is left of tree 2's gain is below the gate
        return X, (x * 100).astype(np.float32), dict(base, learning_rate=1.0, min_gain_to_split=1.0)
    if name == "zero_band_leaves":          # shrunk leaf values inside +-1e-35
        return X, np.where(x > 1, 2e-35, -3e-35).astype(np.float32), dict(base, boost_from_average="false")
    if name == "binary_all_positive":       # pavg = 1 is clamped to 1 - kEpsilon, and no split has gain
        return X, np.ones(n, np.float32), dict(base, objective="binary", min_gain_to_split=1e-9)
    # mean label in (0, kEpsilon]: balanced +-1 labels and two tiny ones; no init score, no bias
    y = np.where(x > 1, 1.0, -1.0).astype(np.float32)
    y[[0, 2]] = np.float32(1e-13)
    return X, y, base


SEMANTICS = ["first_tree_no_split", "first_tree_no_split_no_average", "later_tree_no_split", "zero_band_leaves",
             "binary_all_positive", "tiny_mean_label"]


@pytest.mark.parametrize("name", SEMANTICS)
def test_booster_follows_train_one_iter(lgb, name):
    """B200Booster against the live reference on matrices built to hit each branch of GBDT::TrainOneIter: the trees kept,
    their leaf values (rounded to zero, constant trees, bias) and the training scores.  Values are compared at rtol 1e-12
    with atol 0, not as bytes: the mean label is a pairwise sum here (np.mean) and a sequential one in the reference, so
    the init score, and every leaf and score that carries it, may differ in the last bit.  A zero must still be a zero."""
    from oracle import refapi
    if not refapi.available():
        pytest.skip("oracle/_ref not built")
    X, y, params = _semantics_case(name, np.random.default_rng(11))
    ref_trees, ref_scores = _ref_run(X, y, params, 5)
    bst = lgb.train(params, lgb.Dataset(X, label=y), num_boost_round=5)
    mine = lgb.Model.from_string(bst.to_model().to_string()).trees
    assert [t.num_leaves for t in mine] == [t.num_leaves for t in ref_trees]
    for a, b in zip(mine, ref_trees):
        np.testing.assert_allclose(a.leaf_value, b.leaf_value, rtol=1e-12, atol=0)
        assert a.shrinkage == b.shrinkage and list(a.leaf_count) == list(b.leaf_count)
    raw = bst.scores()
    if params["objective"] == "binary":        # LGBM_BoosterGetPredict returns the sigmoid of the training scores
        raw = np.array([1.0 / (1.0 + math.exp(-v)) for v in raw])
    np.testing.assert_allclose(raw, ref_scores, rtol=1e-12, atol=0)
    if name in ("first_tree_no_split", "first_tree_no_split_no_average", "later_tree_no_split", "binary_all_positive"):
        assert bst.finished
