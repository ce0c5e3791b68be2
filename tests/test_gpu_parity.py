"""GPU parity tests proper: the CUDA path (through the C-ABI of include/lgbm_b200.h) against the oracle
(oracle/lgbm_oracle.c, itself pinned against the compiled reference) on identical binned input.

Tolerance (stated, SURVEY.md §8d / reference test_dual.py:35-36): the WHOLE split sequence exact unless the oracle's
own best-vs-runner-up margin at the first differing split is below 1e-5 relative (helpers.compare_trees); gains /
sums / leaf values within rel 1e-5.  The histogram kernel sums 30-bit fixed-point gradients exactly (int32 hi/lo
shared-memory atomics -> int64 pool): histograms must EQUAL helpers.fixed_point_hist, and differ from the oracle's fp64
sums by at most the one rounding per row, 2^-(k+1) per row of the cell."""
import numpy as np
import pytest

from helpers import assert_hist_equal, cell_counts, compare_trees, fixed_point_hist, synth_identity

pytestmark = pytest.mark.gpu

RTOL = 1e-5


@pytest.fixture(scope="module")
def mods(built_lib):
    import lightgbm_b200 as lgb
    from oracle import oracle_py
    return lgb, oracle_py


def _learner(lgb, lay, const_hess=False, **cfg):
    """const_hess=True selects the count-and-scale histogram kernel (Init's is_constant_hessian), else general hessians."""
    L = lgb.B200TreeLearner(lgb.Config(**cfg))
    L.init(lay, is_constant_hessian=const_hess)
    return L


@pytest.mark.parametrize("n,f,nidx", [(20000, 40, None), (50000, 33, 12345), (3000, 5, 700), (100, 64, 33), (257, 1, None)])
def test_histogram_matches_oracle(mods, n, f, nidx):
    lgb, orc = mods
    bins, y, g, h = synth_identity(n, f, seed=n + f)
    h = (np.abs(np.random.default_rng(1).normal(size=n)) + 0.1).astype(np.float32)
    lay = lgb.Layout.identity(bins)
    L = _learner(lgb, lay, num_leaves=4)
    idx = None if nidx is None else np.sort(np.random.default_rng(7).choice(n, nidx, replace=False)).astype(np.int32)
    got, ms = L.construct_histogram(g, h, idx)
    # every cell IS the exact sum of the rows' fixed-point values (integer arithmetic end to end)
    _, exact, (kg, kh) = fixed_point_hist(bins, idx, g, h)
    assert_hist_equal(got, exact, "general-hessian kernel")
    # and the fixed point rounds each row once: within count * 2^-(k+1) of the oracle's fp64 sums
    want = orc.construct_histogram(lay, idx, g, h)
    cnt = cell_counts(bins, idx)
    assert (np.abs(got[..., 0] - want[..., 0]) <= cnt * 2.0 ** -(kg + 1)).all()
    assert (np.abs(got[..., 1] - want[..., 1]) <= cnt * 2.0 ** -(kh + 1)).all()


@pytest.mark.parametrize("n,f,nidx", [(20000, 40, None), (50000, 70, 12345), (100, 64, 33), (70000, 33, None), (257, 1, None)])
def test_constant_hessian_histogram_matches_oracle(mods, n, f, nidx):
    """The count-and-scale kernel (two column groups per CTA, 16-bit packed counts): hessian entries are exactly
    count * h0; gradient entries are exact sums of 30-bit fixed-point values."""
    lgb, orc = mods
    bins, y, g, h = synth_identity(n, f, seed=n + 3 * f)
    h = np.full(n, 0.7, np.float32)
    lay = lgb.Layout.identity(bins)
    L = _learner(lgb, lay, const_hess=True, num_leaves=4)
    idx = None if nidx is None else np.sort(np.random.default_rng(7).choice(n, nidx, replace=False)).astype(np.int32)
    got, ms = L.construct_histogram(g, h, idx)
    _, exact, (kg, kh) = fixed_point_hist(bins, idx, g, h, const_hess=True)
    assert_hist_equal(got, exact, "constant-hessian kernel")     # hessian cells: count * llrint(h0 * 2^kh) exactly
    want = orc.construct_histogram(lay, idx, g, h)
    cnt = cell_counts(bins, idx)
    assert (np.abs(got[..., 0] - want[..., 0]) <= cnt * 2.0 ** -(kg + 1)).all()
    assert (np.abs(got[..., 1] - want[..., 1]) <= cnt * 2.0 ** -(kh + 1)).all()


def test_histogram_is_deterministic(mods):
    lgb, _ = mods
    bins, y, g, h = synth_identity(40000, 48, seed=3)
    L = _learner(lgb, lgb.Layout.identity(bins), num_leaves=4)
    a, _ = L.construct_histogram(g, h)
    b, _ = L.construct_histogram(g, h)
    assert np.array_equal(a, b)       # bitwise: fixed summation order + integer merge


@pytest.mark.parametrize("const_hess", [False, True])
@pytest.mark.parametrize("n,f,leaves,kw", [
    (20000, 16, 31, {}),
    (50000, 40, 63, {}),
    (8000, 7, 15, dict(min_data_in_leaf=5)),
    (30000, 24, 31, dict(lambda_l2=3.0, lambda_l1=0.5)),
    (30000, 24, 31, dict(max_depth=4)),
    (30000, 24, 31, dict(min_gain_to_split=50.0)),
    (30000, 24, 31, dict(path_smooth=10.0, max_delta_step=0.7)),
    (500, 3, 8, dict(min_data_in_leaf=20)),
])
def test_tree_matches_oracle(mods, n, f, leaves, kw, const_hess):
    lgb, orc = mods
    bins, y, g, h = synth_identity(n, f, seed=11 * n + f)       # h == 1: both histogram kernels apply
    lay = lgb.Layout.identity(bins)
    L = _learner(lgb, lay, const_hess=const_hess, num_leaves=leaves, **kw)
    t = L.train(g, h)
    o = orc.train_tree(lay_for_oracle(lay), g, h, num_leaves=leaves, **kw)
    matched, diverged = compare_trees(t, o, RTOL)
    assert diverged or matched == o.num_leaves - 1
    if not diverged:
        # partition: same rows, same (stable) order in every leaf
        lb, lc, idx = L.get_partition(t.num_leaves)
        for leaf in range(t.num_leaves):
            np.testing.assert_array_equal(idx[lb[leaf]:lb[leaf] + lc[leaf]],
                                          o.indices[o.leaf_begin[leaf]:o.leaf_begin[leaf] + o.leaf_count[leaf]])


def lay_for_oracle(lay):
    return lay        # oracle_py.make_layout derives feat_in_group when the layout has none


def test_non_constant_hessian_and_graph_replay(mods):
    lgb, orc = mods
    n, f = 40000, 20
    bins, y, g, h = synth_identity(n, f, seed=5)
    rng = np.random.default_rng(9)
    p = 1 / (1 + np.exp(-rng.normal(size=n)))
    yb = (rng.random(n) < 1 / (1 + np.exp(-(bins[:, 0] / 127.0 - 1) * 2))).astype(np.float32)
    g = (p - yb).astype(np.float32); h = (p * (1 - p)).astype(np.float32)
    lay = lgb.Layout.identity(bins)
    L = _learner(lgb, lay, num_leaves=31)
    o = orc.train_tree(lay_for_oracle(lay), g, h, num_leaves=31)
    t1 = L.train(g, h)
    t2 = L.train(g, h)           # second call replays the captured CUDA graph
    assert np.array_equal(t1.splits, t2.splits) and np.array_equal(t1.leaf_value, t2.leaf_value)
    matched, diverged = compare_trees(t1, o, RTOL)
    assert diverged or matched == o.num_leaves - 1


def test_bagging_and_feature_mask(mods):
    lgb, orc = mods
    n, f = 30000, 12
    bins, y, g, h = synth_identity(n, f, seed=21)
    lay = lgb.Layout.identity(bins)
    rng = np.random.default_rng(2)
    bag = np.sort(rng.choice(n, n // 2, replace=False)).astype(np.int32)
    mask = np.ones(f, np.uint8); mask[[0, 3]] = 0
    L = _learner(lgb, lay, num_leaves=15)
    L.set_bagging_data(bag)
    L.set_feature_mask(mask)
    t = L.train(g, h)
    o = orc.train_tree(lay_for_oracle(lay), g, h, bag_indices=bag, feature_used=mask, num_leaves=15)
    matched, diverged = compare_trees(t, o, RTOL)
    assert diverged or matched == o.num_leaves - 1
    assert not np.isin(t.splits["feature"], [0, 3]).any()
    L.set_bagging_data(None); L.set_feature_mask(None)
    t_all = L.train(g, h)
    o_all = orc.train_tree(lay_for_oracle(lay), g, h, num_leaves=15)
    compare_trees(t_all, o_all, RTOL)


def test_add_prediction_to_score_host_and_device(mods):
    lgb, orc = mods
    n, f = 25000, 10
    bins, y, g, h = synth_identity(n, f, seed=8)
    lay = lgb.Layout.identity(bins)
    L = _learner(lgb, lay, num_leaves=31)
    t = L.train(g, h)
    lb, lc, idx = L.get_partition(t.num_leaves)
    want = np.zeros(n)
    for leaf in range(t.num_leaves):
        want[idx[lb[leaf]:lb[leaf] + lc[leaf]]] += t.leaf_value[leaf]
    score = np.zeros(n)
    L.add_prediction_to_score(t, score)
    np.testing.assert_array_equal(score, want)
    from lightgbm_b200.tree_learner import DeviceArray
    d = DeviceArray(n * 8).upload(np.zeros(n))
    L.add_prediction_to_score(t, d)
    np.testing.assert_array_equal(d.download(np.float64, n), want)
    assert sorted(idx.tolist()) == list(range(n))     # every row in exactly one leaf


def test_booster_device_resident_equals_host_mode(mods):
    lgb, _ = mods
    n, f = 30000, 16
    bins, y, g, h = synth_identity(n, f, seed=13)
    lay = lgb.Layout.identity(bins)
    cfg = lgb.Config(num_leaves=15)
    a = lgb.B200Booster(lay, y, cfg, learning_rate=0.1, device_resident=True)
    b = lgb.B200Booster(lay, y, cfg, learning_rate=0.1, device_resident=False)
    l0 = a.l2()
    for _ in range(5):
        ta, tb = a.update(), b.update()
        assert np.array_equal(ta.splits[["leaf", "feature", "threshold"]], tb.splits[["leaf", "feature", "threshold"]])
    np.testing.assert_allclose(a.scores(), b.scores(), rtol=1e-6, atol=1e-9)
    assert a.l2() < l0 * 0.8
    assert a.learner.kernel_launches > 0


def test_leaf_index_bagging_host_score_and_profiling(mods):
    lgb, orc = mods
    n, f = 20000, 9
    bins, y, g, h = synth_identity(n, f, seed=31)
    lay = lgb.Layout.identity(bins)
    L = _learner(lgb, lay, num_leaves=15)
    bag = np.sort(np.random.default_rng(4).choice(n, n // 3, replace=False)).astype(np.int32)
    L.set_bagging_data(bag)
    t = L.train(g, h)
    li = L.get_leaf_index()
    assert (li[bag] >= 0).all() and (np.delete(li, bag) == -1).all()       # rows outside the bag are in no leaf
    lb, lc, idx = L.get_partition(t.num_leaves)
    for leaf in range(t.num_leaves):
        assert (li[idx[lb[leaf]:lb[leaf] + lc[leaf]]] == leaf).all()
    score = np.zeros(n)
    L.add_prediction_to_score(t, score)                                     # host path: leaf ids D2H + host add
    want = np.where(li >= 0, t.leaf_value[np.maximum(li, 0)], 0.0)
    np.testing.assert_array_equal(score, want)
    # profiling mode (no CUDA graph) grows the identical tree and reports per-kernel times
    L.set_bagging_data(None)
    t_graph = L.train(g, h)
    L.set_profiling(True); L.hist_stats(reset=True)
    t_prof = L.train(g, h)
    L.set_profiling(False)
    assert np.array_equal(t_graph.splits, t_prof.splits) and np.array_equal(t_graph.leaf_value, t_prof.leaf_value)
    ms, rows, nl = L.hist_stats()
    kinds = L.profile_by_kind()
    assert ms > 0 and rows >= n and nl >= 1 and kinds["hist"] > 0 and kinds["scan"] > 0 and kinds["part_flags"] > 0
    L.timer_start(); L.train(g, h); assert L.timer_stop() > 0


def test_row_major_partition_path_matches_column_major(mods):
    """LGBMB200_Config.reserved bit 0 drops the column-major copy; both partition paths must agree."""
    lgb, _ = mods
    import ctypes as C
    from lightgbm_b200 import tree_learner as TL
    n, f = 30000, 20
    bins, y, g, h = synth_identity(n, f, seed=77)
    lay = lgb.Layout.identity(bins)
    a = _learner(lgb, lay, num_leaves=31)
    ta = a.train(g, h)
    cfg = lgb.Config(num_leaves=31)
    orig = cfg.to_c

    def to_c_no_t():
        c = orig(); c.reserved = 1; return c
    cfg.to_c = to_c_no_t
    b = lgb.B200TreeLearner(cfg); b.init(lay)
    tb = b.train(g, h)
    assert np.array_equal(ta.splits, tb.splits) and np.array_equal(ta.leaf_count, tb.leaf_count)


def test_binary_objective_device_resident_equals_host_mode(mods):
    """Binary logloss gradients on the device (binary_objective.hpp:105-121) vs the numpy host path."""
    lgb, _ = mods
    n, f = 30000, 12
    bins, _, _, _ = synth_identity(n, f, seed=41)
    rng = np.random.default_rng(3)
    y = (rng.random(n) < 1 / (1 + np.exp(-((bins[:, 0] / 127.0 - 1) * 2 - (bins[:, 1] / 127.0 - 1))))).astype(np.float32)
    lay = lgb.Layout.identity(bins)
    cfg = lgb.Config(num_leaves=15)
    a = lgb.B200Booster(lay, y, cfg, learning_rate=0.2, device_resident=True, objective="binary")
    b = lgb.B200Booster(lay, y, cfg, learning_rate=0.2, device_resident=False, objective="binary")
    l0 = a.logloss()
    for _ in range(6):
        ta, tb = a.update(), b.update()
        assert np.array_equal(ta.splits[["leaf", "feature", "threshold"]], tb.splits[["leaf", "feature", "threshold"]])
    np.testing.assert_allclose(a.scores(), b.scores(), rtol=1e-5, atol=1e-7)
    assert a.logloss() < l0 * 0.9
