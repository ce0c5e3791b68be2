"""The restatements of one boosting iteration (tests/helpers.py) on the CPU: the counter-based uniforms are uniform and
independent where the device relies on it, GOSS keeps what goss.hpp keeps, the routing rule replays Tree::Split, and the
host side of the booster follows GBDT::TrainOneIter (zero band, kEpsilon gates, constant trees).  The GPU file
tests/test_gpu_boosting_exact.py holds the device to these restatements byte for byte."""
import math

import numpy as np
import pytest

import helpers as H

N = 1 << 18


def _binomial_ok(count, m, p, sigmas=6.0):
    return abs(count - m * p) <= sigmas * math.sqrt(m * p * (1 - p)) + 1


@pytest.mark.parametrize("stream", [H.QUANT_G_STREAM, H.QUANT_H_STREAM, H.GOSS_STREAM])
def test_counter_uniform_is_uniform(stream):
    u = H.counter_uniform(7, 3, np.arange(N), stream)
    assert u.min() >= 0.0 and u.max() < 1.0
    counts = np.bincount((u * 64).astype(np.int64), minlength=64)
    chi2 = float(np.sum((counts - N / 64) ** 2 / (N / 64)))
    assert chi2 < 150, chi2                                           # 63 degrees of freedom: p ~ 1e-8


def test_counter_uniform_independent_values():
    """Every (row, stream) pair has its own counter, and different iterations and seeds give different sequences."""
    rows = np.arange(N)
    u = {s: H.counter_uniform(7, 3, rows, s) for s in (H.QUANT_G_STREAM, H.QUANT_H_STREAM, H.GOSS_STREAM)}
    allv = np.concatenate(list(u.values()))
    assert len(np.unique(allv)) == len(allv)                          # no two (row, stream) share a value
    for a, b in ((H.QUANT_G_STREAM, H.GOSS_STREAM), (H.QUANT_H_STREAM, H.GOSS_STREAM), (H.QUANT_G_STREAM, H.QUANT_H_STREAM)):
        assert abs(np.corrcoef(u[a], u[b])[0, 1]) < 0.02
    assert abs(np.corrcoef(u[H.GOSS_STREAM], H.counter_uniform(7, 4, rows, H.GOSS_STREAM))[0, 1]) < 0.02
    assert abs(np.corrcoef(u[H.GOSS_STREAM], H.counter_uniform(8, 3, rows, H.GOSS_STREAM))[0, 1]) < 0.02
    # seed and iteration are 32-bit on the device
    assert np.array_equal(H.counter_uniform(7 + (1 << 32), 3, rows[:64], 0), u[0][:64])


@pytest.mark.parametrize("p", [0.5, 0.1, 0.02])
def test_counter_uniform_pairs_are_drawn_independently(p):
    """Rows 2k and 2k + 1 are both drawn at rate p^2 within a binomial bound (a draw shared by the pair gives p)."""
    u = H.counter_uniform(7, 3, np.arange(N), H.GOSS_STREAM) < p
    both = int(np.sum(u[0::2] & u[1::2]))
    assert _binomial_ok(both, N // 2, p * p), (both, N // 2 * p * p)
    assert _binomial_ok(int(u.sum()), N, p)


def test_goss_reference_ties_and_rates():
    rng = np.random.default_rng(1)
    n = 1000
    g = rng.choice(np.float32([0.5, 1.0, 2.0]), n).astype(np.float32)
    h = np.ones(n, np.float32)
    bag, g2, h2 = H.goss_reference(g, h, 0.1, 0.2, seed=3, iteration=5)
    # 10% top: the threshold is 2.0, and every row holding 2.0 (a third of them) is kept as is
    top = g == 2.0
    assert top.sum() > 100 and np.all(np.isin(np.nonzero(top)[0], bag))
    assert np.array_equal(g2[top], g[top])
    drawn = np.setdiff1d(bag, np.nonzero(top)[0])
    mult = np.float32(n - 100) / np.float32(200)
    assert np.array_equal(g2[drawn], g[drawn] * mult) and np.array_equal(h2[drawn], h[drawn] * mult)
    rest = np.setdiff1d(np.arange(n), drawn)
    assert np.array_equal(g2[rest], g[rest])
    assert np.all(np.diff(bag) > 0)
    # top_k = n keeps everything unscaled
    bag, g2, h2 = H.goss_reference(g, h, 1.0, 0.0, seed=3, iteration=5)
    assert np.array_equal(bag, np.arange(n)) and np.array_equal(g2, g)
    # top_k floored to 1, other_k = 0: the largest key only (all its ties)
    g1 = np.arange(n, dtype=np.float32)
    bag, _, _ = H.goss_reference(g1, h, 0.0001, 0.0005, seed=3, iteration=5)
    assert list(bag) == [n - 1]
    # all keys equal: the threshold is that key, every row is kept
    bag, _, _ = H.goss_reference(np.ones(n, np.float32), h, 0.2, 0.1, seed=3, iteration=5)
    assert len(bag) == n


def test_route_rows_reference_replays_splits():
    from lightgbm_b200.tree_learner import SPLIT_DTYPE, Layout
    rng = np.random.default_rng(2)
    bins = rng.integers(0, 8, (500, 3), dtype=np.uint8)
    lay = Layout.identity(bins, num_bin=8)
    sp = np.zeros(3, SPLIT_DTYPE)
    sp[0] = (0, 0, 3, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0)        # leaf 0: col 0 <= 3 stays, else leaf 1
    sp[1] = (1, 1, 5, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0)        # leaf 1: col 1 <= 5 stays, else leaf 2
    sp[2] = (0, 2, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0)        # leaf 0: col 2 <= 0 stays, else leaf 3
    want = np.where(bins[:, 0] <= 3, np.where(bins[:, 2] <= 0, 0, 3), np.where(bins[:, 1] <= 5, 1, 2))
    assert np.array_equal(H.route_rows_reference(lay, sp), want)
    bag = np.arange(0, 500, 3)
    got = H.route_rows_reference(lay, sp, bag)
    assert np.array_equal(got[bag], want[bag]) and np.all(np.delete(got, bag) == -1)
    s = rng.normal(size=500)
    lv = np.array([0.5, -1.0, 2.0, 1e-300])
    out = H.boost_step_reference(s, lv, got)
    assert np.array_equal(out[bag], s[bag] + lv[want[bag]]) and np.array_equal(np.delete(out, bag), np.delete(s, bag))


def test_binary_gradients_reference_overflow_and_signs():
    s = np.array([0.0, -0.0, 800.0, -800.0, 30.0, -30.0])
    g, h = H.binary_gradients_reference(s, np.float32([1, 0, 1, 1, 0, 0]), 1.0)
    assert g[0] == np.float32(-0.5) and g[1] == np.float32(0.5) and h[0] == np.float32(0.25)
    assert g[2] == 0.0 and h[2] == 0.0                                 # exp(800) overflows: response -0
    assert g[3] == np.float32(-1.0)
    g2, _ = H.l2_gradients_reference(np.array([1.0 + 2 ** -40]), np.float32([1.0]))
    assert g2[0] == np.float32(2 ** -40)                              # the difference is taken in double


def test_tree_shrinkage_and_bias_round_to_zero():
    """Tree::Shrinkage / AddBias send leaf values in the zero band to 0 (what the model text holds), so the score update
    adds the same values the model predicts."""
    from lightgbm_b200.tree_learner import SPLIT_DTYPE, Tree
    t = Tree(3, np.zeros(2, SPLIT_DTYPE), np.array([1e-34, -5e-35, 2.0]), np.ones(3), np.ones(3, np.int32), np.ones(3, np.int32), 0.0, 3.0)
    t.shrinkage(0.1)
    assert t.leaf_value[0] == 0.0 and t.leaf_value[1] == 0.0 and t.leaf_value[2] == 2.0 * 0.1
    t.leaf_value = np.array([1e-35, 1.0, -2.0])
    t.add_bias(-1.0)
    assert list(t.leaf_value) == [-1.0, 0.0, -3.0]
    t.as_constant(0.25, 77)
    assert t.num_leaves == 1 and list(t.leaf_value) == [0.25] and list(t.leaf_count) == [77] and t.shrink == 1.0
