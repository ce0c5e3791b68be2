"""Seeded cases of the bit-exact histogram and prediction tests, and a subprocess entry point for the ones that run under
a developer switch (LGBMB200_SPLIT_K, LGBMB200_DEBUG, LGBMB200_PRED_PASS: lightgbm_b200/csrc/learner.cu), so that the
setting cannot reach other tests.

    python tests/exact_worker.py <case name> <out.npz>

runs the case on cuda:0 under the caller's environment and saves what it computed; the test compares it."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

G_TOP = np.nextafter(np.float32(1), np.float32(0))      # max|g| just below 2^0: |q| = 2^30 - 64


def occupancy_data(sign, n=200_000, c=64, seed=5):
    """Worst-case occupancy: columns 0..3 put every row in stored value 0, 1, 254 and 255 (even and odd count half-word
    of the count-and-scale kernel), columns 4..11 put 90 % of the rows in one value, the rest are uniform.  Gradients of
    one sign (or mixed) with |g| at G_TOP for 90 % of the rows, so |q| is within 64 of 2^30 in the crowded cells."""
    rng = np.random.default_rng(seed)
    bins = rng.integers(0, 256, (n, c), dtype=np.uint8)
    for j, v in enumerate((0, 1, 254, 255)):
        bins[:, j] = v
    for j in range(4, 12):
        bins[rng.random(n) < 0.9, j] = (37 * j) % 256
    mag = np.where(rng.random(n) < 0.9, G_TOP, rng.random(n).astype(np.float32) * G_TOP).astype(np.float32)
    s = {"pos": 1.0, "neg": -1.0, "mixed": np.where(rng.random(n) < 0.5, 1.0, -1.0)}[sign]
    g = (mag * s).astype(np.float32)
    h = np.where(rng.random(n) < 0.9, G_TOP, rng.random(n).astype(np.float32) * G_TOP + 1e-3).astype(np.float32)
    return bins, g, h


LEAF_CASES = {
    # name: (learner config overrides, is_constant_hessian, bagging, feature mask)
    "plain": (dict(), False, False, False),
    "bagging": (dict(), False, True, False),
    "feature_mask": (dict(), False, False, True),
    "const_hess": (dict(), True, False, False),
    "quant4": (dict(use_quantized_grad=True, num_grad_quant_bins=4), False, False, False),
    "quant15": (dict(use_quantized_grad=True, num_grad_quant_bins=15), False, False, False),
    "quant16": (dict(use_quantized_grad=True, num_grad_quant_bins=16), False, False, False),
    "quant64": (dict(use_quantized_grad=True, num_grad_quant_bins=64), False, False, False),
}
LEAF_PARAMS = dict(num_leaves=31, min_data_in_leaf=1, min_sum_hessian_in_leaf=1e-3)


def leaf_data(name, n=120_000, c=40, seed=3):
    """Identity layout with skewed columns; float gradients; (bag, mask) per LEAF_CASES."""
    cfg, const_hess, bagging, masking = LEAF_CASES[name]
    rng = np.random.default_rng(seed)
    bins = rng.integers(0, 255, (n, c), dtype=np.uint8)
    bins[rng.random((n, c)) < 0.5] = 0
    bins[:, 5] = np.where(rng.random(n) < 0.97, 9, 200).astype(np.uint8)
    y = (bins[:, :6].astype(np.float64) / 127.0 - 1) @ rng.normal(size=6) + 0.3 * rng.normal(size=n)
    g = (-y).astype(np.float32)
    h = np.ones(n, np.float32) if const_hess else (rng.random(n) * 0.9 + 0.1).astype(np.float32)
    bag = np.sort(rng.choice(n, n // 2, replace=False)).astype(np.int32) if bagging else None
    mask = None
    if masking:
        mask = np.ones(c, np.uint8)
        mask[[0, 2, 17, 33]] = 0
    return bins, g, h, bag, mask, dict(LEAF_PARAMS, stochastic_rounding=False, **cfg), const_hess


def train_case(lgb, name):
    """Train the case; returns (learner, layout, tree, partition, every leaf's histogram read-back)."""
    bins, g, h, bag, mask, cfg, const_hess = leaf_data(name)
    lay = lgb.Layout.identity(bins)
    L = lgb.B200TreeLearner(lgb.Config(**cfg))
    L.init(lay, is_constant_hessian=const_hess)
    if bag is not None:
        L.set_bagging_data(bag)
    if mask is not None:
        L.set_feature_mask(mask)
    t = L.train(g, h)
    part = L.get_partition(t.num_leaves)
    hists = np.stack([L.get_leaf_histogram(i) for i in range(t.num_leaves)])
    return L, lay, t, part, hists


def predict_case(dtype, seed=31, ncol=40):
    """A 33-tree synthetic model and rows on and next to its thresholds (tests/helpers.py)."""
    import helpers as H
    rng = np.random.default_rng(seed)
    m = H.synthetic_model(rng, 33, ncol, features=[0, ncol - 1] + list(rng.integers(0, ncol, 8)))
    return m, H.boundary_matrix(H.model_columns(m, ncol, dtype == np.float64), 300, rng, dtype)


def main():
    name, out = sys.argv[1], sys.argv[2]
    import lightgbm_b200 as lgb
    if name == "predict":
        res = {}
        for dt in (np.float32, np.float64):
            m, X = predict_case(dt)
            res[np.dtype(dt).name] = m.predict_raw(X)
        np.savez(out, **res)
        return
    if name.startswith("occupancy_"):
        _, sign, kernel = name.split("_")
        bins, g, h = occupancy_data(sign)
        const = kernel == "ch"
        if const:
            h = np.full(len(g), G_TOP, np.float32)
        L = lgb.B200TreeLearner(lgb.Config(num_leaves=4))
        L.init(lgb.Layout.identity(bins, num_bin=256), is_constant_hessian=const)
        hist, _ = L.construct_histogram(g, h)
        np.savez(out, hist=hist)
        return
    _, lay, t, (lb, lc, idx), hists = train_case(lgb, name)
    np.savez(out, splits=t.splits.view(np.uint8), leaf_value=t.leaf_value, leaf_count=t.leaf_count, hists=hists,
             lb=lb, lc=lc, idx=idx)


if __name__ == "__main__":
    main()
