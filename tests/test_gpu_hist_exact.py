"""Bit-exact histograms.  k_hist_a + k_hist_reduce (and k_hist_q for quantized training) sum fixed-point integers, so
every cell the learner reports must EQUAL helpers.fixed_point_hist (quantized: the integer sums of the discretized
values) — no tolerance.  The cases are chosen by the path they take through the kernels:

  * explicit hook (construct_histogram), both kernels, C across the 32- and 64-column group boundaries and N across
    the 32-row stage, the 65 504-row flush interval and a multi-flush size: identity rows (TMA tiles when N >= 32,
    gathered otherwise) and sorted subsets (gathered rows);
  * worst-case occupancy: every row in one stored value (0, 1, 254, 255) with |q| within 64 of 2^30, with the default
    work split and with one CTA per column-group set walking all 200 000 rows (three full flush intervals);
  * every leaf after Train: root and smaller children come from the kernel over the leaf-ordered (g, h) copies,
    larger children from k_scan's in-place parent - smaller;
  * the developer switches (no TMA, no packed quantized kernel, no leaf-ordered copies) give the same bits."""
import os
import subprocess
import sys

import numpy as np
import pytest

from exact_worker import G_TOP, LEAF_CASES, LEAF_PARAMS, leaf_data, occupancy_data, train_case
from helpers import assert_hist_equal, cell_counts, fixed_point_hist, int_hist

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
FLUSH_ROWS = 65504          # kAFlushRows (hist_atom_kernel.cuh)


@pytest.fixture(scope="module")
def lgb(built_lib):
    import lightgbm_b200
    return lightgbm_b200


def _run_worker(case, tmp_path, env_extra):
    out = str(tmp_path / f"{case}.npz")
    env = dict(os.environ, **env_extra)
    r = subprocess.run([sys.executable, os.path.join(HERE, "exact_worker.py"), case, out], env=env,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    return dict(np.load(out))


# ---------------------------------------------------------------------------------------------------- explicit hook

@pytest.mark.parametrize("n", [1, 31, 32, 33, 1000, 65504, 65505, 200_001])
@pytest.mark.parametrize("c", [1, 31, 32, 33, 63, 64, 65, 127, 128, 129, 200])
def test_explicit_hook_bit_exact(lgb, c, n):
    """Both kernels (general hessian: one 32-column group per CTA; constant hessian: two), identity rows and a sorted
    subset, against the exact fixed point.  The scale comes from all N rows also for the subset."""
    rng = np.random.default_rng(1000 * c + n)
    bins = rng.integers(0, 256, (n, c), dtype=np.uint8)
    g = (rng.normal(size=n) * 2).astype(np.float32)
    h = (rng.random(n) + 0.01).astype(np.float32)
    hc = np.full(n, 0.7, np.float32)
    lay = lgb.Layout.identity(bins, num_bin=256)
    subset = np.sort(rng.choice(n, max(1, n // 2), replace=False)).astype(np.int32)
    for const in (False, True):
        L = lgb.B200TreeLearner(lgb.Config(num_leaves=4))
        L.init(lay, is_constant_hessian=const)
        hh = hc if const else h
        for rows in (None, subset):
            got, _ = L.construct_histogram(g, hh, rows)
            _, want, _ = fixed_point_hist(bins, rows, g, hh, const_hess=const)
            assert_hist_equal(got, want, f"C={c} N={n} const_hess={const} rows={'identity' if rows is None else len(rows)}")
        L.free()


# ---------------------------------------------------------------------------------------------- worst-case occupancy

def _check_occupancy(hist, sign, kernel):
    bins, g, h = occupancy_data(sign)
    const = kernel == "ch"
    if const:
        h = np.full(len(g), G_TOP, np.float32)
    sums, want, (kg, _) = fixed_point_hist(bins, None, g, h, const_hess=const)
    # the path was reached: whole columns in one cell (>= 3 flush intervals of rows), |q| within 64 of 2^30
    assert cell_counts(bins)[:4, [0, 1, 254, 255]].diagonal().min() >= 3 * FLUSH_ROWS
    assert kg == 30 and int(np.rint(np.ldexp(np.float64(G_TOP), kg))) == 2 ** 30 - 64
    assert_hist_equal(hist, want, f"occupancy sign={sign} kernel={kernel}")


@pytest.mark.parametrize("kernel", ["general", "ch"])
@pytest.mark.parametrize("sign", ["pos", "neg", "mixed"])
def test_worst_case_occupancy_default_split(lgb, sign, kernel):
    """Default work split: many CTAs per set; the crowded cells are summed from many scratch blocks."""
    bins, g, h = occupancy_data(sign)
    const = kernel == "ch"
    if const:
        h = np.full(len(g), G_TOP, np.float32)
    L = lgb.B200TreeLearner(lgb.Config(num_leaves=4))
    L.init(lgb.Layout.identity(bins, num_bin=256), is_constant_hessian=const)
    hist, _ = L.construct_histogram(g, h)
    _check_occupancy(hist, sign, kernel)


@pytest.mark.parametrize("kernel", ["general", "ch"])
@pytest.mark.parametrize("sign", ["pos", "neg", "mixed"])
def test_worst_case_occupancy_one_cta_per_set(tmp_path, built_lib, sign, kernel):
    """LGBMB200_SPLIT_K=1e-9 leaves one CTA group per set group, so ONE CTA takes all 200 000 rows of its set: it
    fills a cell with exactly 65 504 rows three times (count half-word, |hi| * rows and the wrapping lo sum at their
    limits) and flushes after each interval."""
    n = occupancy_data(sign)[0].shape[0]
    assert n // FLUSH_ROWS >= 3
    out = _run_worker(f"occupancy_{sign}_{kernel}", tmp_path, {"LGBMB200_SPLIT_K": "1e-9"})
    _check_occupancy(out["hist"], sign, kernel)


# ------------------------------------------------------------------------------------------- every leaf after Train

def leaf_plan(tree, num_leaves_cfg, min_data_in_leaf, max_depth=-1):
    """Which pool slots hold a leaf's histogram when Train returns (learner.cu EnqueueTree, partition_kernel.cuh
    k_part_scatter, scan_kernel.cuh k_scan).  Split i of leaf p makes children p (left) and i + 1 (right); the child
    with fewer rows (the right one on equal counts) is histogrammed by the kernel into a new slot, which holds every
    cell of every column; the other child keeps the parent's slot, which k_scan rewrites in place as parent - smaller on
    the slice of every feature it scans for the parent (unmasked, and splittable in the parent).  The children of the
    last split a full tree makes (split num_leaves - 2), and both children of a split where BeforeFindBestSplit said no
    (max_depth, or both children under 2 * min_data_in_leaf), are never histogrammed.

    Returns {leaf: (role, parent_leaves)}: role 'smaller' / 'larger', parent_leaves = the final leaves under the
    parent (its rows)."""
    class Node:
        def __init__(self, depth):
            self.kids, self.leaf, self.depth = None, None, depth

        def leaves(self):
            return [self.leaf] if self.kids is None else self.kids[0].leaves() + self.kids[1].leaves()

    root = Node(0)
    cur = {0: root}
    made = {}
    for i, s in enumerate(tree.splits):
        p = cur[int(s["leaf"])]
        l, r = Node(p.depth + 1), Node(p.depth + 1)
        p.kids = (l, r)
        cur[int(s["leaf"])], cur[i + 1] = l, r
        lc, rc = int(s["left_count"]), int(s["right_count"])
        do_find = not (max_depth > 0 and p.depth + 1 >= max_depth) and not (lc < 2 * min_data_in_leaf and rc < 2 * min_data_in_leaf)
        hist = do_find and i < num_leaves_cfg - 2
        left_smaller = lc < rc
        made[int(s["leaf"])] = (hist, "smaller" if left_smaller else "larger", p)
        made[i + 1] = (hist, "larger" if left_smaller else "smaller", p)
    for leaf, node in cur.items():
        node.leaf = leaf
    plan = {}
    for leaf, (hist, role, p) in made.items():
        if hist:
            plan[leaf] = (role, p.leaves())
    return plan


def check_leaf_histograms(bins, tree, part, hists, want_fn, cfg, mask=None, nslice=254, lo=1):
    """Compare every valid slot with want_fn(rows); returns the number of leaves checked."""
    lb, lc, idx = part
    rows = [np.sort(idx[lb[i]:lb[i] + lc[i]]) for i in range(tree.num_leaves)]
    plan = leaf_plan(tree, cfg["num_leaves"], cfg.get("min_data_in_leaf", 20), cfg.get("max_depth", -1))
    C = bins.shape[1]
    mm = {}
    for leaf in range(tree.num_leaves):
        b = bins[rows[leaf]]
        mm[leaf] = (b.min(axis=0), b.max(axis=0)) if len(b) else (np.full(C, 255), np.zeros(C))
    checked = 0
    for leaf, (role, parent_leaves) in plan.items():
        want = want_fn(rows[leaf])
        if role == "smaller":
            assert_hist_equal(hists[leaf], want, f"leaf {leaf} (smaller child: kernel)")
        else:
            pmin = np.min([mm[q][0] for q in parent_leaves], axis=0)
            pmax = np.max([mm[q][1] for q in parent_leaves], axis=0)
            # splittable in the parent: with min_data_in_leaf = 1, any feature with two distinct values in the parent
            # (a split of random float gradients with exactly zero gain improvement does not occur)
            feats = [f for f in range(C) if pmin[f] != pmax[f] and (mask is None or mask[f])]
            assert feats
            got, exp = hists[leaf][feats, lo:lo + nslice], want[feats, lo:lo + nslice]
            assert_hist_equal(got, exp, f"leaf {leaf} (larger child: parent - smaller)")
        checked += 1
    return checked


def _want_fn(name, bins, g, h, bag, const_hess, cfg):
    if cfg.get("use_quantized_grad"):
        from oracle import oracle_py
        qg, qh, _, _ = oracle_py.discretize(g, h, cfg["num_grad_quant_bins"], const_hess)
        return lambda rows: int_hist(bins, rows, qg.astype(np.int64), qh.astype(np.int64))
    return lambda rows: fixed_point_hist(bins, rows, g, h, const_hess=const_hess)[1]


@pytest.mark.parametrize("name", list(LEAF_CASES))
def test_every_leaf_histogram_after_train(lgb, name):
    """Root / smaller children: kernel over the leaf-ordered (g, h) copies and the gathered rows (k_hist_q for
    quantized training with <= 15 bins, k_hist_a otherwise).  Larger children: parent - smaller in int64."""
    bins, g, h, bag, mask, cfg, const_hess = leaf_data(name)
    L, lay, t, part, hists = train_case(lgb, name)
    assert t.num_leaves == LEAF_PARAMS["num_leaves"]
    checked = check_leaf_histograms(bins, t, part, hists, _want_fn(name, bins, g, h, bag, const_hess, cfg), cfg, mask)
    # a full 31-leaf tree: 29 splits whose children were histogrammed, most of their children still leaves
    assert checked >= 10, checked


_DEFAULT_RUNS = {}


@pytest.mark.parametrize("bits", [2, 64, 256])
def test_developer_switches_same_bits(tmp_path, built_lib, bits):
    """LGBMB200_DEBUG=2 (no TMA staging), 64 (quantized training without the packed-cell kernel), 256 (no leaf-ordered
    (g, h) copies: gathered by row id) grow the same trees with the same histograms, bit for bit."""
    from lightgbm_b200.tree_learner import SPLIT_DTYPE

    class _T:
        pass
    for name in ("plain", "bagging", "const_hess", "quant4"):
        if name not in _DEFAULT_RUNS:
            _DEFAULT_RUNS[name] = _run_worker(name, tmp_path, {"LGBMB200_DEBUG": "0"})
        a = _DEFAULT_RUNS[name]
        b = _run_worker(name, tmp_path, {"LGBMB200_DEBUG": str(bits)})
        assert np.array_equal(a["splits"], b["splits"]), name
        assert np.array_equal(a["leaf_value"], b["leaf_value"]) and np.array_equal(a["idx"], b["idx"]), name
        cfg = leaf_data(name)[5]
        t = _T()
        t.splits = a["splits"].view(SPLIT_DTYPE)
        t.num_leaves = len(t.splits) + 1
        plan = leaf_plan(t, cfg["num_leaves"], cfg["min_data_in_leaf"])
        assert len(plan) >= 10
        for leaf in plan:        # every slot that holds a leaf's histogram (both roles)
            assert_hist_equal(b["hists"][leaf], a["hists"][leaf], f"{name} leaf {leaf} DEBUG={bits}")
