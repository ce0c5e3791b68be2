"""The plain restatements of the value -> bin pass and of prediction (tests/helpers.py) against the reference, CPU only.

tests/test_gpu_boundary_exact.py holds the device kernels to these restatements bit for bit on inputs that sit on and next
to every bin bound and threshold.  Here the restatements themselves are pinned: they reproduce every stored byte of the
reference-built binning fixtures and every raw score of the reference-trained model fixtures, and, where oracle/_ref is
built, the live reference agrees with them on the adversarial matrices, including values inside the zero band."""
import ctypes as C
import glob
import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import helpers as H  # noqa: E402

BIN_GOLD = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "binning_*.npz")))
MODEL_GOLD = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "model_*.npz")))
TREE_COUNTS = (1, 2, 15, 16, 17, 31, 32, 33)


def _fixture_meta(d):
    meta = dict(num_columns=int(d["dims"][1]), num_features=int(d["dims"][2]), feat_column=d["feat_column"], feat_lo=d["feat_lo"],
                feat_num_bin=d["feat_num_bin"], feat_most_freq_bin=d["feat_mfb"], feat_missing_type=d["feat_missing"],
                feat_real_index=d["feat_real_index"])
    ub, o = [], 0
    for nb in d["feat_num_bin"]:
        ub.append(d["ub_concat"][o:o + nb]); o += nb
    return meta, ub


def test_fixture_counts():
    assert len(BIN_GOLD) == 11 and len(MODEL_GOLD) == 5


@pytest.mark.parametrize("path", BIN_GOLD, ids=[os.path.basename(p)[8:-4] for p in BIN_GOLD])
def test_value_to_bin_restatement_reproduces_the_reference_bytes(path):
    d = np.load(path)
    meta, ub = _fixture_meta(d)
    got = H.value_to_bin_reference(d["X"], meta, ub)
    assert got.tobytes() == np.ascontiguousarray(d["bins"]).tobytes()


@pytest.mark.parametrize("path", MODEL_GOLD, ids=[os.path.basename(p)[6:-4] for p in MODEL_GOLD])
def test_predict_restatement_reproduces_the_reference_scores(path):
    from lightgbm_b200.model import Model
    d = np.load(path)
    m = Model.from_string(bytes(d["model"]).decode())
    assert H.predict_raw_reference(m, d["X"]).tobytes() == d["raw"].tobytes()
    assert H.predict_raw_reference(m, d["X"].astype(np.float64)).tobytes() == d["raw"].tobytes()


def test_generators_cover_the_depth_edges_and_the_tree_shapes():
    """The binner features reach every searchable-bound count of BOUND_COUNTS; the synthetic trees include 254-deep chains
    and single leaves; the stump grid puts every threshold under all six decision types."""
    rng = np.random.default_rng(1)
    X = H.binner_fit_matrix(rng)
    assert X.shape[1] == len(H.BOUND_COUNTS) + 5
    m = H.synthetic_model(rng, 8, 10)
    depth = []
    for t in m.trees:
        d = np.zeros(max(t.num_leaves - 1, 1), np.int64)
        for i in range(t.num_leaves - 1):
            for c in (t.left_child[i], t.right_child[i]):
                if c >= 0:
                    d[c] = d[i] + 1
        depth.append(int(d.max()) + 1 if t.num_leaves > 1 else 0)
    assert 254 in depth and 0 in depth
    pool = H.threshold_pool(rng)
    g = H.stump_grid_model(pool, 7)
    assert len(g.trees) == 6 * len(pool)
    assert {int(t.decision_type[0]) for t in g.trees} == {0, 2, 4, 6, 8, 10}


# ---------------------------------------------------------------------------------------------------- live reference
def _ref():
    from oracle import refapi
    if not refapi.available():
        pytest.skip("oracle/_ref not built")
    return refapi


def test_zero_band_threshold_goes_where_the_reference_sends_it():
    """A row whose value is exactly -kZeroThreshold at a node with threshold -kZeroThreshold: LGBM_BoosterPredictForMat
    reads the value as 0.0 and goes right, where a plain `x <= t` would go left.  The same for a threshold of 0 and a value
    just above it inside the band (left, where the plain compare goes right)."""
    refapi = _ref()
    for t, x, want in ((-H.K_ZERO, -H.K_ZERO, "right"), (0.0, 5e-36, "left"), (float(np.nextafter(-H.K_ZERO, 0.0)), -H.K_ZERO, "right")):
        for dt in (0, 2, 8, 10):                    # missing type None / NaN, both default directions
            m = H.text_model([H.stump_grid_model([t], 1).trees[0]], 1)
            m.trees[0].decision_type[0] = dt
            m = H.text_model(m.trees, 1)
            leaf = {"left": m.trees[0].leaf_value[0], "right": m.trees[0].leaf_value[1]}
            plain = leaf["left"] if x <= t else leaf["right"]
            loaded = refapi.RefLoadedBooster(m.to_string())
            for dtype in (np.float32, np.float64):
                X = np.array([[x]], dtype)
                ref = loaded.predict(X)[0]
                assert ref == leaf[want] != plain, (t, x, dt, dtype)
                assert H.predict_raw_reference(m, X)[0] == ref
            loaded.free()


def _models(rng, ncol):
    yield "stump_grid", H.stump_grid_model(H.threshold_pool(rng), ncol)
    for k in TREE_COUNTS:
        yield f"trees{k}", H.synthetic_model(rng, k, ncol, features=[0, ncol - 1] + list(rng.integers(0, ncol, 6)))


def test_live_reference_predicts_the_restatement_on_adversarial_rows():
    refapi = _ref()
    rng = np.random.default_rng(20)
    ncol = 9
    for name, m in _models(rng, ncol):
        loaded = refapi.RefLoadedBooster(m.to_string())
        for dtype in (np.float32, np.float64):
            X = H.boundary_matrix(H.model_columns(m, ncol, dtype == np.float64), 64, rng, dtype)
            want = loaded.predict(X)
            got = H.predict_raw_reference(m, X)
            bad = np.flatnonzero(got != want)
            assert got.tobytes() == want.tobytes(), f"{name} {np.dtype(dtype).name}: {len(bad)} rows differ, first {bad[:5]}"
        loaded.free()


BINNER_VARIANTS = {
    "nan_missing": dict(),
    "zero_as_missing": dict(zero_as_missing="true"),
    "no_missing": dict(use_missing="false"),
}


def binner_params(**kw):
    return dict(dict(max_bin=255, min_data_in_bin=1, min_data_in_leaf=1, feature_pre_filter="false", enable_bundle="false"), **kw)


def _valid_dataset(refapi, train, X, params):
    """LGBM_DatasetCreateFromMat(X, reference=train): the training Dataset's bin mappers, one feature per stored column."""
    X = np.ascontiguousarray(X)
    h = C.c_void_p()
    refapi._check(refapi.lib().LGBM_DatasetCreateFromMat(X.ctypes.data_as(C.c_void_p), C.c_int(0 if X.dtype == np.float32 else 1),
                                                         C.c_int32(X.shape[0]), C.c_int32(X.shape[1]), C.c_int(1),
                                                         C.c_char_p(refapi.params_str(params)), train.handle, C.byref(h)))
    ds = refapi.RefDataset.__new__(refapi.RefDataset)
    ds.handle, ds.num_data = h, X.shape[0]
    return ds


@pytest.mark.parametrize("variant", list(BINNER_VARIANTS))
@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_live_reference_bins_adversarial_values_as_the_restatement(variant, dtype):
    """Mappers fitted on binner_fit_matrix, then a matrix of values on and next to every bound binned with them."""
    refapi = _ref()
    rng = np.random.default_rng(21)
    Xf = H.binner_fit_matrix(rng, dtype=dtype)
    params = dict(binner_params(**BINNER_VARIANTS[variant]), device_type="cuda", verbosity=-1)
    train = refapi.RefDataset(Xf, None, params)
    lay = train.layout()
    if variant == "nan_missing":
        searchable = {int(nb) - 1 - (1 if mt == H.MISSING_NAN else 0) for nb, mt in zip(lay.feat_num_bin, lay.feat_missing)}
        assert searchable >= set(H.BOUND_COUNTS)
    meta = dict(num_columns=lay.num_columns, num_features=lay.num_features, feat_column=lay.feat_column, feat_lo=lay.feat_lo,
                feat_num_bin=lay.feat_num_bin, feat_most_freq_bin=lay.feat_mfb, feat_missing_type=lay.feat_missing,
                feat_real_index=lay.feat_real_index)
    Xa = H.boundary_matrix(H.binner_columns(meta, lay.bin_upper_bound, Xf.shape[1], dtype == np.float64), 64, rng, dtype)
    valid = _valid_dataset(refapi, train, Xa, params)
    v = valid.layout()
    vmeta = dict(meta, num_columns=v.num_columns, feat_column=v.feat_column, feat_lo=v.feat_lo)
    got = H.value_to_bin_reference(Xa, vmeta, lay.bin_upper_bound)
    bad = np.argwhere(got != v.bins)
    assert got.tobytes() == v.bins.tobytes(), f"{len(bad)} bytes differ, first (row, column) {bad[:5].tolist()}"
    valid.free(); train.free()


def test_binner_fit_matches_the_reference_on_the_boundary_features():
    """The layouts and bounds the GPU tests bin with are the reference's (the binner is pinned on the fixtures; this ties
    the generated features to it as well)."""
    refapi = _ref()
    from lightgbm_b200 import Binner
    for seed, make, extra in ((22, H.binner_fit_matrix, {}), (23, H.binner_sparse_matrix, dict(enable_bundle="true"))):
        X = make(np.random.default_rng(seed))
        params = binner_params(**extra)
        ref = refapi.RefDataset(X, None, dict(params, device_type="cuda", verbosity=-1)).layout()
        b = Binner(params).fit(X)
        m = b.layout_meta()
        assert (m["num_columns"], m["num_features"]) == (ref.num_columns, ref.num_features)
        for mine, theirs in (("feat_column", "feat_column"), ("feat_lo", "feat_lo"), ("feat_most_freq_bin", "feat_mfb"),
                             ("feat_missing_type", "feat_missing"), ("feat_real_index", "feat_real_index")):
            np.testing.assert_array_equal(m[mine], getattr(ref, theirs), err_msg=mine)
        for f, ub in enumerate(b.bin_upper_bounds()):
            assert ub.tobytes() == np.asarray(ref.bin_upper_bound[f], np.float64).tobytes()
        assert H.value_to_bin_reference(X, m, b.bin_upper_bounds()).tobytes() == ref.bins.tobytes()
        b.free()
