"""The value -> bin pass (binning.cuh) and the predictor (predict.cuh) bit for bit against their plain restatements
(tests/helpers.py), on values that sit on and next to every bin bound and threshold, on every launch path.

tests/test_boundary_reference.py pins the restatements to the reference.  Here the device must equal them exactly:
  * binning: float32 and float64, host and device-resident input, identity order and the bundled two-step path, 1 .. 100
    features across the 32-feature tiles, 1 .. 65 rows, and rows crossing host chunks and row pieces;
  * prediction: column counts either side of the 64-row tile / 32-row tile / k_predict_wide limits, 1 .. 65 rows, three
    host chunks and a ragged tail, the device-resident single launch, 1 .. 33 trees (odd counts, pass boundaries, the pair
    walk), 254-deep chains and single leaves, the zero band, and LGBMB200_PRED_PASS = 2 / 5 / 32."""
import os
import subprocess
import sys

import numpy as np
import pytest

import helpers as H
from exact_worker import predict_case

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
TREE_COUNTS = (1, 2, 15, 16, 17, 31, 32, 33)
ROWS_BIN = (1, 63, 64, 65)
ROWS_PRED = (1, 31, 32, 33, 63, 64, 65)


@pytest.fixture(scope="module")
def lgb(built_lib):
    import lightgbm_b200
    return lightgbm_b200


def _params(**kw):
    return dict(dict(max_bin=255, min_data_in_bin=1, min_data_in_leaf=1, feature_pre_filter="false", enable_bundle="false"), **kw)


def _first_diff(got, want):
    bad = np.argwhere(np.asarray(got) != np.asarray(want))
    return f"{len(bad)} entries differ, first {bad[:4].tolist()}"


# ---------------------------------------------------------------------------------------------------- binning
def _binner_case(lgb, Xf, params, rng, rows=64):
    b = lgb.Binner(params).fit(Xf)
    meta, ub = b.layout_meta(), b.bin_upper_bounds()
    Xa = H.boundary_matrix(H.binner_columns(meta, ub, Xf.shape[1], Xf.dtype == np.float64), rows, rng, Xf.dtype)
    return b, meta, Xa, H.value_to_bin_reference(Xa, meta, ub)


def _check_transform(lgb, b, X, want, what):
    from lightgbm_b200.tree_learner import DeviceArray
    host, _ = b.transform(X, to_device=False)
    assert host.tobytes() == want.tobytes(), f"{what} host -> host: {_first_diff(host, want)}"
    dev, _ = b.transform(X, to_device=True)
    got = dev.download()
    assert got.tobytes() == want.tobytes(), f"{what} host -> device: {_first_diff(got, want)}"
    dx = DeviceArray(X.nbytes).upload(X)
    dev2, _ = b.transform((dx, X.dtype), to_device=True, data_rows=X.shape[0])
    got = dev2.download()
    dx.free()
    assert got.tobytes() == want.tobytes(), f"{what} device -> device: {_first_diff(got, want)}"


@pytest.mark.parametrize("variant", [dict(), dict(zero_as_missing="true"), dict(use_missing="false")], ids=["nan", "zero", "nomissing"])
@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_binning_bounds_at_every_search_depth(lgb, dtype, variant):
    """Features with 0 .. 254 searchable bounds (every depth edge of search_bounds_smem), values on and next to each."""
    rng = np.random.default_rng(40)
    b, meta, Xa, want = _binner_case(lgb, H.binner_fit_matrix(rng, dtype=dtype), _params(**variant), rng)
    if not variant:
        searchable = {int(nb) - 1 - (1 if mt == H.MISSING_NAN else 0) for nb, mt in zip(meta["feat_num_bin"], meta["feat_missing_type"])}
        assert searchable >= set(H.BOUND_COUNTS)
    for rows in ROWS_BIN + (Xa.shape[0],):
        _check_transform(lgb, b, np.ascontiguousarray(Xa[:rows]), want[:rows], f"{rows} rows")


@pytest.mark.parametrize("bundle", [False, True], ids=["identity", "bundled"])
@pytest.mark.parametrize("nfeat", [1, 31, 32, 33, 63, 65, 100])
def test_binning_feature_tiles(lgb, nfeat, bundle):
    """1 .. 100 features across the 32-feature tiles of k_value_to_bin_tile; bundled layouts also go through
    k_bundle_columns, and the adversarial rows have every sub-feature of a bundle off its most frequent bin at once."""
    rng = np.random.default_rng(41 + nfeat)
    dtype = np.float32 if nfeat % 2 else np.float64
    if bundle and nfeat >= 3:
        Xf = H.binner_sparse_matrix(rng, c=nfeat, dtype=dtype)
    else:
        base = H.binner_fit_matrix(rng, dtype=dtype)
        Xf = np.ascontiguousarray(base[:, [j % base.shape[1] for j in range(nfeat)]])
    b, meta, Xa, want = _binner_case(lgb, Xf, _params(enable_bundle=str(bundle).lower()), rng)
    if bundle and nfeat >= 3:
        assert meta["num_columns"] < meta["num_features"]
    for rows in ROWS_BIN + (Xa.shape[0],):
        _check_transform(lgb, b, np.ascontiguousarray(Xa[:rows]), want[:rows], f"{rows} rows")


@pytest.mark.parametrize("case", ["f64_bundled_1000", "f32_identity_1000"])
def test_binning_host_chunks_and_row_pieces(lgb, case):
    """Host input is sent in chunks of max(1024, 128 MiB / (ncol * esize)) rows and the bundled path cuts a chunk into
    pieces of 16 MiB / Fp rows: 1000 float64 columns give 16 777-row chunks and 16 640-row pieces, 1000 float32 columns
    33 554-row chunks.  Two chunks and a ragged third."""
    rng = np.random.default_rng(42)
    f64 = case.startswith("f64")
    dtype = np.float64 if f64 else np.float32
    if f64:
        Xf = H.binner_sparse_matrix(rng, n=4000, c=1000, dtype=dtype)
    else:
        base = H.binner_fit_matrix(rng, dtype=dtype)
        Xf = np.ascontiguousarray(base[:, [j % base.shape[1] for j in range(1000)]])
    b, meta, Xa, want = _binner_case(lgb, Xf, _params(enable_bundle=str(f64).lower()), rng)
    chunk = (128 << 20) // (Xf.shape[1] * Xf.dtype.itemsize)
    n = 2 * chunk + 1237
    reps = -(-n // Xa.shape[0])
    X = np.ascontiguousarray(np.tile(Xa, (reps, 1))[:n])
    W = np.tile(want, (reps, 1))[:n]
    host, _ = b.transform(X, to_device=False)
    assert host.tobytes() == W.tobytes(), _first_diff(host, W)
    if f64:
        assert meta["num_columns"] < meta["num_features"]
        Fp = (int(meta["num_features"]) + 15) // 16 * 16
        assert (16 << 20) // Fp // 64 * 64 < chunk                # a chunk is cut into two pieces


# ---------------------------------------------------------------------------------------------------- prediction
def _predict_all_ways(m, X, want, what):
    from lightgbm_b200.tree_learner import DeviceArray
    got = m.predict_raw(X)
    assert got.tobytes() == want.tobytes(), f"{what} host: {_first_diff(got, want)}"
    dx = DeviceArray(X.nbytes).upload(X)
    out = DeviceArray(8 * X.shape[0])
    m.predict_raw((dx, X.dtype), data_shape=X.shape, out=out)
    got = out.download(np.float64, X.shape[0])
    dx.free(); out.free()
    assert got.tobytes() == want.tobytes(), f"{what} device-resident: {_first_diff(got, want)}"


def test_zero_band_rows_follow_the_reference(lgb):
    """A value of exactly -kZeroThreshold at a threshold of -kZeroThreshold goes right (the reference reads the value as
    0.0), and so on for every threshold and value in and around the zero band, under all six decision types."""
    pool = np.array([-H.K_ZERO, 0.0, -0.0, H.K_ZERO, 5e-36, -5e-36, float(np.nextafter(-H.K_ZERO, -np.inf)),
                     float(np.nextafter(-H.K_ZERO, 0.0)), float(np.nextafter(H.K_ZERO, 0.0)), -1.0, 1.0])
    m = H.stump_grid_model(pool, 1)
    for dtype in (np.float32, np.float64):
        X = np.ascontiguousarray(H.boundary_values(pool, dtype == np.float64).astype(dtype)[:, None])
        _predict_all_ways(m, X, H.predict_raw_reference(m, X), np.dtype(dtype).name)
    one = H.text_model(H.stump_grid_model([-H.K_ZERO], 1).trees[:1], 1)         # missing type None, default right
    assert one.predict_raw(np.array([[-H.K_ZERO]], np.float32))[0] == one.trees[0].leaf_value[1]


@pytest.mark.parametrize("num_trees", TREE_COUNTS)
@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_predict_tree_counts_and_shapes(lgb, num_trees, dtype):
    """Random, 254-deep chain, balanced and single-leaf trees; thresholds from the pool; every missing type and default
    direction; rows on and next to every threshold."""
    rng = np.random.default_rng(50 + num_trees)
    ncol = 9
    m = H.synthetic_model(rng, num_trees, ncol)
    X = H.boundary_matrix(H.model_columns(m, ncol, dtype == np.float64), 100, rng, dtype)
    want = H.predict_raw_reference(m, X)
    for rows in ROWS_PRED + (X.shape[0],):
        _predict_all_ways(m, np.ascontiguousarray(X[:rows]), want[:rows], f"{rows} rows")


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_predict_threshold_grid(lgb, dtype):
    """Every pool threshold under all six decision types, every adversarial value in every column."""
    rng = np.random.default_rng(51)
    m = H.stump_grid_model(H.threshold_pool(rng), 5)
    X = H.boundary_matrix(H.model_columns(m, 5, dtype == np.float64), 64, rng, dtype)
    _predict_all_ways(m, X, H.predict_raw_reference(m, X), "grid")


# 16 trees per pass: float32 stages 64-row tiles up to 415 columns, 32-row tiles up to 1759, wider rows go to
# k_predict_wide; float64 switches at 207 / 208 and 879 / 880.
@pytest.mark.parametrize("dtype,ncol", [(np.float32, c) for c in (415, 416, 1759, 1760)] + [(np.float64, c) for c in (207, 208, 879, 880)],
                         ids=lambda v: v if isinstance(v, int) else np.dtype(v).name)
def test_predict_launch_paths(lgb, dtype, ncol):
    rng = np.random.default_rng(60 + ncol)
    m = H.synthetic_model(rng, 33, ncol, features=[0, ncol - 1, ncol // 2])
    X = H.boundary_matrix(H.model_columns(m, ncol, dtype == np.float64), 200, rng, dtype)
    want = H.predict_raw_reference(m, X)
    for rows in ROWS_PRED + (X.shape[0],):
        _predict_all_ways(m, np.ascontiguousarray(X[:rows]), want[:rows], f"{rows} rows")


@pytest.mark.parametrize("dtype,ncol", [(np.float32, 416), (np.float64, 880)], ids=["f32_416", "f64_880"])
def test_predict_three_host_chunks_and_a_ragged_tail(lgb, dtype, ncol):
    """Host rows go in chunks of max(1024, 64 MiB / (ncol * esize)) on two streams: three chunks and a ragged tail."""
    rng = np.random.default_rng(70)
    m = H.synthetic_model(rng, 17, ncol, features=[0, ncol - 1, 3])
    X = H.boundary_matrix(H.model_columns(m, ncol, dtype == np.float64), 300, rng, dtype)
    want = H.predict_raw_reference(m, X)
    chunk = (64 << 20) // (ncol * np.dtype(dtype).itemsize)
    n = 3 * chunk + 777
    reps = -(-n // X.shape[0])
    big = np.ascontiguousarray(np.tile(X, (reps, 1))[:n])
    W = np.tile(want, reps)[:n]
    got = m.predict_raw(big)
    assert got.tobytes() == W.tobytes(), _first_diff(got, W)


@pytest.mark.parametrize("pred_pass", [2, 5, 32])
def test_pred_pass_gives_the_same_bits(tmp_path, lgb, pred_pass):
    """LGBMB200_PRED_PASS (trees per pass of k_predict) in a subprocess: the same bits as the restatement."""
    out = str(tmp_path / "predict.npz")
    r = subprocess.run([sys.executable, os.path.join(HERE, "exact_worker.py"), "predict", out],
                       env=dict(os.environ, LGBMB200_PRED_PASS=str(pred_pass)), capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    got = np.load(out)
    for dtype in (np.float32, np.float64):
        m, X = predict_case(dtype)
        want = H.predict_raw_reference(m, X)
        assert got[np.dtype(dtype).name].tobytes() == want.tobytes(), f"{np.dtype(dtype).name}: {_first_diff(got[np.dtype(dtype).name], want)}"
