"""ctypes binding of the plain-C oracle (oracle/lgbm_oracle.c).  TEST INFRASTRUCTURE ONLY — the checker
for the CUDA path; nothing under lightgbm_b200/ may import this module."""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from dataclasses import dataclass

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "liblgbm_oracle.so")
_lib = None


class _OrcLayout(C.Structure):
    _fields_ = [("num_data", C.c_int32), ("num_columns", C.c_int32), ("num_features", C.c_int32)] + \
               [(k, C.c_void_p) for k in ("feat_column", "feat_lo", "feat_num_bin", "feat_mfb", "feat_default_bin",
                                          "feat_missing", "feat_real_index", "feat_in_group")]


class _OrcParams(C.Structure):
    _fields_ = [("num_leaves", C.c_int32), ("max_depth", C.c_int32), ("min_data_in_leaf", C.c_int32),
                ("min_sum_hessian_in_leaf", C.c_double), ("lambda_l1", C.c_double), ("lambda_l2", C.c_double),
                ("min_gain_to_split", C.c_double), ("max_delta_step", C.c_double), ("path_smooth", C.c_double)]


class _OrcSplit(C.Structure):
    _fields_ = [("leaf", C.c_int32), ("feature", C.c_int32), ("threshold", C.c_int32), ("default_left", C.c_int32),
                ("left_count", C.c_int32), ("right_count", C.c_int32), ("gain", C.c_double),
                ("left_sum_gradient", C.c_double), ("left_sum_hessian", C.c_double), ("left_output", C.c_double),
                ("right_sum_gradient", C.c_double), ("right_sum_hessian", C.c_double), ("right_output", C.c_double),
                ("second_gain", C.c_double)]


SPLIT_DTYPE = np.dtype([("leaf", "i4"), ("feature", "i4"), ("threshold", "i4"), ("default_left", "i4"),
                        ("left_count", "i4"), ("right_count", "i4"), ("gain", "f8"),
                        ("left_sum_gradient", "f8"), ("left_sum_hessian", "f8"), ("left_output", "f8"),
                        ("right_sum_gradient", "f8"), ("right_sum_hessian", "f8"), ("right_output", "f8"),
                        ("second_gain", "f8")], align=True)
assert SPLIT_DTYPE.itemsize == C.sizeof(_OrcSplit)


class _OrcTree(C.Structure):
    _fields_ = [("num_leaves", C.c_int32), ("splits", C.c_void_p), ("leaf_value", C.c_void_p),
                ("leaf_weight", C.c_void_p), ("leaf_count", C.c_void_p), ("leaf_depth", C.c_void_p),
                ("leaf_begin", C.c_void_p), ("indices", C.c_void_p),
                ("root_sum_gradient", C.c_double), ("root_sum_hessian", C.c_double)]


def build(force: bool = False) -> str:
    src = os.path.join(_HERE, "lgbm_oracle.c")
    if force or not os.path.exists(_LIB_PATH) or os.path.getmtime(_LIB_PATH) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _HERE, "liblgbm_oracle.so"], stdout=subprocess.DEVNULL)
    return _LIB_PATH


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
        _lib.orc_train_tree.restype = C.c_int
        _lib.orc_train_tree_quant.restype = C.c_int
        _lib.orc_partition.restype = C.c_int32
        _lib.orc_find_best_threshold.restype = C.c_int
    return _lib


DEFAULT_PARAMS = dict(num_leaves=31, max_depth=-1, min_data_in_leaf=20, min_sum_hessian_in_leaf=1e-3, lambda_l1=0.0,
                      lambda_l2=0.0, min_gain_to_split=0.0, max_delta_step=0.0, path_smooth=0.0)


def make_params(**kw) -> _OrcParams:
    d = dict(DEFAULT_PARAMS)
    for k, v in kw.items():
        if k in d:
            d[k] = v
    return _OrcParams(**d)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def make_layout(lay):
    """lay: oracle.refapi.Layout (or anything with the same attributes).  Returns (struct, keepalive)."""
    keep = [np.ascontiguousarray(getattr(lay, k), dtype=np.int32) for k in
            ("feat_column", "feat_lo", "feat_num_bin", "feat_mfb", "feat_default_bin", "feat_missing",
             "feat_real_index")]
    in_group = getattr(lay, "feat_in_group", None)
    if in_group is None:
        in_group = np.bincount(keep[0], minlength=lay.num_columns)[keep[0]]
    keep.append(np.ascontiguousarray(in_group, dtype=np.int32))
    s = _OrcLayout(lay.num_data, lay.num_columns, lay.num_features, *[_p(a) for a in keep])
    return s, keep


@dataclass
class OracleTree:
    num_leaves: int
    splits: np.ndarray        # SPLIT_DTYPE[num_leaves-1]
    leaf_value: np.ndarray
    leaf_weight: np.ndarray
    leaf_count: np.ndarray
    leaf_depth: np.ndarray
    leaf_begin: np.ndarray
    indices: np.ndarray
    root_sum_gradient: float
    root_sum_hessian: float


def train_tree(lay, grad, hess, bag_indices=None, feature_used=None, **params) -> OracleTree:
    L, keep = make_layout(lay)
    P = make_params(**params)
    NL = P.num_leaves
    bins = np.ascontiguousarray(lay.bins, dtype=np.uint8)
    g = np.ascontiguousarray(grad, dtype=np.float32)
    h = np.ascontiguousarray(hess, dtype=np.float32)
    splits = np.zeros(max(NL - 1, 1), dtype=SPLIT_DTYPE)
    lv, lw = np.zeros(NL), np.zeros(NL)
    lc, ld, lb = (np.zeros(NL, np.int32) for _ in range(3))
    idx = np.zeros(max(lay.num_data, 1), np.int32)
    T = _OrcTree(0, _p(splits), _p(lv), _p(lw), _p(lc), _p(ld), _p(lb), _p(idx), 0.0, 0.0)
    bag = None if bag_indices is None else np.ascontiguousarray(bag_indices, dtype=np.int32)
    fu = None if feature_used is None else np.ascontiguousarray(feature_used, dtype=np.uint8)
    r = lib().orc_train_tree(C.byref(L), _p(bins), _p(g), _p(h), None if bag is None else _p(bag),
                             C.c_int32(0 if bag is None else len(bag)), None if fu is None else _p(fu),
                             C.byref(P), C.byref(T))
    if r != 0:
        raise RuntimeError("orc_train_tree failed")
    n = T.num_leaves
    return OracleTree(n, splits[:n - 1].copy(), lv[:n], lw[:n], lc[:n], ld[:n], lb[:n], idx,
                      T.root_sum_gradient, T.root_sum_hessian)


class _OrcQuant(C.Structure):
    _fields_ = [("num_grad_quant_bins", C.c_int32), ("is_constant_hessian", C.c_int32), ("renew_leaf", C.c_int32),
                ("grad_scale", C.c_double), ("hess_scale", C.c_double)]


def discretize(grad, hess, num_grad_quant_bins=4, is_constant_hessian=False, random_g=None, random_h=None):
    """GradientDiscretizer::DiscretizeGradients; returns (int8 g, int8 h, grad_scale, hess_scale)."""
    g = np.ascontiguousarray(grad, dtype=np.float32); h = np.ascontiguousarray(hess, dtype=np.float32)
    Q = _OrcQuant(num_grad_quant_bins, 1 if is_constant_hessian else 0, 0, 0.0, 0.0)
    qg, qh = np.zeros(len(g), np.float32), np.zeros(len(g), np.float32)
    rg = None if random_g is None else np.ascontiguousarray(random_g, dtype=np.float64)
    rh = None if random_h is None else np.ascontiguousarray(random_h, dtype=np.float64)
    lib().orc_discretize(_p(g), _p(h), C.c_int32(len(g)), C.byref(Q), None if rg is None else _p(rg),
                         None if rh is None else _p(rh), _p(qg), _p(qh))
    return qg.astype(np.int8), qh.astype(np.int8), Q.grad_scale, Q.hess_scale


def train_tree_quant(lay, grad, hess, num_grad_quant_bins=4, is_constant_hessian=False, renew_leaf=False,
                     bag_indices=None, feature_used=None, random_g=None, random_h=None, **params) -> OracleTree:
    """SerialTreeLearner::Train with use_quantized_grad=true: stochastic_rounding=false, or the per-row uniforms of
    stochastic rounding in random_g / random_h (as discretize() takes them)."""
    L, keep = make_layout(lay)
    P = make_params(**params)
    NL = P.num_leaves
    bins = np.ascontiguousarray(lay.bins, dtype=np.uint8)
    g = np.ascontiguousarray(grad, dtype=np.float32)
    h = np.ascontiguousarray(hess, dtype=np.float32)
    splits = np.zeros(max(NL - 1, 1), dtype=SPLIT_DTYPE)
    lv, lw = np.zeros(NL), np.zeros(NL)
    lc, ld, lb = (np.zeros(NL, np.int32) for _ in range(3))
    idx = np.zeros(max(lay.num_data, 1), np.int32)
    T = _OrcTree(0, _p(splits), _p(lv), _p(lw), _p(lc), _p(ld), _p(lb), _p(idx), 0.0, 0.0)
    Q = _OrcQuant(num_grad_quant_bins, 1 if is_constant_hessian else 0, 1 if renew_leaf else 0, 0.0, 0.0)
    bag = None if bag_indices is None else np.ascontiguousarray(bag_indices, dtype=np.int32)
    fu = None if feature_used is None else np.ascontiguousarray(feature_used, dtype=np.uint8)
    rg = None if random_g is None else np.ascontiguousarray(random_g, dtype=np.float64)
    rh = None if random_h is None else np.ascontiguousarray(random_h, dtype=np.float64)
    r = lib().orc_train_tree_quant(C.byref(L), _p(bins), _p(g), _p(h), None if bag is None else _p(bag),
                                   C.c_int32(0 if bag is None else len(bag)), None if fu is None else _p(fu),
                                   C.byref(P), C.byref(Q), None if rg is None else _p(rg), None if rh is None else _p(rh),
                                   C.byref(T))
    if r != 0:
        raise RuntimeError("orc_train_tree_quant failed")
    n = T.num_leaves
    t = OracleTree(n, splits[:n - 1].copy(), lv[:n], lw[:n], lc[:n], ld[:n], lb[:n], idx,
                   T.root_sum_gradient, T.root_sum_hessian)
    t.grad_scale, t.hess_scale = Q.grad_scale, Q.hess_scale
    return t


def construct_histogram(lay, indices, grad, hess) -> np.ndarray:
    L, keep = make_layout(lay)
    bins = np.ascontiguousarray(lay.bins, dtype=np.uint8)
    g = np.ascontiguousarray(grad, dtype=np.float32)
    h = np.ascontiguousarray(hess, dtype=np.float32)
    hist = np.zeros((lay.num_columns, 256, 2), dtype=np.float64)
    idx = None if indices is None else np.ascontiguousarray(indices, dtype=np.int32)
    n = lay.num_data if idx is None else len(idx)
    lib().orc_construct_histogram(C.byref(L), _p(bins), None if idx is None else _p(idx), C.c_int32(n), _p(g), _p(h),
                                  _p(hist))
    return hist


def partition(lay, feature, threshold, default_left, indices):
    L, keep = make_layout(lay)
    bins = np.ascontiguousarray(lay.bins, dtype=np.uint8)
    idx = np.ascontiguousarray(indices, dtype=np.int32).copy()
    nl = lib().orc_partition(C.byref(L), _p(bins), C.c_int(feature), C.c_int(threshold), C.c_int(default_left),
                             _p(idx), C.c_int32(len(idx)))
    return idx, int(nl)
