"""Host-side mirror of the reference plug-in interface `class TreeLearner`
(reference include/LightGBM/tree_learner.h:27-114) over the C-ABI of include/lgbm_b200.h.

Same method names, argument meaning and error behaviour (errors raise, like Log::Fatal unwinding to
the C API): Init / ResetConfig / SetBaggingData / Train / AddPredictionToScore.  The compute happens
in lightgbm_b200/lib/liblgbm_b200.so (hand-written sm_90a CUDA); there is no CPU path here.
"""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass, field

import numpy as np

from ._lib import check, lib

MISSING_NONE, MISSING_ZERO, MISSING_NAN = 0, 1, 2


class _CConfig(C.Structure):
    _fields_ = [("num_leaves", C.c_int32), ("max_depth", C.c_int32), ("min_data_in_leaf", C.c_int32),
                ("gpu_device_id", C.c_int32), ("min_sum_hessian_in_leaf", C.c_double), ("lambda_l1", C.c_double),
                ("lambda_l2", C.c_double), ("min_gain_to_split", C.c_double), ("max_delta_step", C.c_double),
                ("path_smooth", C.c_double), ("use_cuda_graph", C.c_int32), ("reserved", C.c_int32),
                ("use_quantized_grad", C.c_int32), ("num_grad_quant_bins", C.c_int32), ("quant_train_renew_leaf", C.c_int32),
                ("stochastic_rounding", C.c_int32), ("seed", C.c_int32), ("pad_", C.c_int32)]


class _CLayout(C.Structure):
    _fields_ = [("num_data", C.c_int32), ("num_columns", C.c_int32), ("num_features", C.c_int32)] + \
               [(k, C.c_void_p) for k in ("feat_column", "feat_lo", "feat_num_bin", "feat_most_freq_bin",
                                          "feat_default_bin", "feat_missing_type", "feat_real_index")]


class _CSplit(C.Structure):
    _fields_ = [("leaf", C.c_int32), ("feature", C.c_int32), ("threshold", C.c_int32), ("default_left", C.c_int32),
                ("left_count", C.c_int32), ("right_count", C.c_int32), ("gain", C.c_double),
                ("left_sum_gradient", C.c_double), ("left_sum_hessian", C.c_double), ("left_output", C.c_double),
                ("right_sum_gradient", C.c_double), ("right_sum_hessian", C.c_double), ("right_output", C.c_double)]


SPLIT_DTYPE = np.dtype([("leaf", "i4"), ("feature", "i4"), ("threshold", "i4"), ("default_left", "i4"),
                        ("left_count", "i4"), ("right_count", "i4"), ("gain", "f8"),
                        ("left_sum_gradient", "f8"), ("left_sum_hessian", "f8"), ("left_output", "f8"),
                        ("right_sum_gradient", "f8"), ("right_sum_hessian", "f8"), ("right_output", "f8")], align=True)
assert SPLIT_DTYPE.itemsize == C.sizeof(_CSplit)


class _CTree(C.Structure):
    _fields_ = [("num_leaves", C.c_int32), ("splits", C.c_void_p), ("leaf_value", C.c_void_p),
                ("leaf_weight", C.c_void_p), ("leaf_count", C.c_void_p), ("leaf_depth", C.c_void_p),
                ("root_sum_gradient", C.c_double), ("root_sum_hessian", C.c_double),
                ("grad_scale", C.c_double), ("hess_scale", C.c_double)]


@dataclass
class Config:
    """The Config fields the hot path reads (reference include/LightGBM/config.h; SURVEY.md §5)."""
    num_leaves: int = 31
    max_depth: int = -1
    min_data_in_leaf: int = 20
    min_sum_hessian_in_leaf: float = 1e-3
    lambda_l1: float = 0.0
    lambda_l2: float = 0.0
    min_gain_to_split: float = 0.0
    max_delta_step: float = 0.0
    path_smooth: float = 0.0
    gpu_device_id: int = -1
    use_cuda_graph: bool = True
    reserved: int = 0                     # bit 0: no column-major partition copy (include/lgbm_b200.h)
    use_quantized_grad: bool = False      # reference config.h:626-651
    num_grad_quant_bins: int = 4
    quant_train_renew_leaf: bool = False
    stochastic_rounding: bool = True
    seed: int = 0

    def to_c(self) -> _CConfig:
        return _CConfig(self.num_leaves, self.max_depth, self.min_data_in_leaf, self.gpu_device_id,
                        self.min_sum_hessian_in_leaf, self.lambda_l1, self.lambda_l2, self.min_gain_to_split,
                        self.max_delta_step, self.path_smooth, 1 if self.use_cuda_graph else 0, int(self.reserved),
                        1 if self.use_quantized_grad else 0, int(self.num_grad_quant_bins),
                        1 if self.quant_train_renew_leaf else 0, 1 if self.stochastic_rounding else 0, int(self.seed), 0)


@dataclass
class Layout:
    """Binned training matrix + per-feature metadata: what `Dataset` hands to TreeLearner::Init
    (reference dataset.h:638-647,806-810,985-1000).  See include/lgbm_b200.h LGBMB200_Layout."""
    bins: object                     # [num_data, num_columns] uint8 stored group values: np.ndarray, or a matrix already in HBM
                                     # (dataset.DeviceMatrix: anything with .shape and .ptr)
    feat_column: np.ndarray
    feat_lo: np.ndarray
    feat_num_bin: np.ndarray
    feat_mfb: np.ndarray
    feat_default_bin: np.ndarray
    feat_missing: np.ndarray
    feat_real_index: np.ndarray
    bin_upper_bound: list = field(default_factory=list)   # per feature: bin -> real threshold (RealThreshold)

    @property
    def num_data(self):
        return self.bins.shape[0]

    @property
    def num_columns(self):
        return self.bins.shape[1]

    @property
    def num_features(self):
        return len(self.feat_column)

    @staticmethod
    def identity(bins: np.ndarray, num_bin: int = 255) -> "Layout":
        """One feature per column, stored value == bin, most_freq_bin = default_bin = 0, no missing —
        what the reference Dataset produces for integer-valued features in [0, num_bin) (SURVEY.md §8c(ii))."""
        n, f = bins.shape
        z = np.zeros(f, np.int32)
        return Layout(np.ascontiguousarray(bins, dtype=np.uint8), np.arange(f, dtype=np.int32), np.ones(f, np.int32),
                      np.full(f, num_bin, np.int32), z.copy(), z.copy(), z.copy(), np.arange(f, dtype=np.int32))

    @staticmethod
    def from_attrs(o) -> "Layout":
        """Adopt any object with the same attribute names (e.g. oracle.refapi.Layout in the tests)."""
        return Layout(np.ascontiguousarray(o.bins, dtype=np.uint8),
                      *[np.ascontiguousarray(getattr(o, k), dtype=np.int32) for k in
                        ("feat_column", "feat_lo", "feat_num_bin", "feat_mfb", "feat_default_bin", "feat_missing",
                         "feat_real_index")], bin_upper_bound=list(getattr(o, "bin_upper_bound", [])))

    def column_slice(self, col_lo: int, col_hi: int) -> "Layout":
        """Feature-shard: keep the features whose column is in [col_lo, col_hi) (all rows)."""
        keep = np.nonzero((self.feat_column >= col_lo) & (self.feat_column < col_hi))[0]
        return Layout(np.ascontiguousarray(self.bins[:, col_lo:col_hi]), (self.feat_column[keep] - col_lo).astype(np.int32),
                      self.feat_lo[keep].copy(), self.feat_num_bin[keep].copy(), self.feat_mfb[keep].copy(),
                      self.feat_default_bin[keep].copy(), self.feat_missing[keep].copy(),
                      self.feat_real_index[keep].copy(),
                      bin_upper_bound=[self.bin_upper_bound[i] for i in keep] if self.bin_upper_bound else [])


@dataclass
class Tree:
    """Flat POD tree: the fields Tree::Split fills (reference include/LightGBM/tree.h:543-585)."""
    num_leaves: int
    splits: np.ndarray               # SPLIT_DTYPE[num_leaves-1], node i == i-th split
    leaf_value: np.ndarray
    leaf_weight: np.ndarray
    leaf_count: np.ndarray
    leaf_depth: np.ndarray
    root_sum_gradient: float
    root_sum_hessian: float
    shrink: float = 1.0              # product of the rates applied so far / the bias added: the model text needs them for
    bias: float = 0.0                # the internal node values (lightgbm_b200/model.py)

    def shrinkage(self, rate: float) -> None:
        """Tree::Shrinkage (reference include/LightGBM/tree.h:187-200): leaf values in the zero band become 0, so the
        score update adds what the model text holds."""
        self.leaf_value = round_to_zero(self.leaf_value * rate)
        self.shrink *= rate

    def add_bias(self, val: float) -> None:
        """Tree::AddBias (reference tree.h:211-230)."""
        self.leaf_value = round_to_zero(self.leaf_value + val)
        self.bias += val

    def as_constant(self, val: float, count: int) -> None:
        """Tree::AsConstantTree (tree.h:232-240): one leaf holding `val`, weight 0, `count` rows, shrinkage 1."""
        self.num_leaves = 1
        self.splits = self.splits[:0]
        self.leaf_value, self.leaf_weight = np.array([float(val)]), np.zeros(1)
        self.leaf_count, self.leaf_depth = np.array([count], np.int32), np.zeros(1, np.int32)
        self.shrink, self.bias = 1.0, 0.0


K_ZERO = float(np.float32(1e-35))            # kZeroThreshold (meta.h:56): the float literal, widened


def round_to_zero(a) -> np.ndarray:
    """Tree::MaybeRoundToZero (tree.h:258-260) on every element: |v| <= kZeroThreshold becomes 0."""
    a = np.array(a, np.float64)
    a[np.abs(a) <= K_ZERO] = 0.0
    return a


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


class DeviceArray:
    """A raw HBM allocation owned through the C-ABI (so that callers need no torch for device memory)."""

    def __init__(self, nbytes: int):
        self.ptr = C.c_void_p()
        self.nbytes = int(nbytes)
        check(lib().LGBMB200_DeviceAlloc(C.byref(self.ptr), C.c_int64(self.nbytes)))

    def upload(self, arr: np.ndarray):
        a = np.ascontiguousarray(arr)
        assert a.nbytes <= self.nbytes
        check(lib().LGBMB200_MemcpyH2D(self.ptr, _p(a), C.c_int64(a.nbytes)))
        return self

    def download(self, dtype, count) -> np.ndarray:
        out = np.empty(count, dtype=dtype)
        check(lib().LGBMB200_MemcpyD2H(_p(out), self.ptr, C.c_int64(out.nbytes)))
        return out

    def free(self):
        if self.ptr:
            lib().LGBMB200_DeviceFree(self.ptr)
            self.ptr = C.c_void_p()

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class PinnedArray:
    """numpy view over cudaMallocHost memory (for the host-buffer e2e path)."""

    def __init__(self, shape, dtype):
        self.dtype = np.dtype(dtype)
        self.shape = (shape,) if np.isscalar(shape) else tuple(shape)
        n = int(np.prod(self.shape)) * self.dtype.itemsize
        self.ptr = C.c_void_p()
        check(lib().LGBMB200_HostAllocPinned(C.byref(self.ptr), C.c_int64(n)))
        buf = (C.c_byte * n).from_address(self.ptr.value)
        self.array = np.frombuffer(buf, dtype=self.dtype).reshape(self.shape)

    def free(self):
        if self.ptr:
            self.array = None
            lib().LGBMB200_HostFreePinned(self.ptr)
            self.ptr = C.c_void_p()


def _ptr_of(x):
    """host numpy array -> (pointer, on_device=0); DeviceArray / int / torch cuda tensor -> (pointer, 1)."""
    if isinstance(x, DeviceArray):
        return x.ptr, 1
    if isinstance(x, np.ndarray):
        return _p(x), 0
    if hasattr(x, "data_ptr"):       # torch tensor (plumbing only)
        return C.c_void_p(x.data_ptr()), 1 if x.is_cuda else 0
    return C.c_void_p(int(x)), 1


class B200TreeLearner:
    """Mirror of `TreeLearner` for ("serial", "cuda") — reference tree_learner.cpp:47-49."""

    def __init__(self, config: Config):
        self.config = config
        self.handle = C.c_void_p()
        c = config.to_c()
        check(lib().LGBMB200_LearnerCreate(C.byref(c), C.byref(self.handle)))
        self.layout = None

    # TreeLearner::Init(const Dataset* train_data, bool is_constant_hessian)
    def init(self, layout: Layout, is_constant_hessian: bool = False) -> None:
        on_device = hasattr(layout.bins, "ptr")
        bins = layout.bins if on_device else np.ascontiguousarray(layout.bins, dtype=np.uint8)
        keep = [np.ascontiguousarray(a, dtype=np.int32) for a in
                (layout.feat_column, layout.feat_lo, layout.feat_num_bin, layout.feat_mfb, layout.feat_default_bin,
                 layout.feat_missing, layout.feat_real_index)]
        cl = _CLayout(layout.num_data, layout.num_columns, layout.num_features, *[_p(a) for a in keep])
        check(lib().LGBMB200_LearnerInit(self.handle, C.byref(cl), bins.ptr if on_device else _p(bins), C.c_int32(1 if is_constant_hessian else 0)))
        self.layout = layout

    # TreeLearner::ResetConfig(const Config*)
    def reset_config(self, config: Config) -> None:
        self.config = config
        c = config.to_c()
        check(lib().LGBMB200_LearnerResetConfig(self.handle, C.byref(c)))

    # ColSampler by-tree mask
    def set_feature_mask(self, feature_used) -> None:
        if feature_used is None:
            check(lib().LGBMB200_LearnerSetFeatureMask(self.handle, None))
        else:
            m = np.ascontiguousarray(feature_used, dtype=np.uint8)
            assert len(m) == self.layout.num_features
            check(lib().LGBMB200_LearnerSetFeatureMask(self.handle, _p(m)))

    # TreeLearner::SetBaggingData(const Dataset* subset, const data_size_t* used_indices, data_size_t num_data)
    def set_bagging_data(self, used_indices) -> None:
        if used_indices is None:
            check(lib().LGBMB200_LearnerSetBaggingData(self.handle, None, C.c_int32(0), C.c_int32(0)))
            return
        if isinstance(used_indices, np.ndarray):
            used_indices = np.ascontiguousarray(used_indices, dtype=np.int32)
            n = len(used_indices)
        else:
            n = used_indices.nbytes // 4 if isinstance(used_indices, DeviceArray) else used_indices.numel()
        ptr, dev = _ptr_of(used_indices)
        check(lib().LGBMB200_LearnerSetBaggingData(self.handle, ptr, C.c_int32(n), C.c_int32(dev)))

    # GOSSStrategy::Bagging on the device (goss.hpp:30-77): gradients / hessians are DeviceArrays, modified in place
    def goss_sample(self, grad_dev, hess_dev, top_rate: float, other_rate: float, seed: int = 0, iteration: int = 0) -> int:
        n = C.c_int32(0)
        check(lib().LGBMB200_LearnerGossSample(self.handle, _ptr_of(grad_dev)[0], _ptr_of(hess_dev)[0], C.c_double(top_rate),
                                               C.c_double(other_rate), C.c_int32(seed), C.c_int32(iteration), C.byref(n)))
        return n.value

    def get_bagging_data(self, n: int) -> np.ndarray:
        out = np.empty(n, np.int32)
        check(lib().LGBMB200_LearnerGetBaggingData(self.handle, _p(out), C.c_int32(n)))
        return out

    # Tree* TreeLearner::Train(const score_t* gradients, const score_t* hessians, bool is_first_tree)
    def train(self, gradients, hessians, is_first_tree: bool = False) -> Tree:
        if isinstance(gradients, np.ndarray):
            gradients = np.ascontiguousarray(gradients, dtype=np.float32)
            hessians = np.ascontiguousarray(hessians, dtype=np.float32)
            assert len(gradients) == self.layout.num_data == len(hessians)
        gp, gd = _ptr_of(gradients)
        hp, hd = _ptr_of(hessians)
        assert gd == hd, "gradients and hessians must live on the same side"
        nl = self.config.num_leaves
        splits = np.zeros(nl - 1, dtype=SPLIT_DTYPE)
        lv, lw = np.zeros(nl), np.zeros(nl)
        lc, ld = np.zeros(nl, np.int32), np.zeros(nl, np.int32)
        t = _CTree(0, _p(splits), _p(lv), _p(lw), _p(lc), _p(ld), 0.0, 0.0, 0.0, 0.0)
        check(lib().LGBMB200_LearnerTrain(self.handle, gp, hp, C.c_int32(gd), C.byref(t)))
        n = t.num_leaves
        tree = Tree(n, splits[:n - 1].copy(), lv[:n].copy(), lw[:n].copy(), lc[:n].copy(), ld[:n].copy(),
                    t.root_sum_gradient, t.root_sum_hessian)
        tree.grad_scale, tree.hess_scale = t.grad_scale, t.hess_scale     # use_quantized_grad: this tree's scales
        return tree

    # void TreeLearner::AddPredictionToScore(const Tree* tree, double* out_score)
    def add_prediction_to_score(self, tree: Tree, out_score) -> None:
        lv = np.ascontiguousarray(tree.leaf_value, dtype=np.float64)
        if isinstance(out_score, np.ndarray):
            assert out_score.dtype == np.float64 and out_score.flags.c_contiguous
        sp, sd = _ptr_of(out_score)
        check(lib().LGBMB200_LearnerAddPredictionToScore(self.handle, _p(lv), C.c_int32(tree.num_leaves), sp, C.c_int32(sd)))

    # GBDT::UpdateScore with a bagging set: every row (bagged or not) through the last tree, device score
    def add_prediction_all_rows(self, tree: Tree, score_dev) -> None:
        lv = np.ascontiguousarray(tree.leaf_value, dtype=np.float64)
        check(lib().LGBMB200_LearnerAddPredictionAllRows(self.handle, _p(lv), C.c_int32(tree.num_leaves), _ptr_of(score_dev)[0]))

    # DataPartition::GetIndexOnLeaf for all leaves of the last tree
    def get_partition(self, num_leaves: int):
        lb, lc = np.zeros(num_leaves, np.int32), np.zeros(num_leaves, np.int32)
        idx = np.full(self.layout.num_data, -1, np.int32)
        check(lib().LGBMB200_LearnerGetPartition(self.handle, _p(lb), _p(lc), _p(idx)))
        return lb, lc, idx

    def get_leaf_histogram(self, leaf: int) -> np.ndarray:
        out = np.zeros((self.layout.num_columns, 256, 2))
        check(lib().LGBMB200_LearnerGetLeafHistogram(self.handle, C.c_int32(leaf), _p(out)))
        return out

    # Dataset::ConstructHistograms on an explicit row set (kernel-level parity + roofline hook)
    def construct_histogram(self, gradients, hessians, indices=None, want_hist: bool = True):
        if isinstance(gradients, np.ndarray):
            gradients = np.ascontiguousarray(gradients, dtype=np.float32)
            hessians = np.ascontiguousarray(hessians, dtype=np.float32)
        gp, gd = _ptr_of(gradients)
        hp, _ = _ptr_of(hessians)
        out = np.zeros((self.layout.num_columns, 256, 2)) if want_hist else None
        ms = C.c_float(0)
        idx = None if indices is None else np.ascontiguousarray(indices, dtype=np.int32)
        check(lib().LGBMB200_LearnerConstructHistogram(self.handle, gp, hp, C.c_int32(gd), None if idx is None else _p(idx),
                                                       C.c_int32(0 if idx is None else len(idx)),
                                                       None if out is None else _p(out), C.byref(ms)))
        return out, ms.value

    # ---- feature-shard bootstrap (see lightgbm_b200/distributed.py)
    def comm_export(self) -> bytes:
        buf = (C.c_uint8 * 64)()
        check(lib().LGBMB200_LearnerCommExport(self.handle, buf))
        return bytes(buf)

    def comm_connect(self, rank: int, world: int, all_handles: bytes, feature_offsets) -> None:
        assert len(all_handles) == 64 * world
        off = np.ascontiguousarray(feature_offsets, dtype=np.int32)
        assert len(off) == world + 1
        hb = (C.c_uint8 * len(all_handles)).from_buffer_copy(all_handles)
        check(lib().LGBMB200_LearnerCommConnect(self.handle, C.c_int32(rank), C.c_int32(world), hb, _p(off)))

    def comm_export_columns(self) -> bytes:
        buf = (C.c_uint8 * 64)()
        check(lib().LGBMB200_LearnerCommExportColumns(self.handle, buf))
        return bytes(buf)

    def comm_share_columns(self, all_column_handles: bytes) -> None:
        """Replicate every rank's partition columns locally (NVLink peer copies); barrier afterwards."""
        hb = (C.c_uint8 * len(all_column_handles)).from_buffer_copy(all_column_handles)
        check(lib().LGBMB200_LearnerCommShareColumns(self.handle, hb))

    def comm_export_pool(self) -> bytes:
        buf = (C.c_uint8 * 64)()
        check(lib().LGBMB200_LearnerCommExportPool(self.handle, buf))
        return bytes(buf)

    def comm_connect_rows(self, rank: int, world: int, comm_handles: bytes, pool_handles: bytes) -> None:
        assert len(comm_handles) == 64 * world == len(pool_handles)
        a = (C.c_uint8 * len(comm_handles)).from_buffer_copy(comm_handles)
        b = (C.c_uint8 * len(pool_handles)).from_buffer_copy(pool_handles)
        check(lib().LGBMB200_LearnerCommConnectRows(self.handle, C.c_int32(rank), C.c_int32(world), a, b))

    def get_leaf_index(self) -> np.ndarray:
        out = np.empty(self.layout.num_data, np.int32)
        check(lib().LGBMB200_LearnerGetLeafIndex(self.handle, _p(out)))
        return out

    def get_leaf_index_range8(self, lo: int, hi: int, out: np.ndarray) -> np.ndarray:
        assert out.dtype == np.uint8 and out.flags.c_contiguous and len(out) >= hi - lo
        check(lib().LGBMB200_LearnerGetLeafIndexRange8(self.handle, C.c_int32(lo), C.c_int32(hi), _p(out)))
        return out

    def timer_start(self) -> None:
        check(lib().LGBMB200_LearnerTimerStart(self.handle))

    def timer_stop(self) -> float:
        ms = C.c_float(0)
        check(lib().LGBMB200_LearnerTimerStop(self.handle, C.byref(ms)))
        return ms.value

    def l2_gradients(self, score_dev, label_dev, grad_dev, hess_dev, n: int) -> None:
        check(lib().LGBMB200_L2Gradients(self.handle, _ptr_of(score_dev)[0], _ptr_of(label_dev)[0],
                                         _ptr_of(grad_dev)[0], _ptr_of(hess_dev)[0], C.c_int32(n)))

    def binary_gradients(self, score_dev, label_dev, grad_dev, hess_dev, n: int, sigmoid: float = 1.0) -> None:
        check(lib().LGBMB200_BinaryGradients(self.handle, _ptr_of(score_dev)[0], _ptr_of(label_dev)[0],
                                             _ptr_of(grad_dev)[0], _ptr_of(hess_dev)[0], C.c_int32(n), C.c_double(sigmoid)))

    def set_profiling(self, enable: bool) -> None:
        check(lib().LGBMB200_LearnerSetProfiling(self.handle, C.c_int32(1 if enable else 0)))

    def hist_stats(self, reset: bool = False):
        ms, rows, n = C.c_double(0), C.c_double(0), C.c_int64(0)
        check(lib().LGBMB200_LearnerHistStats(self.handle, C.c_int32(1 if reset else 0), C.byref(ms), C.byref(rows), C.byref(n)))
        return ms.value, rows.value, n.value

    def profile_by_kind(self) -> dict:
        out = np.zeros(9)
        check(lib().LGBMB200_LearnerProfileByKind(self.handle, _p(out)))
        names = ("_", "prep", "part_flags", "part_count", "part_scatter", "memset", "hist", "scan", "select")
        return {n: float(v) for n, v in zip(names, out) if n != "_"}

    @property
    def kernel_launches(self) -> int:
        return int(lib().LGBMB200_LearnerKernelLaunches(self.handle))

    def free(self):
        if self.handle:
            lib().LGBMB200_LearnerFree(self.handle)
            self.handle = C.c_void_p()

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass
