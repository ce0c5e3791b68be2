"""Model text writer / reader and prediction (SURVEY.md §8 f-4), numerical splits, one tree per iteration.

  * `ModelTree.from_learner_tree` replays the learner's split records the way Tree::Split does
    (reference include/LightGBM/tree.h:543-585, src/io/tree.cpp:65-79) into the arrays of the model text;
  * `Model.to_string` writes GBDT::SaveModelToString / Tree::ToString (src/boosting/gbdt_model_text.cpp:314-400,
    src/io/tree.cpp:343-413): same keys, same order, same number formats ({:g} and {:.17g}), so that
    LGBM_BoosterLoadModelFromString of the unmodified reference loads it;
  * `Model.from_string` reads a model text written by either side (gbdt_model_text.cpp:421-620, tree.cpp:686-800);
  * `Model.predict` scores a dense float matrix on the device (csrc/predict.cuh) — raw scores bit-identical to
    LGBM_BoosterPredictForMat(C_API_PREDICT_RAW_SCORE), and the objective's output transform on top.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field

import numpy as np

from ._lib import check, lib
from .tree_learner import Layout, Tree, _p, round_to_zero


def _g(x) -> str:
    return format(float(x), "g")


def _g17(x) -> str:
    return format(float(x), ".17g")


def _join(a, fmt) -> str:
    return " ".join(fmt(v) for v in a)


@dataclass
class ModelTree:
    """The arrays Tree::ToString writes."""
    num_leaves: int
    split_feature: np.ndarray        # real feature index, int32 [num_leaves - 1]
    split_gain: np.ndarray           # float32
    threshold: np.ndarray            # float64 real-valued thresholds
    decision_type: np.ndarray        # int8: bit 0 categorical, bit 1 default left, bits 2..3 missing type
    left_child: np.ndarray
    right_child: np.ndarray
    leaf_value: np.ndarray
    leaf_weight: np.ndarray
    leaf_count: np.ndarray
    internal_value: np.ndarray
    internal_weight: np.ndarray
    internal_count: np.ndarray
    shrinkage: float = 1.0

    @staticmethod
    def from_learner_tree(t: Tree, layout: Layout, shrinkage: float = 1.0, bias: float = 0.0) -> "ModelTree":
        """`t`: the learner's tree with UNSHRUNK split outputs in its split records and its final leaf values already
        shrunk / biased by the caller (B200Booster.update); `shrinkage`, `bias`: what the caller applied, for the internal
        values (Tree::Shrinkage / Tree::AddBias, tree.h:188-230)."""
        assert layout.bin_upper_bound, "the layout carries no bin upper bounds: real-valued thresholds are unknown"
        L = t.num_leaves
        n = L - 1
        sf = np.zeros(n, np.int32); sg = np.zeros(n, np.float32); th = np.zeros(n, np.float64); dt = np.zeros(n, np.int8)
        lc = np.zeros(n, np.int32); rc = np.zeros(n, np.int32)
        iv = np.zeros(n, np.float64); iw = np.zeros(n, np.float64); ic = np.zeros(n, np.int32)
        value = np.zeros(L, np.float64)
        parent = np.full(L, -1, np.int64)
        for node in range(n):
            s = t.splits[node]
            leaf, new_leaf = int(s["leaf"]), node + 1
            p = parent[leaf]
            if p >= 0:
                if lc[p] == ~leaf:
                    lc[p] = node
                else:
                    rc[p] = node
            f = int(s["feature"])
            sf[node] = layout.feat_real_index[f]
            sg[node] = np.float32(s["gain"])
            th[node] = layout.bin_upper_bound[f][int(s["threshold"])]          # Dataset::RealThreshold (dataset.h:853)
            dt[node] = (2 if s["default_left"] else 0) | (int(layout.feat_missing[f]) << 2)
            lc[node], rc[node] = ~leaf, ~new_leaf
            parent[leaf] = parent[new_leaf] = node
            iw[node] = s["left_sum_hessian"] + s["right_sum_hessian"]
            iv[node] = value[leaf]
            ic[node] = s["left_count"] + s["right_count"]
            lo, ro = float(s["left_output"]), float(s["right_output"])
            value[leaf] = 0.0 if np.isnan(lo) else lo
            value[new_leaf] = 0.0 if np.isnan(ro) else ro
        iv = round_to_zero(iv * shrinkage)
        if bias != 0.0:
            iv = round_to_zero(iv + bias)
        return ModelTree(L, sf, sg, th, dt, lc, rc, round_to_zero(t.leaf_value), np.asarray(t.leaf_weight, np.float64).copy(),
                         np.asarray(t.leaf_count, np.int32).copy(), iv, iw, ic,
                         shrinkage=1.0 if bias != 0.0 else float(shrinkage))

    # Tree::ToString
    def to_string(self) -> str:
        n = self.num_leaves - 1
        out = [f"num_leaves={self.num_leaves}", "num_cat=0",
               "split_feature=" + _join(self.split_feature[:n], str),
               "split_gain=" + _join(self.split_gain[:n], _g),
               "threshold=" + _join(self.threshold[:n], _g17),
               "decision_type=" + _join(self.decision_type[:n], lambda v: str(int(v))),
               "left_child=" + _join(self.left_child[:n], str),
               "right_child=" + _join(self.right_child[:n], str),
               "leaf_value=" + _join(self.leaf_value[:self.num_leaves], _g17),
               "leaf_weight=" + _join(self.leaf_weight[:self.num_leaves], _g17),
               "leaf_count=" + _join(self.leaf_count[:self.num_leaves], str),
               "internal_value=" + _join(self.internal_value[:n], _g),
               "internal_weight=" + _join(self.internal_weight[:n], _g),
               "internal_count=" + _join(self.internal_count[:n], str),
               "is_linear=0",
               "shrinkage=" + _g(self.shrinkage), "", ""]
        return "\n".join(out)

    @staticmethod
    def from_string(block: str) -> "ModelTree":
        kv = {}
        for line in block.split("\n"):
            if "=" in line:
                k, v = line.split("=", 1)
                kv[k.strip()] = v.strip()
        L = int(kv["num_leaves"])
        if int(kv.get("num_cat", "0")) != 0:
            raise ValueError("categorical splits are not supported")
        if int(kv.get("is_linear", "0")) != 0:
            raise ValueError("linear trees are not supported")

        def arr(key, dtype, n):
            s = kv.get(key, "")
            a = np.array(s.split(), dtype=np.float64 if dtype != np.int64 else np.int64) if s else np.zeros(0)
            assert len(a) >= n, f"{key}: {len(a)} values, {n} expected"
            return a[:n].astype(dtype)
        n = L - 1
        return ModelTree(L, arr("split_feature", np.int32, n), arr("split_gain", np.float32, n), arr("threshold", np.float64, n),
                         arr("decision_type", np.int8, n), arr("left_child", np.int32, n), arr("right_child", np.int32, n),
                         arr("leaf_value", np.float64, L), arr("leaf_weight", np.float64, L) if "leaf_weight" in kv else np.zeros(L),
                         arr("leaf_count", np.int32, L) if "leaf_count" in kv else np.zeros(L, np.int32),
                         arr("internal_value", np.float64, n), arr("internal_weight", np.float64, n) if "internal_weight" in kv else np.zeros(n),
                         arr("internal_count", np.int32, n), shrinkage=float(kv.get("shrinkage", "1")))


@dataclass
class Model:
    """A boosted model: what GBDT::SaveModelToString writes (num_class = 1)."""
    trees: list = field(default_factory=list)
    max_feature_idx: int = 0
    objective: str = "regression"                  # ObjectiveFunction::ToString(): "regression", "binary sigmoid:1"
    feature_names: list = field(default_factory=list)
    feature_infos: list = field(default_factory=list)
    parameters: str = ""
    _pred: object = None

    # --- writer
    def to_string(self) -> str:
        names = self.feature_names or [f"Column_{i}" for i in range(self.max_feature_idx + 1)]
        infos = self.feature_infos or ["none"] * (self.max_feature_idx + 1)
        head = ["tree", "version=v4", "num_class=1", "num_tree_per_iteration=1", "label_index=0",
                f"max_feature_idx={self.max_feature_idx}", f"objective={self.objective}",
                "feature_names=" + " ".join(names), "feature_infos=" + " ".join(infos)]
        blocks = [f"Tree={i}\n" + t.to_string() + "\n" for i, t in enumerate(self.trees)]
        head.append("tree_sizes=" + " ".join(str(len(b.encode())) for b in blocks))
        text = "\n".join(head) + "\n\n" + "".join(blocks) + "end of trees\n"
        imp = self.feature_importance()
        pairs = sorted(((int(v), names[i]) for i, v in enumerate(imp) if int(v) > 0), key=lambda p: -p[0])       # stable: ties keep feature order
        text += "\nfeature_importances:\n" + "".join(f"{n}={v}\n" for v, n in pairs)
        if self.parameters:
            text += "\nparameters:\n" + self.parameters + "\nend of parameters\n"
        return text

    def feature_importance(self) -> np.ndarray:
        """split counts (GBDT::FeatureImportance, importance_type = 0: splits with positive gain)"""
        imp = np.zeros(self.max_feature_idx + 1, np.float64)
        for t in self.trees:
            for i in range(t.num_leaves - 1):
                if t.split_gain[i] > 0:
                    imp[t.split_feature[i]] += 1.0
        return imp

    # --- reader
    @staticmethod
    def from_string(text: str) -> "Model":
        head, _, rest = text.partition("\nTree=")
        kv = {}
        for line in head.split("\n"):
            if "=" in line:
                k, v = line.split("=", 1)
                kv[k] = v
        if int(kv.get("num_class", "1")) != 1 or int(kv.get("num_tree_per_iteration", "1")) != 1:
            raise ValueError("multi-class models are not supported")
        m = Model(max_feature_idx=int(kv["max_feature_idx"]), objective=kv.get("objective", "regression").strip(),
                  feature_names=kv.get("feature_names", "").split(), feature_infos=kv.get("feature_infos", "").split())
        body = ("Tree=" + rest) if rest else ""
        body, _, tail = body.partition("end of trees")
        for block in body.split("Tree=")[1:]:
            m.trees.append(ModelTree.from_string(block.split("\n", 1)[1]))
        if "\nparameters:\n" in tail:
            m.parameters = tail.split("\nparameters:\n", 1)[1].split("\nend of parameters", 1)[0]
        return m

    # --- prediction on the device
    def _predictor(self, device: int = -1):
        if self._pred is None:
            T = len(self.trees)
            nl = np.array([t.num_leaves for t in self.trees], np.int32)
            cat = lambda k, dt: (np.concatenate([getattr(t, k)[:t.num_leaves - 1] for t in self.trees]).astype(dt) if T else np.zeros(0, dt))  # noqa: E731
            sf, th, dtp = cat("split_feature", np.int32), cat("threshold", np.float64), cat("decision_type", np.int8)
            lc, rc = cat("left_child", np.int32), cat("right_child", np.int32)
            lv = np.concatenate([t.leaf_value[:t.num_leaves] for t in self.trees]).astype(np.float64) if T else np.zeros(0)
            h = C.c_void_p()
            check(lib().LGBMB200_PredictorCreate(C.c_int32(device), C.c_int32(T), _p(nl), _p(sf), _p(th), _p(dtp), _p(lc), _p(rc), _p(lv),
                                                 C.c_int32(self.max_feature_idx), C.byref(h)))
            self._pred = h
        return self._pred

    def predict_raw(self, X, return_ms: bool = False, data_shape: tuple | None = None, out=None):
        """Raw scores of the rows of X.  `X`: a host row-major matrix, or a (DeviceArray, dtype) pair already in HBM (then
        pass data_shape = (rows, cols)).  `out`: None for a host float64 array, or a DeviceArray of at least 8 * rows bytes
        that receives the scores and is returned.  Input and output both on the device run as one launch, nothing staged."""
        if isinstance(X, tuple):
            dev, dtype = X
            rows, cols = (int(v) for v in data_shape)
            src, code, on_dev = dev.ptr, (0 if np.dtype(dtype) == np.float32 else 1), 1
        else:
            X = np.ascontiguousarray(X)
            if X.dtype not in (np.float32, np.float64):
                X = X.astype(np.float64)
            assert X.ndim == 2
            (rows, cols), src, code, on_dev = X.shape, _p(X), (0 if X.dtype == np.float32 else 1), 0
        if out is None:
            res = np.empty(rows, np.float64)
            dst, out_dev = _p(res), 0
        else:
            assert out.nbytes >= 8 * rows
            res, dst, out_dev = out, out.ptr, 1
        ms = C.c_float(0)
        check(lib().LGBMB200_PredictorPredict(self._predictor(), src, C.c_int32(code), C.c_int32(rows), C.c_int32(cols),
                                              C.c_int32(on_dev), dst, C.c_int32(out_dev), C.byref(ms)))
        return (res, float(ms.value)) if return_ms else res

    def predict(self, X: np.ndarray, raw_score: bool = False) -> np.ndarray:
        raw = self.predict_raw(X)
        if raw_score or not self.objective.startswith("binary"):
            return raw
        sig = 1.0
        for tok in self.objective.split():
            if tok.startswith("sigmoid:"):
                sig = float(tok.split(":", 1)[1])
        return 1.0 / (1.0 + np.exp(-sig * raw))          # BinaryLogloss::ConvertOutput (binary_objective.hpp:167-169)

    def free(self):
        if self._pred is not None:
            lib().LGBMB200_PredictorFree(self._pred)
            self._pred = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass
