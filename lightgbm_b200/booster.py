"""Minimal mirror of GBDT::TrainOneIter (reference src/boosting/gbdt.cpp:352-460) around the tree learner,
for the objectives the BASELINE configs need (L2 regression; custom gradients).

Two modes, matching the reference's `boosting_on_gpu_` switch (gbdt.cpp:110-135):
  device_resident=True  : label / score / grad / hess live in HBM; gradients (regression_objective.hpp:127-142),
                          Train and the score update never leave the device ("next" row f-1 of SURVEY.md §8).
  device_resident=False : the caller (or this class) owns host arrays; every iteration copies grad/hess
                          host->device inside Train and the scores device->host, i.e. the path the
                          link-time seam of INTEGRATION.md exercises.
"""
from __future__ import annotations

import math
import os
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from .tree_learner import B200TreeLearner, Config, DeviceArray, Layout, Tree


_POOL: ThreadPoolExecutor | None = None
K_EPSILON = float(np.float32(1e-15))     # kEpsilon (meta.h:54): the float literal, widened


def _host_threads() -> int:
    try:
        return max(1, min(16, len(os.sched_getaffinity(0))))
    except AttributeError:
        return max(1, min(16, os.cpu_count() or 1))


def _parallel_rows(n: int, fn) -> None:
    """Host objectives run row-chunked on a few threads, as the reference's OpenMP loops do
    (regression_objective.hpp:127-142); numpy ufunc inner loops release the GIL."""
    global _POOL
    nt = _host_threads()
    if nt == 1 or n < (1 << 18):
        fn(0, n)
        return
    if _POOL is None:
        _POOL = ThreadPoolExecutor(max_workers=nt)
    per = (n + nt - 1) // nt
    list(_POOL.map(lambda t: fn(t * per, min(n, (t + 1) * per)), range(nt)))


class B200Booster:
    def __init__(self, layout: Layout, label: np.ndarray, config: Config, learning_rate: float = 0.1,
                 boost_from_average: bool = True, device_resident: bool = True, learner: B200TreeLearner | None = None,
                 pinned: bool = False, objective: str = "regression", sigmoid: float = 1.0,
                 data_sample_strategy: str = "bagging", top_rate: float = 0.2, other_rate: float = 0.1, bagging_seed: int = 3):
        assert data_sample_strategy in ("bagging", "goss")
        self.goss = data_sample_strategy == "goss"
        # GOSS lives on the device here; with host buffers it is the reference GBDT's own GOSSStrategy that samples and
        # scores the out-of-bag rows (the drop-in of integration/), not this mirror
        assert not (self.goss and not device_resident), "data_sample_strategy='goss' needs device_resident=True"
        self.top_rate, self.other_rate, self.bagging_seed = float(top_rate), float(other_rate), int(bagging_seed)
        if learner is None:
            learner = B200TreeLearner(config)
            # RegressionL2loss::IsConstantHessian() is true for unweighted L2 (regression_objective.hpp:165-171);
            # BinaryLogloss is not; GOSS rescales hessians (GOSSStrategy::IsHessianChange, goss.hpp:105 -> gbdt.cpp:124).
            # update_custom() on such a learner must pass equal hessians too.
            learner.init(layout, is_constant_hessian=(objective == "regression" and not self.goss))
        self.learner = learner
        self.n = layout.num_data
        self.lr = float(learning_rate)
        self.device_resident = device_resident
        self.label = np.ascontiguousarray(label, dtype=np.float32)
        self.trees: list[Tree] = []
        self.host_ms = {"gradients": 0.0, "train": 0.0, "score": 0.0}   # wall-clock split of update(), host mode
        assert objective in ("regression", "binary")
        self.objective, self.sigmoid = objective, float(sigmoid)
        # BoostFromAverage (gbdt.cpp:327-350): the scores start from the objective's init score, and tree 0 carries it as
        # a bias, only when it is larger than kEpsilon
        self.boost_from_average = bool(boost_from_average)
        init = self._automatic_init_score() if boost_from_average else 0.0
        self.init_score = init if abs(init) > K_EPSILON else 0.0
        self.finished = False          # TrainOneIter returned true: no tree could split (gbdt.cpp:448-456)
        score0 = np.full(self.n, self.init_score, dtype=np.float64)
        if device_resident:
            self.d_label = DeviceArray(self.n * 4).upload(self.label)
            self.d_score = DeviceArray(self.n * 8).upload(score0)
            self.d_grad = DeviceArray(self.n * 4)
            self.d_hess = DeviceArray(self.n * 4)
        else:
            self.score = score0
            if pinned:
                from .tree_learner import PinnedArray
                self._pg, self._ph = PinnedArray(self.n, np.float32), PinnedArray(self.n, np.float32)
                self.grad, self.hess = self._pg.array, self._ph.array
                self.hess[:] = 1.0
            else:
                self.grad = np.empty(self.n, np.float32)
                self.hess = np.ones(self.n, np.float32)

    def update(self) -> Tree:
        """One boosting iteration: gradients -> Train -> Shrinkage -> UpdateScore."""
        if self.device_resident:
            if self.objective == "regression":
                self.learner.l2_gradients(self.d_score, self.d_label, self.d_grad, self.d_hess, self.n)
            else:
                self.learner.binary_gradients(self.d_score, self.d_label, self.d_grad, self.d_hess, self.n, self.sigmoid)
            if self.goss and len(self.trees) >= int(1.0 / self.lr):
                # GOSSStrategy::Bagging (goss.hpp:30-77) on the device: no sampling during the first 1/lr iterations
                self.learner.goss_sample(self.d_grad, self.d_hess, self.top_rate, self.other_rate, self.bagging_seed, len(self.trees))
            tree = self.learner.train(self.d_grad, self.d_hess)
        else:
            t0 = time.perf_counter()
            if self.objective == "regression":
                def l2(lo, hi):    # g = score - label, h = 1
                    np.subtract(self.score[lo:hi], self.label[lo:hi], out=self.grad[lo:hi], casting="unsafe")
                _parallel_rows(self.n, l2)
            else:
                def logloss(lo, hi):
                    lab = np.where(self.label[lo:hi] > 0, 1.0, -1.0)
                    resp = -lab * self.sigmoid / (1.0 + np.exp(lab * self.sigmoid * self.score[lo:hi]))
                    self.grad[lo:hi] = resp
                    self.hess[lo:hi] = np.abs(resp) * (self.sigmoid - np.abs(resp))
                _parallel_rows(self.n, logloss)
            t1 = time.perf_counter()
            tree = self.learner.train(self.grad, self.hess)
            t2 = time.perf_counter()
            self.host_ms["gradients"] += (t1 - t0) * 1e3
            self.host_ms["train"] += (t2 - t1) * 1e3
        if tree.num_leaves <= 1:
            return self._no_split(tree)
        tree.shrinkage(self.lr)
        if self.device_resident:
            if self.goss and len(self.trees) >= int(1.0 / self.lr):
                self.learner.add_prediction_all_rows(tree, self.d_score)      # out-of-bag rows are scored too (gbdt.cpp:505-530)
            else:
                self.learner.add_prediction_to_score(tree, self.d_score)
        else:
            t3 = time.perf_counter()
            self.learner.add_prediction_to_score(tree, self.score)
            self.host_ms["score"] += (time.perf_counter() - t3) * 1e3
        if not self.trees and self.init_score != 0.0:
            tree.add_bias(self.init_score)     # gbdt.cpp:424-427 (first tree carries the average)
        self.trees.append(tree)
        return tree

    def _no_split(self, tree: Tree) -> Tree:
        """TrainOneIter when the tree cannot split (gbdt.cpp:427-456): the first tree becomes the constant init score, a
        later one is the constant 0 and is dropped; either way training has finished."""
        if self.trees:
            tree.as_constant(0.0, self.n)
        else:
            init = self.init_score
            if not self.boost_from_average:
                # the init score the scores never started from is added now, whatever its size
                init = self._automatic_init_score()
                if self.device_resident:
                    self.d_score.upload(self.scores() + init)
                else:
                    self.score += init
            tree.as_constant(init, self.n)
            self.trees.append(tree)
        self.finished = True
        return tree

    def _automatic_init_score(self) -> float:
        """ObjectiveFunction::BoostFromScore: RegressionL2loss the mean label; BinaryLogloss log(p / (1 - p)) / sigmoid
        with p clamped to [kEpsilon, 1 - kEpsilon] (binary_objective.hpp:139-165)."""
        if self.objective == "regression":
            return float(np.mean(self.label, dtype=np.float64))
        pavg = float(np.count_nonzero(self.label > 0)) / self.n
        pavg = max(min(pavg, 1.0 - K_EPSILON), K_EPSILON)
        return math.log(pavg / (1.0 - pavg)) / self.sigmoid

    def update_custom(self, grad, hess) -> Tree:
        """LGBM_BoosterUpdateOneIterCustom (c_api.h:801): caller-provided gradients."""
        tree = self.learner.train(grad, hess)
        tree.shrinkage(self.lr)
        self.trees.append(tree)
        return tree

    def to_model(self, parameters: str = ""):
        """The trees grown so far as a model-text object (GBDT::SaveModelToString): `.to_string()` is loadable by the
        reference's LGBM_BoosterLoadModelFromString, `.predict(X)` scores raw float matrices on the device."""
        from .model import Model, ModelTree
        lay = self.learner.layout
        mfi = int(getattr(lay, "num_total_features", 0) or (int(np.max(lay.feat_real_index)) + 1)) - 1
        obj = "regression" if self.objective == "regression" else f"binary sigmoid:{self.sigmoid:g}"
        return Model([ModelTree.from_learner_tree(t, lay, t.shrink, t.bias) for t in self.trees], max_feature_idx=mfi, objective=obj,
                     parameters=parameters)

    def scores(self) -> np.ndarray:
        if self.device_resident:
            return self.d_score.download(np.float64, self.n)
        return self.score

    def logloss(self) -> float:
        s = self.scores()
        p = 1.0 / (1.0 + np.exp(-self.sigmoid * s))
        y = self.label > 0
        return float(-np.mean(np.where(y, np.log(np.maximum(p, 1e-15)), np.log(np.maximum(1 - p, 1e-15)))))

    def l2(self) -> float:
        s = self.scores()
        return float(np.mean((s - self.label) ** 2))


class RowSlicedHostBooster:
    """Host-buffer L2 boosting for `world` feature-sharded ranks (one process per GPU): every rank holds ALL rows of its
    column slice on the device, but only rows [lo, hi) of the HOST label / score.  Per iteration a rank computes the
    gradients of its own row slice, copies those 4 (hi - lo) bytes host->device from pinned memory, and the full
    gradient vector is assembled on every GPU by one all-gather over NVLink (torch.distributed / NCCL: plumbing); after
    Train it fetches the leaf ids of its own rows (1 byte each) and updates its slice of the host score.  Host work and
    PCIe traffic per rank are 1/world of the single-process path (VERDICT r1 item 5: at 8 GPUs every rank used to
    recompute all N gradients and ship the same 40 MB)."""

    def __init__(self, learner: B200TreeLearner, label_full: np.ndarray, learning_rate: float, rank: int, world: int, dist, torch):
        self.learner, self.lr, self.dist, self.torch = learner, float(learning_rate), dist, torch
        n = len(label_full)
        self.n, self.per = n, (n + world - 1) // world
        self.lo, self.hi = min(n, rank * self.per), min(n, (rank + 1) * self.per)
        init = float(np.mean(label_full, dtype=np.float64))
        self.label = np.ascontiguousarray(label_full[self.lo:self.hi], dtype=np.float32)
        self.score = np.full(self.hi - self.lo, init, dtype=np.float64)
        self.h_grad = torch.zeros(self.per, dtype=torch.float32).pin_memory()
        self.grad = self.h_grad.numpy()
        self.d_local = torch.zeros(self.per, dtype=torch.float32, device="cuda")
        self.d_full = torch.zeros(self.per * world, dtype=torch.float32, device="cuda")
        self.d_hess = torch.ones(self.per * world, dtype=torch.float32, device="cuda")
        self.leaf8 = np.zeros(self.per, dtype=np.uint8)
        self.host_ms = {"gradients": 0.0, "train": 0.0, "score": 0.0}
        self.trees = []

    def update(self) -> Tree:
        t0 = time.perf_counter()
        m = self.hi - self.lo

        def l2(a, b):
            np.subtract(self.score[a:b], self.label[a:b], out=self.grad[a:b], casting="unsafe")
        _parallel_rows(m, l2)
        t1 = time.perf_counter()
        self.d_local.copy_(self.h_grad, non_blocking=True)
        self.dist.all_gather_into_tensor(self.d_full, self.d_local)
        self.torch.cuda.current_stream().synchronize()         # the learner runs on its own stream
        tree = self.learner.train(self.d_full, self.d_hess)
        t2 = time.perf_counter()
        tree.shrinkage(self.lr)
        if tree.num_leaves > 1:
            self.learner.get_leaf_index_range8(self.lo, self.hi, self.leaf8)
            lv = tree.leaf_value

            def add(a, b):
                self.score[a:b] += lv[self.leaf8[a:b]]
            _parallel_rows(m, add)
        t3 = time.perf_counter()
        self.host_ms["gradients"] += (t1 - t0) * 1e3; self.host_ms["train"] += (t2 - t1) * 1e3; self.host_ms["score"] += (t3 - t2) * 1e3
        self.trees.append(tree)
        return tree


def train(params: dict, train_set, num_boost_round: int = 100) -> B200Booster:
    """`lightgbm.train(params, lgb.Dataset(X, y), num_boost_round)` for the objectives this mirror knows (regression,
    binary) — raw floats in, binned on the device (dataset.py), boosted with gradients and scores resident in HBM."""
    p = dict(params or {})
    obj = p.get("objective", "regression")
    obj = {"regression_l2": "regression", "l2": "regression", "mse": "regression"}.get(obj, obj)
    cfg = Config(num_leaves=int(p.get("num_leaves", 31)), max_depth=int(p.get("max_depth", -1)),
                 min_data_in_leaf=int(p.get("min_data_in_leaf", 20)), min_sum_hessian_in_leaf=float(p.get("min_sum_hessian_in_leaf", 1e-3)),
                 lambda_l1=float(p.get("lambda_l1", 0.0)), lambda_l2=float(p.get("lambda_l2", 0.0)),
                 min_gain_to_split=float(p.get("min_gain_to_split", 0.0)))
    train_set.params = {**p, **train_set.params}
    lay = train_set.construct().layout
    lay.num_total_features = train_set.num_feature()
    b = B200Booster(lay, train_set.get_label(), cfg, learning_rate=float(p.get("learning_rate", 0.1)),
                    boost_from_average=str(p.get("boost_from_average", "true")).lower() not in ("false", "0"),
                    objective=obj, sigmoid=float(p.get("sigmoid", 1.0)),
                    data_sample_strategy=p.get("data_sample_strategy", "bagging"), top_rate=float(p.get("top_rate", 0.2)),
                    other_rate=float(p.get("other_rate", 0.1)), bagging_seed=int(p.get("bagging_seed", 3)))
    for _ in range(num_boost_round):
        b.update()
        if b.finished:
            break
    return b
