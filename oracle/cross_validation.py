"""CPU restatement (test infrastructure) of the cross-validation the reference's regression examples run
(regression/examples/GPExample.scala:17-27, Airfoil.scala:18-24, Synthetics.scala:25-33): Spark 3.1's CrossValidator with
a RegressionEvaluator and a ParamGridBuilder grid.  Spark's source is not part of this project; each step below restates
Spark 3.1's documented behaviour.

- Folds: Spark's MLUtils.kFold draws per partition and is not reproducible; the project's split is
  fold(i) = floor(u(seed, 200, i) * numFolds) with the K-means generator `u` (oracle.kmeans).
- Split: fold k's training set is every row outside fold k, in row order (Spark filters the frame, keeping its order);
  its validation set is fold k's rows.
- Experts: the training set is grouped as any training shard, GPC:26-31 (oracle.ppa.get_expert_labels_and_kernels).
- Grid: the Cartesian product of the added grids; the first param added varies fastest (each later param's values form
  the outer loop of Spark's flatMap build).
- Metrics: RegressionMetrics without weights and without throughOrigin.
- Model selection: each map's metric summed over the folds in order and divided by numFolds; the first best map wins
  (Scala's maxBy / minBy), larger being better for r2 and var only."""
from __future__ import annotations

import math

import numpy as np

from .kmeans import u
from .ppa import get_expert_labels_and_kernels
from .regression import bcm_objective


def fold_assignment(n: int, num_folds: int, seed: int) -> np.ndarray:
    return np.array([math.floor(u(seed, 200, i) * num_folds) for i in range(n)], dtype=np.int64)


def split(fold_of: np.ndarray, k: int):
    """(training row indices, validation row indices) of fold k, each in row order."""
    idx = np.arange(len(fold_of))
    return idx[fold_of != k], idx[fold_of == k]


def fold_experts(X, y, fold_of, k: int, kernel_factory, dataset_size_for_expert: int):
    train, _ = split(fold_of, k)
    return get_expert_labels_and_kernels(X[train], y[train], kernel_factory, dataset_size_for_expert)


def fold_bcm_objective(X, y, fold_of, k: int, kernel_factory, dataset_size_for_expert: int, theta):
    """The BCM objective (GPR:55-68 summed over the experts, GPC:73-78) of fold k's training set at theta."""
    return bcm_objective(fold_experts(X, y, fold_of, k, kernel_factory, dataset_size_for_expert), np.asarray(theta))


def param_grid(grid):
    """grid: [(name, values), ...] in the order the params were added."""
    maps = [{}]
    for name, values in grid:
        new = []
        for v in values:
            for m in maps:
                mm = dict(m)
                mm[name] = v
                new.append(mm)
        maps = new
    return maps


def metric(name: str, y, p) -> float:
    y = [float(v) for v in y]
    p = [float(v) for v in p]
    n = len(y)
    ybar = sum(y) / n
    ss_err = sum((a - b) ** 2 for a, b in zip(y, p))
    if name == "mse":
        return ss_err / n
    if name == "rmse":
        return math.sqrt(ss_err / n)
    if name == "mae":
        return sum(abs(a - b) for a, b in zip(y, p)) / n
    if name == "r2":
        return 1.0 - ss_err / sum((a - ybar) ** 2 for a in y)
    if name == "var":
        return sum((b - ybar) ** 2 for b in p) / n
    raise ValueError(name)


def larger_is_better(name: str) -> bool:
    return name in ("r2", "var")


def best_index(avg_metrics, name: str) -> int:
    best = 0
    for i, v in enumerate(avg_metrics):
        if (v > avg_metrics[best]) if larger_is_better(name) else (v < avg_metrics[best]):
            best = i
    return best
