"""CPU restatement (test infrastructure) of the model selection the reference's classification examples run
(classification/examples/MNIST.scala:34-40, Iris.scala:29-35): Spark 3.1's TrainValidationSplit with a
MulticlassClassificationEvaluator.  Spark's source is not part of this project; each step below restates Spark 3.1's
documented behaviour.

- Split: Spark's randomSplit depends on the partitioning and is not reproducible; the project's split trains row i iff
  u(seed, 201, i) < trainRatio, with the K-means generator `u` (oracle.kmeans).  Both sides keep their row order.
- Metrics: MulticlassMetrics without weights.  Per true label l (ascending): n_l rows, tp_l rows predicted l, fp_l other
  rows predicted l; precision_l = tp_l / (tp_l + fp_l) (0 when l is never predicted), recall_l = tp_l / n_l,
  f1_l = 2 p r / (p + r) (0 when p + r = 0).  weightedPrecision, weightedRecall and f1 sum the per-label value times
  n_l / n over the labels in order; accuracy is sum tp_l / n.  All are larger-is-better.
- Model selection: the first map with the best validation metric wins (Scala's maxBy / minBy).
- Binary pipeline at fixed theta: the Laplace loop from f = 0 per expert (GPCls:60), the projected process with
  y := f (GPCls:62-65), class 1 iff f* > 0."""
from __future__ import annotations

import numpy as np

from .classification import classification_likelihood_and_gradient, classification_model_outputs
from .kmeans import u
from .ppa import get_expert_labels_and_kernels, group_for_experts, projected_process

METRICS = ("f1", "accuracy", "weightedPrecision", "weightedRecall")


def train_mask(n: int, train_ratio: float, seed: int) -> np.ndarray:
    return np.array([u(seed, 201, i) < train_ratio for i in range(n)], dtype=bool)


def split(mask: np.ndarray):
    """(training row indices, validation row indices), each in row order."""
    idx = np.arange(len(mask))
    return idx[mask], idx[~mask]


def metric(name: str, y, p) -> float:
    y = [float(v) for v in y]
    p = [float(v) for v in p]
    n = len(y)
    if name == "accuracy":
        return sum(1 for a, b in zip(y, p) if a == b) / n
    if name not in METRICS:
        raise ValueError(name)
    total = 0.0
    for label in sorted(set(y)):
        n_l = sum(1 for a in y if a == label)
        tp = sum(1 for a, b in zip(y, p) if a == label and b == label)
        fp = sum(1 for a, b in zip(y, p) if a != label and b == label)
        precision = tp / (tp + fp) if tp + fp > 0 else 0.0
        recall = tp / n_l
        if name == "weightedPrecision":
            v = precision
        elif name == "weightedRecall":
            v = recall
        else:
            v = 2.0 * precision * recall / (precision + recall) if precision + recall > 0.0 else 0.0
        total += v * n_l / n
    return total


def best_index(metrics, larger_is_better: bool) -> int:
    best = 0
    for i, v in enumerate(metrics):
        if (v > metrics[best]) if larger_is_better else (v < metrics[best]):
            best = i
    return best


def binary_fixed_theta_predictions(X_train, y_train, X_val, kernel_factory, theta, active_set,
                                   dataset_size_for_expert: int, tol: float):
    """Validation predictions of the binary classifier trained at fixed theta (maxIter = 0): (f*, prediction)."""
    experts = get_expert_labels_and_kernels(X_train, y_train, kernel_factory, dataset_size_for_expert)
    fk = []
    for (ye, ke), idx in zip(experts, group_for_experts(len(X_train), dataset_size_for_expert)):
        f = np.zeros(len(ye))
        classification_likelihood_and_gradient(ye, f, ke, theta, tol)
        fk.append((f, ke))
    predictor, _, _ = projected_process(fk, active_set, kernel_factory, theta)
    fstar = predictor.predict_many(X_val)[0]
    return fstar, classification_model_outputs(fstar)[2]
