"""One-vs-rest over the binary GP classifier (TEST INFRASTRUCTURE -- see oracle/__init__.py).

Spark 3.1's `ml/classification/OneVsRest.scala` / `OneVsRestModel` are not part of the reference project; the reference's
own multiclass example (classification/examples/Iris.scala) wraps its binary classifier in them.  Restated here from
Spark's documented behaviour, not from its source:
  - numClasses = max(label) + 1; class c's binary model is trained on the labels (y == c) ? 1 : 0 with the wrapped
    classifier's params;
  - rawPrediction is the vector over classes of each class model's rawPrediction(1); prediction is its argmax, the
    first maximum winning a tie; there is no probability column.
The one deviation of the product (spark_gp_b200.OneVsRest): a label that is not a non-negative integer raises
ValueError, where Spark silently leaves such a row out of every class's positives.
"""
from __future__ import annotations

import numpy as np

from .classification import classification_likelihood_and_gradient, classification_model_outputs
from .ppa import get_expert_labels_and_kernels, group_for_experts, projected_process


def one_vs_rest_binary_labels(y: np.ndarray, num_classes: int):
    """(y == c) ? 1.0 : 0.0 for every class c: num_classes x n."""
    y = np.asarray(y, dtype=np.float64)
    return np.stack([(y == c).astype(np.float64) for c in range(num_classes)])


def one_vs_rest_model_outputs(class_latents):
    """OneVsRestModel for per-class latent predictions (num_classes x n): rawPrediction[:, c] is class c's binary
    rawPrediction(1) (classification_model_outputs' raw[:, 1] = f_c), prediction the first argmax as float64."""
    raw = np.stack([classification_model_outputs(f)[0][:, 1] for f in class_latents], axis=-1)
    pred = np.zeros(raw.shape[0])
    best = raw[:, 0].copy()
    for c in range(1, raw.shape[1]):                 # strictly greater: the first maximum keeps a tie
        better = raw[:, c] > best
        pred[better] = c
        best[better] = raw[better, c]
    return raw, pred


def one_vs_rest_fixed_theta(X, y, num_classes, kernel_factory, thetas, active_set, dataset_size_for_expert, tol):
    """The binary pipeline per class at fixed hyper-parameters theta_c: the Laplace loop from f = 0 (GPCls:60), then the
    projected process with y := f_c (GPCls:62-65).  Returns per class (latent modes in point order, predictor)."""
    out = []
    n = len(X)
    groups = group_for_experts(n, dataset_size_for_expert)
    for c, yc in enumerate(one_vs_rest_binary_labels(y, num_classes)):
        experts = get_expert_labels_and_kernels(X, yc, kernel_factory, dataset_size_for_expert)
        f_all = np.zeros(n)
        fk = []
        for (ye, ke), idx in zip(experts, groups):
            f = np.zeros(len(ye))
            classification_likelihood_and_gradient(ye, f, ke, thetas[c], tol)
            f_all[idx] = f
            fk.append((f, ke))
        pred, _, _ = projected_process(fk, active_set, kernel_factory, thetas[c])
        out.append((f_all, pred))
    return out
