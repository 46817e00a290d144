"""CPU restatement (test infrastructure) of cross-validation over one-vs-rest, as the reference's Iris example runs it
(classification/examples/Iris.scala: a CrossValidator over `new OneVsRest().setClassifier(gp)`).  The split, the folds
and the model selection are oracle.cross_validation's; each fold model is oracle.one_vs_rest's on the fold's training
rows.  Spark's source is not part of this project; the restatement follows Spark 3.1's documented behaviour:
fold k's model is OneVsRest.fit on fold k's training rows, so its class count is max(label over those rows) + 1, which
may be below the class count of all rows; each class runs the binary pipeline."""
from __future__ import annotations

import numpy as np

from .cross_validation import split
from .one_vs_rest import one_vs_rest_fixed_theta, one_vs_rest_model_outputs


def fold_one_vs_rest_fixed_theta(X, y, fold_of, k: int, kernel_factory, thetas, active_set,
                                 dataset_size_for_expert: int, tol: float):
    """Fold k's one-vs-rest model at fixed hyper-parameters thetas[c] (maxIter = 0) and a fixed active set, on its
    training rows, and its validation outputs: (C_k, per class (latent modes in training-row order, magic vector), raw
    n_val x C_k, prediction)."""
    train, val = split(fold_of, k)
    num_classes = int(np.max(y[train])) + 1
    classes = one_vs_rest_fixed_theta(X[train], y[train], num_classes, kernel_factory, thetas, active_set,
                                      dataset_size_for_expert, tol)
    latents = np.stack([pred.predict_many(X[val])[0] for _, pred in classes])
    raw, prediction = one_vs_rest_model_outputs(latents)
    return num_classes, [(f, pred.magic_vector) for f, pred in classes], raw, prediction
