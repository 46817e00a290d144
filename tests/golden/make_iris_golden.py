"""Generates tests/golden/iris_case.npz from the reference's data/iris.csv (the other fixtures come from make_golden.py,
whose outputs this script leaves untouched).

iris_case.npz -- the reference's multiclass example, classification/examples/Iris.scala: OneVsRest over
GaussianProcessClassifier with datasetSizeForExpert 20 and activeSetSize 30, the default kernel RBFKernel() + 1e-3 Eye,
tol 1e-6, and Iris.scala's label map (versicolor 0, setosa 1, virginica 2).  A fixed split (120 train / 30 test), a
fixed active set and hand-set sigma per class (the point of the fixture is identical inputs, not the optimiser).
Outputs come from the fp64 oracle (oracle/one_vs_rest.py): per-class latent modes, magic vectors and raw test
predictions.

Run:  python tests/golden/make_iris_golden.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import oracle                                                        # noqa: E402
from oracle.one_vs_rest import one_vs_rest_fixed_theta, one_vs_rest_model_outputs   # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
REF_DATA = "/root/reference/data"
NAME2INDEX = {"Iris-versicolor": 0, "Iris-setosa": 1, "Iris-virginica": 2}


def iris():
    rows = [line.strip().split(",") for line in open(os.path.join(REF_DATA, "iris.csv")) if line.strip()]
    X = np.array([[float(v) for v in r[:4]] for r in rows])
    y = np.array([float(NAME2INDEX[r[4]]) for r in rows])
    rng = np.random.default_rng(20261015)
    perm = rng.permutation(len(X))
    test_idx, train_idx = np.sort(perm[:30]), np.sort(perm[30:])
    active_idx = np.sort(rng.permutation(len(train_idx))[:30])
    Xtr, ytr, Xte = X[train_idx], y[train_idx], X[test_idx]
    Z = Xtr[active_idx]
    thetas = np.array([[0.9], [1.6], [1.2]])                        # sigma per class
    factory = oracle.get_kernel(lambda: oracle.RBFKernel(1.0), 1e-3)
    per_class = one_vs_rest_fixed_theta(Xtr, ytr, 3, factory, thetas, Z, 20, 1e-6)
    latent = np.stack([f for f, _ in per_class])
    magic = np.stack([p.magic_vector for _, p in per_class])
    raw_cols = np.stack([p.predict_many(Xte)[0] for _, p in per_class])
    raw, pred = one_vs_rest_model_outputs(raw_cols)
    np.savez_compressed(os.path.join(OUT, "iris_case.npz"), X=X, y=y, train_idx=train_idx, test_idx=test_idx,
                        active_idx=active_idx, thetas=thetas, sigma2=1e-3, tol=1e-6, dataset_size_for_expert=20,
                        latent=latent, magic_vector=magic, raw=raw, prediction=pred)
    print("iris: train %d test %d m %d  hold-out accuracy %.3f  |raw|max %.3f" %
          (len(Xtr), len(Xte), len(Z), np.mean(pred == y[test_idx]), np.abs(raw).max()))


if __name__ == "__main__":
    iris()
