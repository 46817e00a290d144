"""Generates tests/golden/airfoil_cv_case.npz from the reference's data (the GPU tests never read the reference).

All 1503 rows of data/airfoil.csv: the five features standardised as commons/util/Scaling.scala:10-25 does, the raw
labels; the 10-fold split of seed 7 (oracle.cross_validation.fold_assignment); a fixed theta of Airfoil.scala's kernel
`1*ARDRBFKernel(5) + 1.const*EyeKernel` with sigma2 = 1e-4; and the oracle's BCM value and gradient of every fold's
training set at that theta, experts of 100 points."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import oracle                                         # noqa: E402
from oracle.cross_validation import fold_assignment, fold_bcm_objective   # noqa: E402

REF_DATA = "/root/reference/data"
SEED, FOLDS, N_E, SIGMA2 = 7, 10, 100, 1e-4


def main():
    raw = np.loadtxt(os.path.join(REF_DATA, "airfoil.csv"), delimiter=",")
    X = oracle.scale(raw[:, :5])
    y = raw[:, 5].copy()
    fold_of = fold_assignment(len(X), FOLDS, SEED)
    user = lambda: 1.0 * oracle.ARDRBFKernel(5) + oracle.const(1.0) * oracle.EyeKernel()
    factory = oracle.ppa.get_kernel(user, SIGMA2)
    theta = np.array([55.0, 0.9, 0.35, 1.4, 0.25, 1.1])      # a plausible optimum (scale, five ARD betas)
    vals, grads = [], []
    for k in range(FOLDS):
        v, g = fold_bcm_objective(X, y, fold_of, k, factory, N_E, theta)
        vals.append(v)
        grads.append(g)
    np.savez_compressed(os.path.join(HERE, "airfoil_cv_case.npz"), X=X, y=y, fold_of=fold_of, seed=SEED, theta=theta,
                        sigma2=SIGMA2, n_e=N_E, bcm_nll=np.array(vals), bcm_grad=np.array(grads))
    print("airfoil_cv: N=%d folds=%s nll=%s" % (len(X), np.bincount(fold_of), np.round(vals, 4)))


if __name__ == "__main__":
    main()
