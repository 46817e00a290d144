"""Per-expert Laplace approximation for binary GP classification
(TEST INFRASTRUCTURE -- see oracle/__init__.py).

Follows `classification/GaussianProcessClassifier.scala:74-129` (GPCls) line by
line, including its quirks (d3logP sign at :118; f is warm-started and mutated
in place at :105).
"""
from __future__ import annotations

import numpy as np
import scipy.linalg as sla


def _sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


def classification_likelihood_and_gradient(y: np.ndarray, f: np.ndarray, kernel, x: np.ndarray, tol: float,
                                           trace=None):
    """GPCls:74-129.  Mutates `f` in place (the expert's latent mode).  Returns (-logZ, -gradLogZ).

    `trace`, when a list, receives one dict per Newton iteration -- step, cand, old_obj and new_obj (before the
    comparison), accepted, and max_abs_f (max |f| after the iteration) -- and then one {"exit": reason}: "converged"
    (|old_obj - new_obj| <= tol), "step" (step <= tol) or "none" (no iteration ran).  It changes no result."""
    kernel.set_hyperparameters(x)
    K, derivatives = kernel.training_kernel_and_derivative()
    n = len(y)
    old_obj = -np.inf
    new_obj = -np.finfo(np.float64).max            # Double.MinValue
    L = np.zeros((n, n))
    sqrtW = np.zeros((n, n))
    pi = np.zeros(n)
    a = np.zeros(n)
    grad_log_p = np.zeros(n)
    I = np.eye(n)
    step = 1.0
    iterations = 0
    while abs(old_obj - new_obj) > tol and step > tol:                      # :91
        pi = _sigmoid(f)
        W = np.diag(pi * (1.0 - pi))
        sqrtW = np.sqrt(W)
        sw = np.diag(sqrtW)
        B = np.outer(sw, sw) * K + I                                        # :95-97
        L = sla.cholesky(B, lower=True)                                     # :98
        grad_log_p = y - pi
        b = W @ f + grad_log_p
        rhs = sqrtW @ (K @ b)
        inner = sla.solve_triangular(L, rhs, lower=True)
        # :101  `b - sqrtW * L.t \ (L \ ...)`: Scala ranks an operator by its first character and `\`
        # ("other special characters") outranks `*`, so this is b - sqrtW * (L.t \ (L \ rhs)).
        a = b - sqrtW @ sla.solve_triangular(L.T, inner, lower=False)
        new_f = (1.0 - step) * f + step * (K @ a)                            # :102
        new_obj_cand = -float(a @ new_f) / 2.0 + float(np.sum(np.log(_sigmoid((y * 2.0 - 1.0) * new_f))))
        if trace is not None:
            trace.append(dict(step=step, cand=new_obj_cand, old_obj=old_obj, new_obj=new_obj,
                              accepted=bool(new_obj_cand > old_obj)))
            iterations += 1
        if new_obj_cand > old_obj:                                          # :104-107
            f[:] = new_f
            old_obj = new_obj
            new_obj = new_obj_cand
        else:
            step /= 2.0
        if trace is not None:
            trace[-1]["max_abs_f"] = float(np.abs(f).max()) if n else 0.0
    if trace is not None:
        trace.append({"exit": "none" if iterations == 0 else "converged" if not abs(old_obj - new_obj) > tol else "step"})
    logZ = new_obj - float(np.sum(np.log(np.diag(L))))                      # :114
    # :116  R = sqrtW * L.t \ (L \ sqrtW)  -> sqrtW * (L.t \ (L \ sqrtW))  (same precedence argument)
    R = sqrtW @ sla.solve_triangular(L.T, sla.solve_triangular(L, sqrtW, lower=True), lower=False)
    C = sla.solve_triangular(L, sqrtW @ K, lower=True)                      # :117
    d3 = -(2.0 * pi - 1.0) * pi * pi * np.exp(-f)                           # :118 (sign as in the reference)
    s2 = -0.5 * (np.diag(K) - np.diag(C.T @ C)) * d3                        # :119
    grad = []
    for dK in derivatives:                                                  # :121-126
        s1 = 0.5 * float(a @ dK @ a) - 0.5 * float(np.sum(R * dK))
        bb = dK @ grad_log_p
        s3 = bb - K @ (R @ bb)
        grad.append(s1 + float(s2 @ s3))
    return -logZ, -np.array(grad)


def classification_model_outputs(f: np.ndarray):
    """GaussianProcessClassificationModel (GPCls:136-162) for latent predictions f (one per row):
    rawPrediction = (-f, f) (:152-155); probability = raw2probabilityInPlace (:140-148): values(0) = sigmoid(-values(0)) =
    sigmoid(f), values(1) = 1 - values(0) -- the reference's quirk; prediction = Spark's raw2prediction with no thresholds
    set = rawPrediction.argmax (first maximum on ties), i.e. 1.0 iff f > 0."""
    f = np.atleast_1d(np.asarray(f, dtype=np.float64))
    raw = np.stack([-f, f], axis=-1)
    p0 = _sigmoid(-raw[:, 0])
    prob = np.stack([p0, 1.0 - p0], axis=-1)
    pred = np.argmax(raw, axis=-1).astype(np.float64)
    return raw, prob, pred
