"""commons/util/Integrator.scala restated, and the averaged predictive probability built on it.

`Integrator(n).expectedOfFunctionOfNormal(mean, variance, f)` (Integrator.scala:10-15) integrates
x -> f(sqrt(2) * sd * x + mean) with commons-math's n-point Gauss-Hermite rule (`GaussIntegratorFactory.hermite(n)`,
the weight exp(-x^2)) and divides by sqrt(pi): E[f(X)] for X ~ N(mean, variance).  The rule here is numpy's `hermgauss`.
Its only test (IntegratorTest.scala) takes f = sigmoid, (mean, variance) = (0.5, 3) and n = 100: the probability of
class 1 averaged over a latent posterior, GPML eq. 3.25."""
from __future__ import annotations

import numpy as np


def expected_of_function_of_normal(mean: float, variance: float, f, n: int) -> float:
    """Integrator.scala:10-15 for one (mean, variance): a negative variance gives NaN, as sqrt does there."""
    x, w = np.polynomial.hermite.hermgauss(n)
    with np.errstate(invalid="ignore"):
        sd = np.sqrt(variance)
    return float(np.sum(w * f(np.sqrt(2.0) * sd * x + mean)) / np.sqrt(np.pi))


def sigmoid(z):
    """breeze.numerics.sigmoid: 1 / (1 + exp(-z))."""
    with np.errstate(over="ignore"):
        return 1.0 / (1.0 + np.exp(-np.asarray(z, dtype=np.float64)))


def averaged_probability(mean, var, n: int = 100):
    """E[sigmoid(f)], f ~ N(mean, var), elementwise over arrays, with the n-node rule.  One deviation from the Integrator:
    var < 0 is taken as 0 (p = sigmoid(mean) up to the rule's weight sum); a NaN mean or variance still gives NaN."""
    mean = np.asarray(mean, dtype=np.float64)
    var = np.asarray(var, dtype=np.float64)
    x, w = np.polynomial.hermite.hermgauss(n)
    sd2 = np.sqrt(2.0 * np.where(var < 0.0, 0.0, var))          # np.where keeps NaN; np.maximum would too, fmax not
    z = mean[..., None] + sd2[..., None] * x
    return (sigmoid(z) @ w) / np.sqrt(np.pi)
