"""CPU checks of the averaged probability: the library's Gauss-Hermite rule (`sgp_gauss_hermite_rule`, host code that
needs no GPU) against numpy's `hermgauss`, and the oracle's restatement of commons/util/Integrator.scala against SciPy
quadrature."""
import ctypes as C

import numpy as np
import pytest
from scipy import integrate

from oracle import integrator as I


@pytest.fixture(scope="module")
def lib():
    from spark_gp_b200 import build, _native
    build.build_native()
    return _native.load()


def rule(lib, n):
    from spark_gp_b200 import _native as N
    x, w = np.empty(n), np.empty(n)
    assert lib.sgp_gauss_hermite_rule(n, N.ptr(x), N.ptr(w)) == N.SGP_OK
    return x, w


def test_rule_matches_hermgauss_for_every_size(lib):
    worst_x = worst_w = 0.0
    for n in range(1, 257):
        x, w = rule(lib, n)
        x0, w0 = np.polynomial.hermite.hermgauss(n)
        assert np.all(np.diff(x) > 0), n                               # ascending
        assert np.array_equal(x, -x[::-1]) and np.array_equal(w, w[::-1]), n
        assert np.all(w > 0) and np.all(np.isfinite(w)), n
        ex, ew = np.abs(x - x0).max(), (np.abs(w - w0) / w0).max()
        worst_x, worst_w = max(worst_x, ex), max(worst_w, ew)
        assert ex < 1e-13, (n, ex)
        assert ew < 1e-12, (n, ew)
        assert abs(w.sum() / np.sqrt(np.pi) - 1.0) < 1e-14, n
    print("nodes %.1e, weights %.1e relative" % (worst_x, worst_w))


def test_rule_edges(lib):
    x, w = rule(lib, 1)
    assert x[0] == 0.0 and abs(w[0] - np.sqrt(np.pi)) < 1e-15
    x, w = rule(lib, 101)
    assert x[50] == 0.0 and not np.signbit(x[50])                       # the middle node of an odd rule is +0
    x, w = rule(lib, 256)
    assert 1e-212 < w.min() < 1e-209                                    # still a normal double


def test_rule_refusals(lib):
    from spark_gp_b200 import _native as N
    x, w = np.empty(300), np.empty(300)
    for n in (0, -1, 257):
        assert lib.sgp_gauss_hermite_rule(n, N.ptr(x), N.ptr(w)) == N.SGP_E_BADARG
    assert b"[1, 256]" in lib.sgp_last_error(None)
    assert lib.sgp_gauss_hermite_rule(5, None, N.ptr(w)) == N.SGP_E_BADARG
    assert lib.sgp_gauss_hermite_rule(5, N.ptr(x), None) == N.SGP_E_BADARG


def test_engine_rule_binding(lib):
    from spark_gp_b200.engine import ProjectedProcessEngine
    x, w = ProjectedProcessEngine.gauss_hermite_rule(100)
    x0, w0 = rule(lib, 100)
    assert np.array_equal(x, x0) and np.array_equal(w, w0)
    with pytest.raises(ValueError):
        ProjectedProcessEngine.gauss_hermite_rule(0)


def exact(mean, var):
    sd = np.sqrt(var)
    f = lambda t: I.sigmoid(t) * np.exp(-0.5 * ((t - mean) / sd) ** 2) / (sd * np.sqrt(2 * np.pi))
    return integrate.quad(f, mean - 40 * sd, mean + 40 * sd, epsabs=1e-14, epsrel=1e-14, limit=200)[0]


def test_oracle_matches_quadrature_at_integrator_test_case():
    """IntegratorTest.scala: E[sigmoid(f)], f ~ N(0.5, 3), 100 nodes."""
    ref = exact(0.5, 3.0)
    got = I.expected_of_function_of_normal(0.5, 3.0, I.sigmoid, 100)
    assert abs(got - ref) < 1e-13
    assert abs(I.averaged_probability(0.5, 3.0, 100) - got) < 1e-15
    # the rule's own error at a wide posterior is the reference's choice of n, not ours
    assert 1e-8 < abs(I.averaged_probability(5.0, 20.0, 100) - exact(5.0, 20.0)) < 1e-6


def test_oracle_clamp_and_nan():
    mu = np.array([-3.0, 0.0, 0.7, 2.0])
    sig = 1.0 / (1.0 + np.exp(-mu))
    wsum = np.polynomial.hermite.hermgauss(100)[1].sum() / np.sqrt(np.pi)
    for v in (0.0, 1e-300, -1e-12, -5.0):
        p = I.averaged_probability(mu, np.full(4, v), 100)
        assert np.all(np.abs(p - sig * wsum) < 1e-15), v
    assert np.isnan(I.expected_of_function_of_normal(0.5, -1.0, I.sigmoid, 100))    # the Integrator itself
    p = I.averaged_probability(np.array([np.nan, 0.0, 0.0]), np.array([1.0, np.nan, -np.nan]), 100)
    assert np.all(np.isnan(p))
    # far tails: no overflow warning leaks out, the probabilities saturate
    p = I.averaged_probability(np.array([-800.0, 800.0]), np.array([1.0, 1.0]), 100)
    assert p[0] == 0.0 and abs(p[1] - 1.0) < 1e-14


def test_oracle_symmetry():
    rng = np.random.default_rng(0)
    mu, v = rng.standard_normal(50) * 3, rng.random(50) * 10
    assert np.abs(I.averaged_probability(mu, v) + I.averaged_probability(-mu, v) - 1.0).max() < 1e-14
