"""The Laplace Newton loop where it branches, on the GPU against the oracle (run on an H100: `pytest -m gpu`).

Every case of the catalogue in test_host_laplace_newton.py (halvings, step exhaustion, loose tolerances, saturated and
overflowing modes) runs evaluation by evaluation, warm-starting from the device modes as the optimiser does:
sgp_laplace_nll and sgp_laplace_nll_any_size on chip (n <= 117: the same launch, so the same bits), and
sgp_laplace_nll_any_size on the global-memory kernel above.  After every evaluation the value, every gradient component
and the modes are compared with the oracle; the modes pin the control flow, since another branch moves f by O(step).
Gates: test_host_laplace_newton.gates -- TOL_NLL, RTOL_LAP / ATOL_LAP per component and modes 1e-9 max(1, |f|), widened
to 16x the oracle's own spread under a 1-ulp perturbation of K where B is ill-conditioned (at most 1e-6 relative).  A
NaN gradient component must be NaN in exactly the components where the oracle's is.

Also: the classes form in the hard regime against binary uploads of (y == c), bit for bit, on both kernels; and the
refusal of tol >= 1, where no Newton iteration runs and the reference's L \\ sqrtW throws MatrixSingularException.
"""
import numpy as np
import pytest

import spark_gp_b200 as sg
from oracle.classification import classification_likelihood_and_gradient
from test_host_laplace_newton import CASES, ON_CHIP_MAX, case_data, case_id, err_over_gate, gates, oracle_sequence, quiet

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def engs():
    a, b = sg.ProjectedProcessEngine(0), sg.ProjectedProcessEngine(0)
    yield a, b
    a.close()
    b.close()


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.int64)


def upload_one_expert(eng, X, y):
    eng.experts_upload(X, y, np.array([0, len(X)], dtype=np.int64))


@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_case_against_the_oracle_evaluation_by_evaluation(engs, case):
    eng, ref = engs
    X, y, k, _ = case_data(case)
    n = len(y)
    on_chip = n <= ON_CHIP_MAX
    evals = oracle_sequence(case)
    gate = gates(case, evals)
    upload_one_expert(eng, X, y)
    if on_chip:
        upload_one_expert(ref, X, y)
    worst = []
    for i, (ev, gt) in enumerate(zip(evals, gate)):
        kt = k.setHyperparameters(ev["theta"])
        v, g = eng.laplace_nll_any_size(kt, ev["tol"])
        assert eng.last_laplace_path() == (0 if on_chip else 1)
        f = eng.experts_f(n)
        if on_chip:                                           # the on-chip form: the same launch, the same bits
            v2, g2 = ref.laplace_nll(kt, ev["tol"])
            assert bits(v2) == bits(v) and np.array_equal(bits(g2), bits(g)), (case[0], i)
            assert np.array_equal(bits(ref.experts_f(n)), bits(f)), (case[0], i)
        r = err_over_gate(v, np.asarray(g), f, ev, gt)
        worst.append(r)
        assert r <= 1.0, "%s eval %d: err/gate %.3e (value %r vs %r, NaN %s vs %s, |df| %.3e)" % (
            case[0], i, r, v, ev["value"], np.isnan(g).tolist(), np.isnan(ev["grad"]).tolist(),
            float(np.abs(f - ev["f"]).max()))
    print("newton %-14s n=%3d %-9s err/gate per evaluation: %s" % (
        case[0], n, "on chip" if on_chip else "global", " ".join("%.2e" % w for w in worst)))


# ---- the classes form in the hard regime -------------------------------------------------------------------------------
def classes_case(on_chip):
    """The first catalogue case of the size class with a halving or a NaN gradient."""
    return next(c for c in CASES if (c[2] <= ON_CHIP_MAX) == on_chip and {"halving", "nan"} & set(c[8]))


@pytest.mark.parametrize("on_chip", [True, False], ids=["on_chip", "global"])
def test_classes_match_binary_uploads_bitwise_in_the_hard_regime(engs, on_chip):
    """Three classes: class 1 is the case's positives, classes 0 and 2 split its negatives, each class at its own θ
    sequence (the case's, scaled per class); every class's value, gradient and modes equal the binary upload of
    (y == c) bit for bit after every evaluation."""
    eng, ref = engs
    case = classes_case(on_chip)
    X, y, _, _ = case_data(case)
    n = len(y)
    y3 = np.where(y == 1.0, 1.0, np.where(np.arange(n) % 2 == 0, 0.0, 2.0))
    entry = eng.laplace_nll_classes if on_chip else eng.laplace_nll_classes_any_size
    upload_one_expert(eng, X, y3)
    theta_of = lambda c, i: np.asarray(case[6][i]) * np.r_[1.0 + 0.1 * (c - 1), np.ones(len(case[6][i]) - 1)]
    kernel_at = lambda c, i: case_data(case)[2].setHyperparameters(theta_of(c, i))
    got = {c: [] for c in range(3)}
    for i, tol in enumerate(case[7]):
        vals, grads = entry(3, [2, 0, 1], [kernel_at(c, i) for c in (2, 0, 1)], tol)
        assert eng.last_laplace_path() == (0 if on_chip else 1)
        for j, c in enumerate((2, 0, 1)):
            got[c].append((vals[j], grads[j], eng.experts_f_class(c, n)))
    saw_hard = False
    for c in range(3):
        upload_one_expert(ref, X, (y3 == c).astype(np.float64))
        for i, tol in enumerate(case[7]):
            v0, g0 = ref.laplace_nll_any_size(kernel_at(c, i), tol)
            v, g, f = got[c][i]
            assert bits(v) == bits(v0) and np.array_equal(bits(g), bits(g0)), (case[0], c, i)
            assert np.array_equal(bits(f), bits(ref.experts_f(n))), (case[0], c, i)
            saw_hard |= c == 1 and (np.isnan(g0).any() or np.abs(f).max() > 37.0)
    print("classes %s on %s: bit-identical to binary uploads, class 1 saturated or NaN: %s" % (
        case[0], "chip" if on_chip else "global", saw_hard))


# ---- tol >= 1: no Newton iteration runs --------------------------------------------------------------------------------
@pytest.mark.parametrize("on_chip", [True, False], ids=["on_chip", "global"])
def test_tolerance_that_runs_no_iteration_is_refused(engs, on_chip):
    eng, _ = engs
    n = 60 if on_chip else 150
    case = ("refusal", 11, n, 2, 0.3, "ard", [], [], ())
    X, y, k, ke = case_data(case)
    theta = np.array([2.0, 0.8, 1.1])
    kt = k.setHyperparameters(theta)
    upload_one_expert(eng, X, y)
    f0 = np.zeros(n)
    v0, g0 = quiet(classification_likelihood_and_gradient, y, f0, ke, theta, 1e-6)
    eng.laplace_nll_any_size(kt, 1e-6)                        # non-zero modes, to see that a refusal leaves them
    eng.laplace_nll_classes_any_size(2, [1], [kt], 1e-6)      # the classes modes exist
    f_bin, f_cls = eng.experts_f(n), eng.experts_f_class(1, n)
    entries = [lambda t: eng.laplace_nll_any_size(kt, t),
               lambda t: eng.laplace_nll_classes_any_size(2, [1], [kt], t)]
    if on_chip:
        entries += [lambda t: eng.laplace_nll(kt, t), lambda t: eng.laplace_nll_classes(2, [1], [kt], t)]
    for call in entries:
        for tol in (1.0, 1.5, np.inf):
            launches = eng.launch_count()
            with pytest.raises(sg.MatrixSingularException, match="no Newton iteration runs"):
                call(tol)
            assert eng.launch_count() == launches
            assert np.array_equal(bits(eng.experts_f(n)), bits(f_bin))
            assert np.array_equal(bits(eng.experts_f_class(1, n)), bits(f_cls))
    # 0.999 runs one iteration from the warm modes, as the oracle does
    f_ref = f0.copy()
    tr = []
    v1, g1 = quiet(classification_likelihood_and_gradient, y, f_ref, ke, theta, 0.999, trace=tr)
    assert tr[-1]["exit"] != "none"
    v, g = eng.laplace_nll_any_size(kt, 0.999)
    assert abs(v - v1) <= 1e-9 * abs(v1)
    assert np.abs(g - g1).max() <= 1e-9 * np.abs(g1).max()
    assert np.abs(eng.experts_f(n) - f_ref).max() <= 1e-9 * max(1.0, np.abs(f_ref).max())


def test_classifier_with_tol_one_raises_matrix_singular():
    rng = np.random.default_rng(4)
    X = rng.standard_normal((120, 2))
    y = (X[:, 0] > 0).astype(np.float64)
    gp = sg.GaussianProcessClassifier().setDatasetSizeForExpert(40).setActiveSetSize(20).setTol(1.0)
    with pytest.raises(sg.MatrixSingularException):
        gp.fit(X, y)
    with pytest.raises(sg.MatrixSingularException):
        gp.fit(X, y, hyperparameters=gp.getKernel().getHyperparameters())
