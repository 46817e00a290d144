"""One-vs-rest host logic without a GPU: the lock-step optimisation driver, label validation, and the model's argmax."""
import numpy as np
import pytest

from oracle.one_vs_rest import one_vs_rest_binary_labels, one_vs_rest_model_outputs
from spark_gp_b200.classification import OneVsRest, one_vs_rest_labels, one_vs_rest_prediction
from spark_gp_b200.hyperopt import lbfgsb, lbfgsb_lockstep


def objectives(C):
    """Class c: a Rosenbrock-type function with its own scale and minimum, so that the classes stop at different rounds."""
    def make(c):
        a, b = 1.0 + 0.3 * c, 5.0 + 40.0 * c

        def f(x):
            x = np.asarray(x, dtype=np.float64)
            r = b * (x[1] - x[0] ** 2) ** 2 + (a - x[0]) ** 2 + 0.1 * c * x[2] ** 2
            g = np.array([-4 * b * x[0] * (x[1] - x[0] ** 2) - 2 * (a - x[0]), 2 * b * (x[1] - x[0] ** 2), 0.2 * c * x[2]])
            return float(r), g
        return f
    return [make(c) for c in range(C)]


@pytest.mark.parametrize("C,max_iter", [(1, 50), (3, 100), (6, 15), (10, 200)])
def test_lockstep_trajectories_equal_independent_runs(C, max_iter):
    fs = objectives(C)
    x0 = np.array([-1.2, 1.0, 0.5])
    bounds = [(-2.0, 2.0), (None, 3.0), (0.1, None)]
    rounds_seen = []

    def evaluate(batch):
        cs = [c for c, _ in batch]
        assert cs == sorted(set(cs))                    # one point per class and round
        rounds_seen.append(cs)
        return [fs[c](t) for c, t in batch]

    results, rounds = lbfgsb_lockstep(evaluate, [x0] * C, bounds, max_iter, 1e-9)
    assert rounds == len(rounds_seen)
    evals = []
    for c in range(C):
        res0, ev0 = lbfgsb(fs[c], x0, bounds, max_iter, 1e-9)
        res, ev = results[c]
        assert np.array_equal(res.x, res0.x) and res.nit == res0.nit and ev == ev0 and res.fun == res0.fun, c
        evals.append(ev)
    assert rounds == max(evals)
    if C >= 3:
        assert len(set(evals)) > 1                      # classes stopped at different rounds
        assert len(rounds_seen[-1]) < C


def test_lockstep_propagates_an_evaluation_error():
    fs = objectives(3)

    def evaluate(batch):
        if len(batch) == 3 and any(np.asarray(t)[0] > -1.0 for _, t in batch):
            raise ArithmeticError("class failed")
        return [fs[c](t) for c, t in batch]

    with pytest.raises(ArithmeticError, match="class failed"):
        lbfgsb_lockstep(evaluate, [np.array([-1.2, 1.0, 0.5])] * 3, [(None, None)] * 3, 100, 1e-9)


def test_labels_and_num_classes():
    y, C = one_vs_rest_labels([0, 2, 1, 2, 0])
    assert C == 3 and y.dtype == np.float64
    assert one_vs_rest_labels([3.0, 3.0])[1] == 4              # numClasses = max(label) + 1, absent classes included
    for bad in ([0, 1.5], [0, -1], [0, np.nan], [0, np.inf], []):
        with pytest.raises(ValueError):
            one_vs_rest_labels(bad)
    assert np.array_equal(one_vs_rest_binary_labels([0, 2, 1], 3), [[1, 0, 0], [0, 0, 1], [0, 1, 0]])


def test_classifier_type_is_checked():
    with pytest.raises(TypeError):
        OneVsRest().setClassifier(object())
    with pytest.raises(TypeError):
        OneVsRest().fit(np.zeros((4, 1)), [0, 1, 0, 1])


def test_argmax_ties_go_to_the_first_class():
    raw = np.array([[1.0, 1.0, 0.0], [0.0, 2.0, 2.0], [-1.0, -1.0, -1.0], [0.5, -0.2, 0.7], [3.0, 1.0, 3.0]])
    want = np.array([0.0, 1.0, 0.0, 2.0, 0.0])
    assert np.array_equal(one_vs_rest_prediction(raw), want)
    raw_o, pred_o = one_vs_rest_model_outputs(raw.T)
    assert np.array_equal(raw_o, raw) and np.array_equal(pred_o, want)
    rng = np.random.default_rng(4)
    raw = rng.integers(-2, 3, size=(500, 5)).astype(np.float64)    # many ties
    assert np.array_equal(one_vs_rest_prediction(raw), one_vs_rest_model_outputs(raw.T)[1])

