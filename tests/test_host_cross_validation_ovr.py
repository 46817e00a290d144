"""Host side of cross-validation over one-vs-rest (no GPU): the arguments, the (map, fold, class) slot numbering and
grouping, and the oracle's fold-wise one-vs-rest against the one-vs-rest restatement on that fold's rows."""
import numpy as np
import pytest

import oracle
import spark_gp_b200 as sg
from oracle import cross_validation as ocv
from oracle import cross_validation_ovr as ocv_ovr
from oracle.one_vs_rest import one_vs_rest_fixed_theta
from spark_gp_b200.tuning import fold_class_slot_groups, tvs_slot_groups


def test_cross_validator_accepts_one_vs_rest():
    cv = sg.CrossValidator()
    ovr = sg.OneVsRest().setClassifier(sg.GaussianProcessClassifier())
    assert cv.setEstimator(ovr) is cv and cv._estimator is ovr
    assert isinstance(cv._evaluator, sg.RegressionEvaluator)             # the default stays RegressionEvaluator()
    ev = sg.MulticlassClassificationEvaluator("accuracy")
    assert cv.setEvaluator(ev)._evaluator is ev
    cv.setEvaluator(sg.RegressionEvaluator("r2"))
    with pytest.raises(TypeError):
        cv.setEvaluator(object())
    with pytest.raises(TypeError):
        cv.setEstimator(sg.GaussianProcessClassifier())                  # the binary classifier is still refused
    with pytest.raises(TypeError):
        cv.setEstimator(sg.OneVsRest)
    cv = sg.CrossValidator().setEstimator(sg.OneVsRest()).setNumFolds(2)
    with pytest.raises(TypeError, match="setClassifier"):
        cv.fit(np.zeros((6, 1)), np.array([0, 1, 2, 0, 1, 2.0]))         # a OneVsRest without a classifier


def test_fold_class_slot_numbering_and_grouping():
    gp = sg.GaussianProcessClassifier().setKernel(lambda: sg.RBFKernel(1.0))
    gps = [gp.copy(m) for m in [{"sigma2": 1e-3}, {"kernel": lambda: sg.ARDRBFKernel(np.ones(2))}, {"sigma2": 1e-1},
                                {"datasetSizeForExpert": 50}]]
    C = [3, 2, 3]                                 # fold 1's training rows lack class 2
    groups = list(fold_class_slot_groups(gps, C).values())
    fc = [(k, c) for k in range(3) for c in range(C[k])]
    assert groups[0] == [(p, k, c, p * 8 + j) for p in (0, 2) for j, (k, c) in enumerate(fc)]
    assert [g[0][0] for g in groups[1:]] == [1, 3]
    modes = [m for g in groups for _, _, _, m in g]
    assert sorted(modes) == list(range(len(gps) * sum(C)))              # every (p, k, c) owns one mode slot
    # the train/validation split is the one-fold case, numbered p * C + c as before
    assert tvs_slot_groups(gps, 3) == {key: [(p, c, m) for p, _, c, m in slots]
                                       for key, slots in fold_class_slot_groups(gps, [3]).items()}
    assert list(tvs_slot_groups(gps, 3).values())[0] == [(p, c, p * 3 + c) for p in (0, 2) for c in range(3)]


def test_oracle_fold_one_vs_rest_equals_one_vs_rest_on_the_fold_rows():
    rng = np.random.default_rng(3)
    n, d = 90, 2
    X = rng.standard_normal((n, d))
    y = np.digitize(X[:, 0] + 0.3 * X[:, 1], [-0.5, 0.5]).astype(np.float64)
    fold_of = ocv.fold_assignment(n, 3, 5)
    fold_of[y == 2] = 1                           # fold 1's training rows lack class 2
    factory = oracle.get_kernel(lambda: oracle.RBFKernel(1.0), 1e-3)
    Z = X[::9]
    for k in range(3):
        tr, val = ocv.split(fold_of, k)
        C = int(y[tr].max()) + 1
        thetas = np.linspace(0.8, 1.4, C)[:, None]
        Ck, classes, raw, pred = ocv_ovr.fold_one_vs_rest_fixed_theta(X, y, fold_of, k, factory, thetas, Z, 20, 1e-6)
        assert Ck == C == (2 if k == 1 else 3)
        ref = one_vs_rest_fixed_theta(X[tr], y[tr], C, factory, thetas, Z, 20, 1e-6)
        for (f, mv), (f0, p0) in zip(classes, ref):
            assert np.array_equal(f, f0) and np.array_equal(mv, p0.magic_vector)
        raw0 = np.stack([p0.predict_many(X[val])[0] for _, p0 in ref], axis=-1)
        assert np.array_equal(raw, raw0)
        assert np.array_equal(pred, np.argmax(raw0, axis=1).astype(np.float64))
