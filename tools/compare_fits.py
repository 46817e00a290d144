"""Every output of the estimators and model selectors that share the hyper-parameter optimisation, on seeded inputs, in
one .npz: so that two versions of the package can be compared bit for bit.

  python tools/compare_fits.py --package DIR --out A.npz      (DIR holds the spark_gp_b200 package; default: this tree)
  python tools/compare_fits.py --compare A.npz B.npz           (exit code 1 unless every entry is equal bit for bit)

Dumped: hyper-parameters, `last_latent`, every model's magic vector and matrix, raw predictions and predictions on held-out
rows, `last_stats`, `last_objective` (values, evaluations, iterations, rounds, calls, launches), `last_folds`,
`last_predictions`, metrics and `bestIndex`, of:
  binary_chip      GaussianProcessClassifier.fit, 800 x 3, datasetSizeForExpert 100 (on-chip Laplace kernel)
  binary_global    the same with datasetSizeForExpert 200 (global-memory Laplace kernel)
  binary_fixed     the same at given hyper-parameters, and at maxIter 0 (no optimisation)
  ovr_iris         OneVsRest.fit on tests/golden/iris_case.npz's training rows (classification/examples/Iris.scala)
  ovr_fixed        the same at given hyper-parameters
  tvs_binary       TrainValidationSplit over the binary classifier, 3 kernels
  tvs_binary_one_slot_maxIter30 / _maxIter0   the same with one map (one slot), optimised and not
  tvs_ovr          TrainValidationSplit over one-vs-rest on all of Iris, 2 sigma2 values
  tvs_regression   TrainValidationSplit over GaussianProcessRegression, 2 sigma2 values
  cv               a 3-fold CrossValidator over GaussianProcessRegression, 2 sigma2 values
  regression       GaussianProcessRegression.fit"""
from __future__ import annotations

import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def flatten(prefix, value, out):
    if isinstance(value, dict):
        for k, v in value.items():
            flatten("%s.%s" % (prefix, k), v, out)
    elif isinstance(value, (list, tuple)):
        out[prefix + ".len"] = np.array(len(value))
        for i, v in enumerate(value):
            flatten("%s.%d" % (prefix, i), v, out)
    elif value is None:
        out[prefix] = np.array("None")
    else:
        out[prefix] = np.asarray(value)


def model_outputs(model, Xte):
    """A binary classification or regression model: hyper-parameters, magic pair and predictions."""
    rp = model.rawPredictor
    out = dict(theta=model.hyperparameters, magicVector=rp.magicVector, magicMatrix=rp.magicMatrix,
               activeSet=rp.activeSet, prediction=model.predict(Xte))
    if hasattr(model, "predictRaw"):
        out["raw"] = model.predictRaw(Xte)
    return out


def ovr_outputs(model, Xte):
    return dict(thetas=model.hyperparameters, raw=model.predictRaw(Xte), prediction=model.predict(Xte),
                models=[model_outputs(m, Xte) for m in model.models])


def binary_data(n=800, d=3, seed=1):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n + 200, d))
    y = (np.sin(2 * X[:, 0]) + 0.5 * X[:, 1] + 0.3 * rng.standard_normal(n + 200) > 0).astype(np.float64)
    return X[:n], y[:n], X[n:], y[n:]


def run(sg):
    res = {}
    X, y, Xte, _ = binary_data()
    binary = lambda n_e: (sg.GaussianProcessClassifier().setDatasetSizeForExpert(n_e).setActiveSetSize(50)
                          .setKernel(lambda: sg.RBFKernel(1.0)).setMaxIter(30).setSeed(3))
    for name, n_e in (("binary_chip", 100), ("binary_global", 200)):
        gp = binary(n_e)
        model = gp.fit(X, y)
        res[name] = dict(model=model_outputs(model, Xte), last_objective=gp.last_objective, last_latent=gp.last_latent,
                         last_stats=gp.last_stats)
        del model
    gp = binary(100)
    fixed = gp.fit(X, y, hyperparameters=0.7 * gp.getKernel().getHyperparameters())
    unopt = binary(100).setMaxIter(0)
    zero = unopt.fit(X, y)
    res["binary_fixed"] = dict(fixed=model_outputs(fixed, Xte), fixed_latent=gp.last_latent,
                               fixed_objective=gp.last_objective, zero=model_outputs(zero, Xte),
                               zero_latent=unopt.last_latent, zero_objective=unopt.last_objective)
    del fixed, zero

    c = np.load(os.path.join(ROOT, "tests", "golden", "iris_case.npz"))
    Xi, yi = c["X"], c["y"]
    tr, te = c["train_idx"], c["test_idx"]
    iris_gp = lambda: sg.GaussianProcessClassifier().setDatasetSizeForExpert(20).setActiveSetSize(30)
    ovr = sg.OneVsRest().setClassifier(iris_gp())
    model = ovr.fit(Xi[tr], yi[tr])
    res["ovr_iris"] = dict(model=ovr_outputs(model, Xi[te]), last_objective=ovr.last_objective,
                           last_latent=ovr.last_latent)
    thetas = model.hyperparameters * 1.1
    del model
    ovr = sg.OneVsRest().setClassifier(iris_gp())
    model = ovr.fit(Xi[tr], yi[tr], hyperparameters=thetas)
    res["ovr_fixed"] = dict(model=ovr_outputs(model, Xi[te]), last_objective=ovr.last_objective,
                            last_latent=ovr.last_latent)
    del model

    def selection(tvs, model, Xte):
        best = model.bestModel
        return dict(metrics=model.validationMetrics, bestIndex=model.bestIndex, last_objective=model.last_objective,
                    last_predictions=tvs.last_predictions,
                    best=ovr_outputs(best, Xte) if hasattr(best, "models") else model_outputs(best, Xte))

    maps = sg.ParamGridBuilder().addGrid("kernel", [(lambda s: lambda: sg.RBFKernel(s))(s) for s in (0.5, 1.0, 2.0)]).build()
    tvs = (sg.TrainValidationSplit().setEstimator(binary(100)).setEvaluator(sg.MulticlassClassificationEvaluator("accuracy"))
           .setEstimatorParamMaps(maps).setSeed(5))
    res["tvs_binary"] = selection(tvs, tvs.fit(X, y), Xte)
    for maps in ([{}], [{"maxIter": 0}]):
        tvs = (sg.TrainValidationSplit().setEstimator(binary(100))
               .setEvaluator(sg.MulticlassClassificationEvaluator("accuracy")).setEstimatorParamMaps(maps).setSeed(5))
        res["tvs_binary_one_slot_maxIter%d" % maps[0].get("maxIter", 30)] = selection(tvs, tvs.fit(X, y), Xte)
    maps = sg.ParamGridBuilder().addGrid("sigma2", [1e-3, 1e-1]).build()
    tvs = (sg.TrainValidationSplit().setEstimator(sg.OneVsRest().setClassifier(iris_gp()))
           .setEvaluator(sg.MulticlassClassificationEvaluator()).setEstimatorParamMaps(maps).setSeed(2))
    res["tvs_ovr"] = selection(tvs, tvs.fit(Xi, yi), Xi[te])

    rng = np.random.default_rng(13)
    Xr = np.linspace(0, 1, 1500)[:, None]
    yr = np.sin(3 * Xr[:, 0]) + 0.1 * rng.standard_normal(1500)
    Xrt = rng.random((100, 1))
    reg = lambda: (sg.GaussianProcessRegression().setKernel(lambda: 1 * sg.RBFKernel(0.1, 1e-6, 10))
                   .setDatasetSizeForExpert(100).setActiveSetSize(60).setSeed(13).setMaxIter(20))
    tvs = (sg.TrainValidationSplit().setEstimator(reg()).setEvaluator(sg.RegressionEvaluator())
           .setEstimatorParamMaps(maps).setSeed(4))
    res["tvs_regression"] = selection(tvs, tvs.fit(Xr, yr), Xrt)
    cv = sg.CrossValidator().setEstimator(reg()).setEstimatorParamMaps(maps).setNumFolds(3).setSeed(6)
    model = cv.fit(Xr, yr)
    res["cv"] = dict(avgMetrics=model.avgMetrics, bestIndex=model.bestIndex, last_objective=model.last_objective,
                     last_folds={"%d_%d" % pk: v for pk, v in cv.last_folds.items()},
                     best=model_outputs(model.bestModel, Xrt))
    del model
    gp = reg()
    model = gp.fit(Xr, yr)
    res["regression"] = dict(model=model_outputs(model, Xrt), last_objective=gp.last_objective, last_stats=gp.last_stats)
    return res


def compare(a_path, b_path):
    a, b = np.load(a_path), np.load(b_path)
    bad = sorted(set(a.files) ^ set(b.files))
    for k in sorted(set(a.files) & set(b.files)):
        x, y = a[k], b[k]
        if x.dtype != y.dtype or x.shape != y.shape or x.tobytes() != y.tobytes():
            bad.append(k)
    print("%d entries compared, %d differ%s" % (len(set(a.files) | set(b.files)), len(bad),
                                                ": " + ", ".join(bad[:20]) if bad else ""))
    return not bad


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--package", default=ROOT, help="directory that holds the spark_gp_b200 package")
    ap.add_argument("--out")
    ap.add_argument("--compare", nargs=2)
    a = ap.parse_args()
    if a.compare:
        sys.exit(0 if compare(*a.compare) else 1)
    sys.path.insert(0, ROOT)                        # the oracle and test fixtures
    sys.path.insert(0, os.path.abspath(a.package))
    import spark_gp_b200 as sg
    print("package:", os.path.dirname(sg.__file__))
    out = {}
    flatten("fits", run(sg), out)
    np.savez(a.out, **out)
    print("wrote %d entries to %s" % (len(out), a.out))


if __name__ == "__main__":
    main()
