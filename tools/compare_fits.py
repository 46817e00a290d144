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
  tvs_binary_auc   TrainValidationSplit over the binary classifier scored by BinaryClassificationEvaluator
  cv               a 3-fold CrossValidator over GaussianProcessRegression, 2 sigma2 values
  cv_ovr           a 3-fold CrossValidator over one-vs-rest on all of Iris, 2 sigma2 values
  regression       GaussianProcessRegression.fit
  regression_f32   the same on float32 X
  regression_kmeans / regression_explicit   the same with KMeansActiveSetProvider(on_gpu=True) / an explicit active set
Every case runs from host arrays (`host.*`) and from CUDA tensors on cuda:0 (`cuda.*`).  With --group, the data-parallel
fit of the regression, the binary classifier and one-vs-rest over a one-rank NCCL group on cuda:0 (the store on the
loopback address only), from host and CUDA input, is added as `group.*`, with the model selectors over that group:
`tvs_regression`, `cv`, `tvs_binary_auc` and `cv_ovr` as above."""
from __future__ import annotations

import argparse
import os
import socket
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
    elif type(value).__module__.partition(".")[0] == "torch":
        out[prefix] = value.detach().cpu().numpy()
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


def run(sg, put):
    """Every case, its inputs (features, labels, held-out features) through put."""
    res = {}
    X, y, Xte, _ = binary_data()
    X, y, Xte = put(X), put(y), put(Xte)
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
    tr, te = c["train_idx"], c["test_idx"]
    Xi, yi, Xi_tr, yi_tr, Xi_te = (put(a) for a in (c["X"], c["y"], c["X"][tr], c["y"][tr], c["X"][te]))
    iris_gp = lambda: sg.GaussianProcessClassifier().setDatasetSizeForExpert(20).setActiveSetSize(30)
    ovr = sg.OneVsRest().setClassifier(iris_gp())
    model = ovr.fit(Xi_tr, yi_tr)
    res["ovr_iris"] = dict(model=ovr_outputs(model, Xi_te), last_objective=ovr.last_objective,
                           last_latent=ovr.last_latent)
    thetas = model.hyperparameters * 1.1
    del model
    ovr = sg.OneVsRest().setClassifier(iris_gp())
    model = ovr.fit(Xi_tr, yi_tr, hyperparameters=thetas)
    res["ovr_fixed"] = dict(model=ovr_outputs(model, Xi_te), last_objective=ovr.last_objective,
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
    res["tvs_ovr"] = selection(tvs, tvs.fit(Xi, yi), Xi_te)
    tvs = (sg.TrainValidationSplit().setEstimator(binary(100)).setEvaluator(sg.BinaryClassificationEvaluator())
           .setEstimatorParamMaps(maps).setSeed(5))
    res["tvs_binary_auc"] = selection(tvs, tvs.fit(X, y), Xte)
    cv = (sg.CrossValidator().setEstimator(sg.OneVsRest().setClassifier(iris_gp()))
          .setEvaluator(sg.MulticlassClassificationEvaluator()).setEstimatorParamMaps(maps).setNumFolds(3).setSeed(6))
    model = cv.fit(Xi, yi)
    res["cv_ovr"] = dict(avgMetrics=model.avgMetrics, bestIndex=model.bestIndex, last_objective=model.last_objective,
                         last_folds={"%d_%d" % pk: v for pk, v in cv.last_folds.items()},
                         best=ovr_outputs(model.bestModel, Xi_te))
    del model

    rng = np.random.default_rng(13)
    Xr = np.linspace(0, 1, 1500)[:, None]
    yr = np.sin(3 * Xr[:, 0]) + 0.1 * rng.standard_normal(1500)
    Xrt = rng.random((100, 1))
    Xr32 = put(Xr.astype(np.float32))
    Xr, yr, Xrt = put(Xr), put(yr), put(Xrt)
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
    del model
    from spark_gp_b200.regression import ExplicitActiveSetProvider
    Z = np.linspace(0, 1, 40)[:, None]
    for name, data, provider in (("regression_f32", Xr32, None),
                                 ("regression_kmeans", Xr, sg.KMeansActiveSetProvider(on_gpu=True)),
                                 ("regression_explicit", Xr, ExplicitActiveSetProvider(Z))):
        gp = reg() if provider is None else reg().setActiveSetProvider(provider)
        model = gp.fit(data, yr)
        res[name] = dict(model=model_outputs(model, Xrt), last_objective=gp.last_objective, last_stats=gp.last_stats)
        del model
    return res


def run_group(sg, put):
    """The data-parallel fits over a one-rank NCCL group on cuda:0, inputs through put."""
    import torch.distributed as dist
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    import torch
    dist.init_process_group("nccl", init_method="tcp://127.0.0.1:%d" % port, rank=0, world_size=1,
                            device_id=torch.device("cuda", 0))
    try:
        group = dist.group.WORLD
        res = {}
        rng = np.random.default_rng(13)
        # a reshaped column: the row exchange views each row's bytes, which a broadcast column's stride-0 axis refuses
        Xr = np.linspace(0, 1, 1500).reshape(-1, 1)
        yr = np.sin(3 * Xr[:, 0]) + 0.1 * rng.standard_normal(1500)
        Xrt = put(rng.random((100, 1)))
        gp = (sg.GaussianProcessRegression(process_group=group).setKernel(lambda: 1 * sg.RBFKernel(0.1, 1e-6, 10))
              .setDatasetSizeForExpert(100).setActiveSetSize(60).setSeed(13).setMaxIter(20))
        model = gp.fit(put(Xr), put(yr))
        res["regression"] = dict(model=model_outputs(model, Xrt), last_objective=gp.last_objective,
                                 last_stats=gp.last_stats)
        del model
        X, y, Xte, _ = binary_data()
        gp = (sg.GaussianProcessClassifier(process_group=group).setDatasetSizeForExpert(100).setActiveSetSize(50)
              .setKernel(lambda: sg.RBFKernel(1.0)).setMaxIter(30).setSeed(3))
        model = gp.fit(put(X), put(y))
        res["binary"] = dict(model=model_outputs(model, put(Xte)), last_objective=gp.last_objective,
                             last_latent=gp.last_latent, last_stats=gp.last_stats)
        del model
        c = np.load(os.path.join(ROOT, "tests", "golden", "iris_case.npz"))
        tr, te = c["train_idx"], c["test_idx"]
        ovr = sg.OneVsRest().setClassifier(sg.GaussianProcessClassifier(process_group=group)
                                           .setDatasetSizeForExpert(20).setActiveSetSize(30))
        model = ovr.fit(put(c["X"][tr]), put(c["y"][tr]))
        res["ovr_iris"] = dict(model=ovr_outputs(model, put(c["X"][te])), last_objective=ovr.last_objective,
                               last_latent=ovr.last_latent)
        del model
        # the model selectors over the group, as `run` configures them
        maps = sg.ParamGridBuilder().addGrid("sigma2", [1e-3, 1e-1]).build()
        reg = (sg.GaussianProcessRegression(process_group=group).setKernel(lambda: 1 * sg.RBFKernel(0.1, 1e-6, 10))
               .setDatasetSizeForExpert(100).setActiveSetSize(60).setSeed(13).setMaxIter(20))
        tvs = (sg.TrainValidationSplit().setEstimator(reg).setEvaluator(sg.RegressionEvaluator())
               .setEstimatorParamMaps(maps).setSeed(4))
        res["tvs_regression"] = selection_outputs(tvs, tvs.fit(put(Xr), put(yr)), Xrt)
        cv = sg.CrossValidator().setEstimator(reg).setEstimatorParamMaps(maps).setNumFolds(3).setSeed(6)
        res["cv"] = selection_outputs(cv, cv.fit(put(Xr), put(yr)), Xrt)
        tvs = (sg.TrainValidationSplit().setEstimator(gp).setEvaluator(sg.BinaryClassificationEvaluator())
               .setEstimatorParamMaps(maps).setSeed(5))
        res["tvs_binary_auc"] = selection_outputs(tvs, tvs.fit(put(X), put(y)), put(Xte))
        cv = (sg.CrossValidator().setEstimator(ovr).setEvaluator(sg.MulticlassClassificationEvaluator())
              .setEstimatorParamMaps(maps).setNumFolds(3).setSeed(6))
        res["cv_ovr"] = selection_outputs(cv, cv.fit(put(c["X"]), put(c["y"])), put(c["X"][te]))
        return res
    finally:
        dist.destroy_process_group()


def selection_outputs(selector, model, Xte):
    """A model selector's metrics, bestIndex, records and best model."""
    best = model.bestModel
    out = dict(bestIndex=model.bestIndex, last_objective=model.last_objective,
               best=ovr_outputs(best, Xte) if hasattr(best, "models") else model_outputs(best, Xte))
    if hasattr(model, "avgMetrics"):
        out.update(avgMetrics=model.avgMetrics, last_folds={"%d_%d" % pk: v for pk, v in selector.last_folds.items()})
    else:
        out.update(metrics=model.validationMetrics, last_predictions=selector.last_predictions)
    return out


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
    ap.add_argument("--group", action="store_true", help="add the data-parallel fits over a one-rank NCCL group")
    a = ap.parse_args()
    if a.compare:
        sys.exit(0 if compare(*a.compare) else 1)
    sys.path.insert(0, ROOT)                        # the oracle and test fixtures
    sys.path.insert(0, os.path.abspath(a.package))
    import spark_gp_b200 as sg
    print("package:", os.path.dirname(sg.__file__))
    import torch
    host, cuda = (lambda a: a), (lambda a: torch.as_tensor(a, device="cuda:0"))
    out = {}
    flatten("host", run(sg, host), out)
    flatten("cuda", run(sg, cuda), out)
    if a.group:
        flatten("group.host", run_group(sg, host), out)
        flatten("group.cuda", run_group(sg, cuda), out)
    np.savez(a.out, **out)
    print("wrote %d entries to %s" % (len(out), a.out))


if __name__ == "__main__":
    main()
