"""One-vs-rest classification on the GPU (run on an H100: `pytest -m gpu`).

`sgp_laplace_nll_classes` evaluates the binary Laplace objective of several classes in one launch.  Class c's value,
gradient and latent modes must equal, bit for bit, what `sgp_laplace_nll` returns on an upload of the labels (y == c)
after the same sequence of evaluations, whichever other classes are in the call.  `OneVsRest.fit` must then give every
class exactly the binary `GaussianProcessClassifier.fit(X, y == c)` result.

Tolerances against the fp64 oracle (written here once): as test_gpu_parity.test_laplace_nll_gradient_and_modes_vs_oracle,
1e-9 on the value (relative), 1e-7 on the gradient (relative to its largest component), 1e-9 on the modes; raw
predictions of the Iris fixture 1e-5 (TOL_PRED); magic vectors 1e-3 relative (TOL_MAGIC: the default statistics mode
rounds kernel elements to fp32, and the magic vector is a cond(A)-amplified image of that rounding).
"""
import os

import numpy as np
import pytest

import oracle
import spark_gp_b200 as sg
from oracle.classification import classification_likelihood_and_gradient
from oracle.one_vs_rest import one_vs_rest_model_outputs
from spark_gp_b200.hyperopt import group_for_experts, pack_experts
from spark_gp_b200.regression import ExplicitActiveSetProvider

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TOL_PRED, TOL_MAGIC = 1e-5, 1e-3


@pytest.fixture(scope="module")
def engs():
    a, b = sg.ProjectedProcessEngine(0), sg.ProjectedProcessEngine(0)
    yield a, b
    a.close()
    b.close()


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.int64)


KERNELS = {
    "ard": (lambda d: 1.2 * sg.ARDRBFKernel(np.linspace(0.6, 1.1, d)) + sg.const(1e-2) * sg.EyeKernel(),
            lambda d: 1.2 * oracle.ARDRBFKernel(np.linspace(0.6, 1.1, d)) + oracle.const(1e-2) * oracle.EyeKernel()),
    "rbf": (lambda d: sg.RBFKernel(1.3) + sg.const(1e-2) * sg.EyeKernel(),
            lambda d: oracle.RBFKernel(1.3) + oracle.const(1e-2) * oracle.EyeKernel()),
    "two_term": (lambda d: 1.5 * sg.ARDRBFKernel(np.full(d, 0.7)) + 0.5 * sg.RBFKernel(2.0) + sg.const(1e-2) * sg.EyeKernel(),
                 lambda d: 1.5 * oracle.ARDRBFKernel(np.full(d, 0.7)) + 0.5 * oracle.RBFKernel(2.0)
                 + oracle.const(1e-2) * oracle.EyeKernel()),
}


def class_data(N, d, C, seed, missing=None):
    """N points in d dimensions with class indices 0..C-1 from a noisy projection; class `missing` gets no point."""
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((N, d))
    s = np.sin(2 * X[:, 0]) + X[:, -1] + 0.3 * rng.standard_normal(N)
    y = np.digitize(s, np.quantile(s, np.linspace(0, 1, C + 1)[1:-1])).astype(np.float64)
    if missing is not None:
        y[y == missing] = (missing + 1) % C
    return X, y


def theta_of(mk, d, c, step):
    t0 = mk(d).getHyperparameters()
    return t0 * (1.0 + 0.07 * c) * (1.0 + 0.15 * step)


# ---------------- 1. the class-batched entry against single-class uploads, bit for bit --------------------------------
CASES = [  # (kernel, C, n_max, ragged, E, d, missing class)
    ("ard", 2, 40, True, 5, 3, None),
    ("rbf", 3, 117, False, 3, 2, None),
    ("two_term", 10, 30, True, 7, 4, 7),
    ("ard", 3, 117, True, 3, 5, None),
]


@pytest.mark.parametrize("kind,C,n_max,ragged,E,d,missing", CASES)
def test_classes_match_binary_uploads_bitwise(engs, kind, C, n_max, ragged, E, d, missing):
    eng, ref = engs
    n_e = n_max - 1 if ragged else n_max
    N = E * n_e + (E // 2 if ragged else 0)
    assert int(np.floor(N / n_e + 0.5)) == E
    X, y = class_data(N, d, C, seed=C * 100 + n_max, missing=missing)
    if missing is not None:
        assert not np.any(y == missing)
    mk = KERNELS[kind][0]
    tol = 1e-6
    eng.experts_upload(*pack_experts(X, y, n_e))
    # calls: every class in order, every class reversed (warm start), a subset in a permuted order
    calls = [list(range(C)), list(range(C))[::-1], [C - 1, 0] if C > 2 else [1]]
    steps = np.zeros(C, dtype=int)
    got = {c: [] for c in range(C)}
    modes_before = None
    for call in calls:
        thetas = [theta_of(mk, d, c, steps[c]) for c in call]
        if call is calls[-1]:
            modes_before = {c: eng.experts_f_class(c, N) for c in range(C)}
        vals, grads = eng.laplace_nll_classes(C, call, [mk(d).setHyperparameters(t) for t in thetas], tol)
        for i, c in enumerate(call):
            got[c].append((vals[i], grads[i], eng.experts_f_class(c, N)))
            steps[c] += 1
    for c in range(C):                            # classes the last call did not list keep their modes
        if c not in calls[-1]:
            assert np.array_equal(bits(eng.experts_f_class(c, N)), bits(modes_before[c]))
    for c in range(C):
        ref.experts_upload(*pack_experts(X, (y == c).astype(np.float64), n_e))
        for step, (v, g, f) in enumerate(got[c]):
            v0, g0 = ref.laplace_nll(mk(d).setHyperparameters(theta_of(mk, d, c, step)), tol)
            f0 = ref.experts_f(N)
            assert bits(v) == bits(v0), (c, step, v, v0)
            assert np.array_equal(bits(g), bits(g0)), (c, step)
            assert np.array_equal(bits(f), bits(f0)), (c, step)


def test_classes_refusals(engs):
    eng, _ = engs
    mk = KERNELS["rbf"][0]
    X, y = class_data(3 * 118, 2, 3, seed=5)
    eng.experts_upload(*pack_experts(X, y, 118))
    with pytest.raises(ValueError, match="too large"):
        eng.laplace_nll_classes(3, [0], [mk(2)], 1e-6)
    X, y = class_data(300, 2, 3, seed=6)
    eng.experts_upload(*pack_experts(X, y, 100))
    with pytest.raises(sg.TrainingVectorsNotInitializedException):
        eng.experts_f_class(0, 300)                       # no class modes since the upload
    for n_classes, classes in ((3, [3]), (3, [-1]), (3, [0, 0]), (2, [0, 1, 2]), (0, [0])):
        with pytest.raises(ValueError):
            eng.laplace_nll_classes(n_classes, classes, [mk(2)] * len(classes), 1e-6)
    eng.laplace_nll_classes(3, [1], [mk(2)], 1e-6)
    with pytest.raises(ValueError):
        eng.experts_f_class(3, 300)
    assert np.all(eng.experts_f_class(0, 300) == 0.0)     # unlisted classes start at zero
    with pytest.raises(ValueError):                         # kernels of different structure
        eng.laplace_nll_classes(3, [0, 1], [mk(2), KERNELS["ard"][0](2)], 1e-6)


# ---------------- 2. each class against the oracle at fixed theta ------------------------------------------------------
def test_classes_vs_oracle(engs):
    eng, _ = engs
    n, d, n_e, C, tol = 730, 3, 100, 3, 1e-6
    X, y = class_data(n, d, C, seed=31)
    mk, mo = KERNELS["ard"]
    groups = group_for_experts(n, n_e)
    eng.experts_upload(*pack_experts(X, y, n_e))
    fs = {c: [np.zeros(len(g)) for g in groups] for c in range(C)}
    experts = {c: oracle.get_expert_labels_and_kernels(X, (y == c).astype(np.float64), lambda: mo(d), n_e)
               for c in range(C)}
    for step in range(2):
        thetas = [theta_of(mk, d, c, step) for c in range(C)]
        vals, grads = eng.laplace_nll_classes(C, range(C), [mk(d).setHyperparameters(t) for t in thetas], tol)
        for c in range(C):
            v0, g0 = 0.0, 0.0
            for (ye, ke), f in zip(experts[c], fs[c]):
                v, g = classification_likelihood_and_gradient(ye, f, ke, thetas[c], tol)
                v0 += v
                g0 = g0 + g
            assert abs(vals[c] - v0) / abs(v0) < 1e-9
            assert np.abs(grads[c] - g0).max() / np.abs(g0).max() < 1e-7
            f_ref = np.concatenate(fs[c])
            assert np.abs(eng.experts_f_class(c, n) - f_ref).max() < 1e-9 * max(1.0, np.abs(f_ref).max())


# ---------------- 3-5. the estimator on the Iris example -------------------------------------------------------------
def iris():
    c = np.load(os.path.join(GOLD, "iris_case.npz"))
    tr, te = c["train_idx"], c["test_idx"]
    return c, c["X"][tr], c["y"][tr], c["X"][te], c["y"][te]


def iris_gp():
    return sg.GaussianProcessClassifier().setDatasetSizeForExpert(20).setActiveSetSize(30)


@pytest.fixture(scope="module")
def iris_fit():
    c, Xtr, ytr, Xte, yte = iris()
    ovr = sg.OneVsRest().setClassifier(iris_gp())
    model = ovr.fit(Xtr, ytr)
    return ovr, model


def test_iris_fit_equals_binary_fits(iris_fit):
    c, Xtr, ytr, Xte, yte = iris()
    ovr, model = iris_fit
    assert model.numClasses == 3 and len(model.models) == 3
    raw = model.predictRaw(Xte)
    assert raw.shape == (len(Xte), 3)
    for k in range(3):
        gp = iris_gp()
        bm = gp.fit(Xtr, (ytr == k).astype(np.float64))
        m = model.models[k]
        assert np.array_equal(bits(m.hyperparameters), bits(bm.hyperparameters)), k
        assert np.array_equal(bits(ovr.last_latent[k]), bits(gp.last_latent)), k
        assert np.array_equal(bits(m.rawPredictor.magicVector), bits(bm.rawPredictor.magicVector)), k
        assert np.array_equal(bits(m.rawPredictor.magicMatrix), bits(bm.rawPredictor.magicMatrix)), k
        assert np.array_equal(bits(raw[:, k]), bits(bm.predictRaw(Xte)[:, 1])), k
        assert ovr.last_objective["classes"][k]["iterations"] == gp.last_objective["iterations"]
        assert ovr.last_objective["classes"][k]["evaluations"] == gp.last_objective["evaluations"]
    assert ovr.last_objective["rounds"] == max(cl["evaluations"] for cl in ovr.last_objective["classes"])
    assert np.mean(model.predict(Xte) == yte) > 0.8
    assert np.array_equal(model.transform(Xte), model.predict(Xte))


def test_iris_fixed_theta_vs_oracle():
    c, Xtr, ytr, Xte, yte = iris()
    gp = iris_gp().setActiveSetProvider(ExplicitActiveSetProvider(Xtr[c["active_idx"]]))
    ovr = sg.OneVsRest().setClassifier(gp)
    model = ovr.fit(Xtr, ytr, hyperparameters=c["thetas"])
    assert np.abs(ovr.last_latent - c["latent"]).max() < 1e-9 * max(1.0, np.abs(c["latent"]).max())
    for k in range(3):
        mv = model.models[k].rawPredictor.magicVector
        assert np.abs(mv - c["magic_vector"][k]).max() / np.abs(c["magic_vector"][k]).max() < TOL_MAGIC
    raw = model.predictRaw(Xte)
    assert np.abs(raw - c["raw"]).max() <= TOL_PRED * max(1.0, np.abs(c["raw"]).max())
    top2 = np.sort(c["raw"], axis=1)[:, -2:]
    clear = top2[:, 1] - top2[:, 0] > TOL_PRED
    assert np.array_equal(model.predict(Xte)[clear], c["prediction"][clear])
    raw_o, pred_o = one_vs_rest_model_outputs(raw.T)
    assert np.array_equal(model.predict(Xte), pred_o) and np.array_equal(raw_o, raw)


def test_iris_cuda_tensors_equal_host(iris_fit):
    import torch
    _, model = iris_fit
    c, Xtr, ytr, Xte, yte = iris()
    Xt = torch.from_numpy(Xte).cuda()
    raw_t = model.predictRaw(Xt)
    pred_t = model.predict(Xt)
    assert raw_t.is_cuda and pred_t.is_cuda and raw_t.dtype == torch.float64 and pred_t.dtype == torch.float64
    assert np.array_equal(bits(raw_t.cpu().numpy()), bits(model.predictRaw(Xte)))
    assert np.array_equal(pred_t.cpu().numpy(), model.predict(Xte))


def test_iris_model_contexts_never_ran_statistics(iris_fit):
    _, model = iris_fit
    for m in model.models:
        assert m.rawPredictor._engine.last_path() == -1
        assert m.rawPredictor._engine.last_tail_path() == -1


def test_argmax_ties_on_cuda_tensors():
    import torch
    from spark_gp_b200.classification import one_vs_rest_prediction
    raw = np.random.default_rng(4).integers(-2, 3, size=(500, 5)).astype(np.float64)     # many ties
    got = one_vs_rest_prediction(torch.from_numpy(raw).cuda())
    assert np.array_equal(got.cpu().numpy(), one_vs_rest_model_outputs(raw.T)[1])
