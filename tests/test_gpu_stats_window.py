"""GPU tests of the begin..finish window of the statistics path (`sgp_stats_begin`): a begin that fails closes the window,
and one context serves begins of shrinking and growing shapes from its grow-only device buffers."""
import ctypes as C

import numpy as np
import pytest

import oracle
import spark_gp_b200 as sg
from spark_gp_b200 import _native as N
from test_gpu_parity import _oracle_stats_chunked, rel

pytestmark = pytest.mark.gpu

TOL_STATS, TOL_PRED = 1e-6, 1e-5


@pytest.fixture(scope="module")
def eng():
    e = sg.ProjectedProcessEngine(0)
    yield e
    e.close()


def ard(beta, noise=1e-2):
    """(library kernel, oracle kernel factory): 1 * ARD(beta) + noise * Eye."""
    return (1 * sg.ARDRBFKernel(beta) + sg.const(noise) * sg.EyeKernel(),
            lambda: 1 * oracle.ARDRBFKernel(beta) + oracle.const(noise) * oracle.EyeKernel())


def data(rng, n, m, d):
    X = rng.random((n, d))
    y = np.sin(3.0 * X.sum(1)) + 0.05 * rng.standard_normal(n)
    return X, y, X[rng.permutation(n)[:m]]


def oracle_posterior(ok, G0, b0, Z, Xt):
    kernel0 = ok().set_hyperparameters(ok().get_hyperparameters()).set_training_vectors(Z)
    mv0, mm0 = oracle.get_magic_vector(kernel0, G0, b0)
    return oracle.GaussianProjectedProcessRawPredictor(mv0, mm0, kernel0).predict_many(Xt)


def test_failed_begin_closes_window(eng):
    rng = np.random.default_rng(31)
    d = 6
    X, y, Z = data(rng, 4000, 150, d)
    k, ok = ard(np.full(d, np.sqrt(18.0 / d)))
    eng.set_precision(N.SGP_PREC_AUTO)
    eng.begin(k, Z)
    eng.accumulate(X, y)
    eng.finish()
    eng.magic()
    # an RBF term with sigma = 0, through the raw ABI: rejected while the kernel is flattened, before the new shape
    term = (N.KernelTerm * 1)()
    term[0].type, term[0].scale, term[0].sigma = N.SGP_TERM_RBF, 1.0, 0.0
    desc = N.KernelDesc(1, 0, term)
    Zbad = np.ascontiguousarray(Z[:40])
    with pytest.raises(ValueError):
        eng._check(eng._lib.sgp_stats_begin(eng._h, C.byref(desc), N.ptr(Zbad), len(Zbad), d))
    Xs = X[:100]
    for call in (lambda: eng.accumulate(X, y), lambda: eng.finish(), lambda: eng.magic(), lambda: eng.predict(Xs),
                 lambda: eng.cross_kernel(Xs), lambda: eng.kmn_sweep(Xs)):
        with pytest.raises(sg.TrainingVectorsNotInitializedException):
            call()
    eng.begin(k, Z)
    eng.accumulate(X, y)
    G, b = eng.finish()
    G0, b0 = _oracle_stats_chunked(ok, X, y, Z)
    assert rel(G, G0) < TOL_STATS and rel(b, b0) < TOL_STATS


def test_begin_shape_sequence_vs_oracle(eng):
    """Begins that shrink and grow m, d and the non-Eye term count on one context, each followed by a call that AUTO
    sends to the int8 Gram where the kernel qualifies.  The last step goes from an Eye-only kernel to one term at the
    same m and d."""
    rng = np.random.default_rng(32)
    n = 40000
    b8, b20, b4 = np.full(8, np.sqrt(18.0 / 8)), np.full(20, np.sqrt(18.0 / 20)), np.full(4, np.sqrt(9.0 / 4))
    steps = [
        (300, 8, ard(b8)),
        (140, 8, (0.6 * sg.ARDRBFKernel(b8) + 0.4 * sg.RBFKernel(np.sqrt(8 / 36.0)) + sg.const(1e-2) * sg.EyeKernel(),
                  lambda: 0.6 * oracle.ARDRBFKernel(b8) + 0.4 * oracle.RBFKernel(np.sqrt(8 / 36.0))
                  + oracle.const(1e-2) * oracle.EyeKernel())),
        (520, 20, ard(b20)),
        (200, 4, (0.5 * sg.ARDRBFKernel(b4) + 0.3 * sg.ARDRBFKernel(0.5 * b4) + 0.2 * sg.RBFKernel(1.0)
                  + sg.const(1e-2) * sg.EyeKernel(),
                  lambda: 0.5 * oracle.ARDRBFKernel(b4) + 0.3 * oracle.ARDRBFKernel(0.5 * b4) + 0.2 * oracle.RBFKernel(1.0)
                  + oracle.const(1e-2) * oracle.EyeKernel())),
        (200, 8, (sg.const(0.5) * sg.EyeKernel(), lambda: oracle.const(0.5) * oracle.EyeKernel())),
        (200, 8, ard(b8, noise=1.0)),
    ]
    eng.set_precision(N.SGP_PREC_AUTO)
    paths = []
    for m, d, (k, ok) in steps:
        X, y, Z = data(rng, n, m, d)
        eng.begin(k, Z)
        eng.accumulate(X, y)
        paths.append(eng.last_path())
        G, b = eng.finish()
        G0, b0 = _oracle_stats_chunked(ok, X, y, Z)
        eg, eb = rel(G, G0), rel(b, b0)
        print("m=%d d=%d path=%d: dG=%.2e db=%.2e" % (m, d, paths[-1], eg, eb))
        assert G.shape == (m, m) and b.shape == (m,)
        assert eg < TOL_STATS and eb < TOL_STATS
    assert paths[0] == paths[2] == paths[5] == N.SGP_PREC_I8
    assert paths[1] == paths[3] == N.SGP_PREC_I8_DIRECT
    eng.magic()
    Xt = rng.random((300, 8))
    mean, var = eng.predict(Xt)
    m0, v0 = oracle_posterior(steps[-1][2][1], G0, b0, Z, Xt)
    em, ev = rel(mean, m0), float(np.abs(var / v0 - 1).max())
    print("last step: dmean=%.2e dvar=%.2e" % (em, ev))
    assert em < TOL_PRED and ev < TOL_PRED
