"""CPU tests of the kernel DSL's evaluation methods (setTrainingVectors, trainingKernel, trainingKernelDiag,
trainingKernelAndDerivative, crossKernel, selfKernel) with a stand-in engine: what each method hands the library, the
shapes and dtypes it returns, the hyper-parameter order of the derivatives, and the diagonal quantities computed on the
host against the oracle."""
import numpy as np
import pytest

import oracle
import spark_gp_b200 as sg
from spark_gp_b200 import _native as N
from spark_gp_b200.engine import ProjectedProcessEngine


class _StandIn:
    """Records each kernel_eval call and returns K[i][j] = 1000 i + j (and dK[h] = K + h) of the requested shape."""
    calls = []

    def __init__(self, device):
        self.device, self.released = device, False

    def kernel_eval(self, kernel, A, B, derivatives):
        _StandIn.calls.append(dict(eng=self, kernel=kernel, A=A, B=B, derivatives=derivatives))
        n, m = len(A), len(A) if B is None else len(B)
        K = 1000.0 * np.arange(n)[:, None] + np.arange(m)[None, :]
        nh = kernel.numberOfHyperparameters()
        return K, (K[None] + np.arange(nh)[:, None, None] if derivatives else None)

    def release(self):
        self.released = True


@pytest.fixture
def stand_in(monkeypatch):
    _StandIn.calls = []
    monkeypatch.setattr(ProjectedProcessEngine, "acquire", classmethod(lambda cls, device=0: _StandIn(device)))
    return _StandIn


def composite(d):
    """A kernel with nested trainable scalars, a constant, ARD, RBF and Eye terms (library, oracle)."""
    beta = np.linspace(0.0, 1.5, d)
    lib = (sg.Scalar(0.7) * (2.0 * sg.ARDRBFKernel(beta) + sg.Scalar(0.3) * sg.RBFKernel(1.7))
           + sg.const(0.25) * sg.EyeKernel() + sg.WhiteNoiseKernel(0.1, 0.0, 1.0))
    orc = (oracle.Scalar(0.7) * (2.0 * oracle.ARDRBFKernel(beta) + oracle.Scalar(0.3) * oracle.RBFKernel(1.7))
           + oracle.const(0.25) * oracle.EyeKernel() + oracle.WhiteNoiseKernel(0.1, 0.0, 1.0))
    return lib, orc


@pytest.mark.parametrize("call", ["trainingKernel", "trainingKernelDiag", "trainingKernelAndDerivative",
                                  "getTrainingVectors", "crossKernel"])
def test_not_initialised(stand_in, call):
    k = 1 * sg.RBFKernel(0.5) + sg.const(0.1) * sg.EyeKernel()
    args = (np.zeros((2, 3)),) if call == "crossKernel" else ()
    with pytest.raises(sg.TrainingVectorsNotInitializedException):
        getattr(k, call)(*args)
    assert stand_in.calls == []


def test_training_kernel_hands_the_vectors_over(stand_in):
    k, _ = composite(3)
    X = np.arange(12, dtype=np.float32).reshape(4, 3)
    assert k.setTrainingVectors(X, device=1) is k
    K = k.trainingKernel()
    (c,) = stand_in.calls
    assert c["eng"].device == 1 and c["eng"].released and c["B"] is None and not c["derivatives"]
    assert c["A"].dtype == np.float32 and np.array_equal(c["A"], X)   # float32 is kept for the library to convert
    assert K.shape == (4, 4) and K.dtype == np.float64


def test_training_kernel_and_derivative_shapes(stand_in):
    k, _ = composite(3)
    k.setTrainingVectors(np.arange(15).reshape(5, 3))                  # ints become float64
    K, dK = k.trainingKernelAndDerivative()
    (c,) = stand_in.calls
    assert c["A"].dtype == np.float64 and c["derivatives"]
    assert K.shape == (5, 5) and dK.shape == (k.numberOfHyperparameters(), 5, 5)
    assert np.array_equal(dK[2], K + 2)                                # dK[i] is the i-th matrix


def test_cross_kernel_matrix_and_single_vector(stand_in):
    k = sg.ARDRBFKernel(np.array([0.2, 0.3]))
    train = np.array([[1.0, 2.0], [2.0, 3.0], [5.0, 7.0]])
    k.setTrainingVectors(train)
    K = k.crossKernel(np.ones((4, 2)))
    assert K.shape == (4, 3)
    row = k.crossKernel(np.array([1.0, 2.0]))                          # Kernel.scala:81-84
    assert row.shape == (3,) and np.array_equal(row, [0.0, 1.0, 2.0])
    a, b = stand_in.calls
    assert b["A"].shape == (1, 2) and np.array_equal(b["B"], train) and not b["derivatives"]


def test_training_vectors_reach_every_sub_kernel(stand_in):
    k, _ = composite(2)
    X = np.ones((3, 2))
    k.setTrainingVectors(X)
    assert np.array_equal(k.kernel1.kernel1.kernel.kernel2.getTrainingVectors(), X)
    single = sg.RBFKernel(1.0).setTrainingVectors(np.array([1.0, 2.0]))
    assert single.getTrainingVectors().shape == (1, 2)


@pytest.mark.parametrize("d", [1, 4])
def test_descriptors_follow_get_hyperparameters(d):
    """The descriptors passed with the derivatives are in getHyperparameters order: each ARD and RBF descriptor carries
    the hyper-parameter at its position, and a trainable scalar's SCALE descriptor sits at its C."""
    k, _ = composite(d)
    theta = k.getHyperparameters()
    _, arr, nh, _ = ProjectedProcessEngine._descriptors(None, k, d)
    assert nh == len(theta) == k.numberOfHyperparameters()
    kinds = [arr[i].kind for i in range(nh)]
    assert kinds == [N.SGP_HYPER_SCALE, N.SGP_HYPER_SCALE] + [N.SGP_HYPER_ARD_BETA] * d \
        + [N.SGP_HYPER_SCALE, N.SGP_HYPER_RBF_SIGMA, N.SGP_HYPER_SCALE]
    for i in range(nh):
        if arr[i].kind != N.SGP_HYPER_SCALE:
            assert arr[i].value == theta[i]
    assert [arr[i].dim for i in range(2, 2 + d)] == list(range(d))


@pytest.mark.parametrize("d", [1, 5])
def test_self_kernel_and_diag_against_oracle(stand_in, d):
    k, o = composite(d)
    X = np.random.default_rng(0).random((6, d))
    k.setTrainingVectors(X)
    o.set_training_vectors(X)
    assert k.selfKernel(X[0]) == pytest.approx(o.self_kernel(X[0]), rel=1e-15)
    diag = k.trainingKernelDiag()
    assert diag.shape == (6,) and diag.dtype == np.float64
    assert np.allclose(diag, o.training_kernel_diag(), rtol=1e-15, atol=0)
    assert np.allclose(diag, np.diag(o.training_kernel()), rtol=1e-15, atol=0)
    assert stand_in.calls == []                                        # no library call
