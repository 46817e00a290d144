"""The BCM objective of several param maps on one grouped upload (run on an H100: `pytest -m gpu`).

`sgp_bcm_nll_slots` evaluates the BCM objective at several kernels on one grouped upload in one launch over experts x
slots.  Slot s must return, bit for bit, what `sgp_bcm_nll` returns on the same upload at the same kernel, whatever else
is in the call, on the register, shared-memory and LU kernels; and every refusal must come before any launch.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

import spark_gp_b200 as sg
from spark_gp_b200 import _native as N
from spark_gp_b200.hyperopt import pack_experts
from spark_gp_b200.utils import kfold_assignment

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

KERNELS = {
    "ard": lambda d: 1.2 * sg.ARDRBFKernel(np.linspace(0.6, 1.1, d)) + sg.const(1e-2) * sg.EyeKernel(),
    "rbf": lambda d: sg.RBFKernel(1.3) + sg.const(1e-2) * sg.EyeKernel(),
    "two_term": lambda d: (1.5 * sg.ARDRBFKernel(np.full(d, 0.7)) + 0.5 * sg.RBFKernel(2.0)
                           + sg.const(1e-2) * sg.EyeKernel()),
    "eye_only": lambda d: sg.const(0.3) * sg.EyeKernel() + sg.const(1e-2) * sg.EyeKernel(),
}


@pytest.fixture(scope="module")
def eng():
    e = sg.ProjectedProcessEngine(0)
    yield e
    e.close()


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.int64)


def data(N_, d, seed):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((N_, d))
    y = np.sin(2 * X[:, 0]) + X[:, -1] + 0.1 * rng.standard_normal(N_)
    return X, y


def theta_of(mk, d, s):
    return mk(d).getHyperparameters() * (1.0 + 0.05 * (s % 7))


def upload(eng, X, y, n_e, f32=False, device=False):
    Xu = X.astype(np.float32) if f32 else X
    if device:
        import torch
        return eng.experts_upload_grouped(torch.as_tensor(Xu, device="cuda:0"), torch.as_tensor(y, device="cuda:0"),
                                          n_e)
    return eng.experts_upload_grouped(Xu, y, n_e)


# P = 1, 2 and 7 at distinct thetas, a call with a repeated theta, one after another on one upload
CALLS = [[0], [1, 2], [0, 1, 2, 3, 4, 5, 6], [3, 3, 5]]


def check_slots(eng, mk, d, calls=CALLS):
    """Each call's slots (each at theta_of(step)) against sgp_bcm_nll on the same upload, bit for bit.  Returns the
    paths the slots calls took."""
    paths = []
    for call in calls:
        kernels = [mk(d).setHyperparameters(theta_of(mk, d, s)) for s in call]
        vals, grads = eng.bcm_nll_slots(kernels)
        paths.append(eng.last_bcm_path())
        for i, k in enumerate(kernels):
            v0, g0 = eng.bcm_nll(k)
            assert bits(vals[i]) == bits(v0), (call, i, vals[i], v0)
            assert np.array_equal(bits(grads[i]), bits(g0)), (call, i)
    return paths


# ---------------- 1. slots against sgp_bcm_nll, bit for bit ------------------------------------------------------------
CASES = [  # (kernel, N, d, n_e, f32, device upload)
    ("ard", 1003, 3, 60, False, False),
    ("rbf", 1501, 2, 100, True, False),
    ("two_term", 1203, 4, 40, False, True),
    ("eye_only", 613, 2, 50, True, True),
    ("ard", 2500, 5, 100, False, True),
]


@pytest.mark.parametrize("kind,N_,d,n_e,f32,device", CASES)
def test_slots_match_single_calls_bitwise(eng, kind, N_, d, n_e, f32, device):
    X, y = data(N_, d, seed=N_ + d)
    upload(eng, X, y, n_e, f32, device)
    assert check_slots(eng, KERNELS[kind], d) == [0] * len(CALLS)


def test_slots_shared_memory_variant():
    """SGP_BCM_IMPL is read once per process: the shared-memory kernel runs in a subprocess."""
    code = ("import numpy as np, sys; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
            "import test_gpu_bcm_slots as t, spark_gp_b200 as sg\n"
            "e = sg.ProjectedProcessEngine(0)\n"
            "X, y = t.data(1203, 3, 5)\n"
            "t.upload(e, X, y, 90)\n"
            "assert t.check_slots(e, t.KERNELS['ard'], 3) == [0] * len(t.CALLS)\n"
            "t.upload(e, X.astype(np.float32), y, 90, device=True)\n"
            "assert t.check_slots(e, t.KERNELS['two_term'], 3) == [0] * len(t.CALLS)\n"
            "print('smem ok')\n" % (ROOT, os.path.join(ROOT, "tests")))
    env = dict(os.environ, SGP_BCM_IMPL="smem")
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "smem ok" in r.stdout, r.stdout + r.stderr


def test_slots_large_experts_lu(eng):
    X, y = data(1600, 3, seed=8)
    upload(eng, X, y, 400)
    assert check_slots(eng, KERNELS["ard"], 3, [[0, 1, 2], [4]]) == [1, 1]


def test_one_slot_breaks_down(eng):
    """A near-duplicate point (1e-9 apart) in one expert: with a 1e-30 Eye term the on-chip Cholesky breaks down and
    the slot runs LU, alone; the slots with a 1e-2 Eye term keep the on-chip bits."""
    N_, d, n_e = 300, 2, 40
    X, y = data(N_, d, seed=21)
    E = upload(eng, X, y, n_e)
    X[E], y[E] = X[0] + 1e-9, y[0]                          # points 0 and E share expert 0
    upload(eng, X, y, n_e)
    mk = lambda c: 1.0 * sg.RBFKernel(1.0) + sg.const(c) * sg.EyeKernel()
    kernels = [mk(1e-2), mk(1e-30), mk(2e-2)]
    vals, grads = eng.bcm_nll_slots(kernels)
    assert eng.last_bcm_path() == 1
    for s, k in enumerate(kernels):
        v0, g0 = eng.bcm_nll(k)
        assert eng.last_bcm_path() == (1 if s == 1 else 0), s
        assert bits(vals[s]) == bits(v0), s
        assert np.array_equal(bits(grads[s]), bits(g0)), s


# ---------------- 2. refusals, before any launch ------------------------------------------------------------------------
def raw_call(eng, n_eval, kernels):
    """sgp_bcm_nll_slots with n_eval given apart from the kernels listed."""
    descs = (N.KernelDesc * max(len(kernels), 1))()
    keep = []
    for i, k in enumerate(kernels):
        desc, arr, nh, kp = eng._descriptors(k)
        descs[i] = desc
        keep.append((arr, kp))
    vals, grads = np.zeros(max(n_eval, 1)), np.zeros(max(n_eval, 1) * 4)
    arr = keep[0][0] if keep else None
    return eng._lib.sgp_bcm_nll_slots(eng._h, n_eval, descs, arr, nh if kernels else 0, N.ptr(vals), N.ptr(grads))


def test_refusals(eng):
    d = 2
    mk = KERNELS["rbf"]
    X, y = data(300, d, seed=1)
    fresh = sg.ProjectedProcessEngine(0)                  # no upload
    fresh._experts_d = d
    with pytest.raises(sg.TrainingVectorsNotInitializedException):
        fresh.bcm_nll_slots([mk(d)])
    fresh.close()
    for up in (lambda: eng.experts_upload_folds(X, y, kfold_assignment(300, 3, 0), 3, 50),
               lambda: eng.experts_upload(*pack_experts(X, y, 50))):
        up()                                                # a fold upload, an upload of given experts: no one set
        launches = eng.launch_count()
        with pytest.raises(sg.TrainingVectorsNotInitializedException, match="grouped"):
            eng.bcm_nll_slots([mk(d)])
        assert eng.launch_count() == launches
    upload(eng, X, y, 50)
    launches = eng.launch_count()
    assert raw_call(eng, 0, [mk(d)]) == N.SGP_E_BADARG
    assert raw_call(eng, 65536, [mk(d)]) == N.SGP_E_BADARG
    with pytest.raises(ValueError, match="same kernel structure"):              # structures differ (one more term)
        eng.bcm_nll_slots([mk(d), mk(d) + sg.const(0.1) * sg.EyeKernel()])
    # the same term types and hyper-parameter count, in another layout: (scale, sigma, sigma) against (sigma, scale, sigma)
    a = 1.0 * sg.RBFKernel(1.0) + sg.const(0.5) * sg.RBFKernel(2.0) + sg.const(1e-2) * sg.EyeKernel()
    b = sg.const(1.0) * sg.RBFKernel(1.0) + 0.5 * sg.RBFKernel(2.0) + sg.const(1e-2) * sg.EyeKernel()
    assert len(a.getHyperparameters()) == len(b.getHyperparameters())
    with pytest.raises(ValueError, match="same kernel structure"):
        eng.bcm_nll_slots([a, b])
    assert eng.launch_count() == launches
    # more than 46340 points in an expert
    rng = np.random.default_rng(2)
    upload(eng, rng.standard_normal((46341, 1)), rng.standard_normal(46341), 46341)
    launches = eng.launch_count()
    with pytest.raises(ValueError, match="46340"):
        eng.bcm_nll_slots([mk(1)] * 2)
    assert eng.launch_count() == launches
    # three experts of 46 000 points: the LU workspace (2 x 3 x 46 000^2 doubles, 102 GB) exceeds the device
    upload(eng, rng.standard_normal((138000, 1)), rng.standard_normal(138000), 46000)
    launches = eng.launch_count()
    with pytest.raises(sg.SgpError, match="error %d" % N.SGP_E_NOMEM):
        eng.bcm_nll_slots([mk(1)] * 2)
    assert eng.launch_count() == launches


def test_singular_slot_is_named(eng):
    """Every point equal and no Eye term to speak of: the kernel matrix is all ones, exactly singular on LU as well."""
    X = np.zeros((200, 2))
    y = np.random.default_rng(3).standard_normal(200)
    upload(eng, X, y, 50)
    mk = lambda c: 1.0 * sg.RBFKernel(1.0) + sg.const(c) * sg.EyeKernel()
    with pytest.raises(sg.MatrixSingularException, match="slot 1:"):
        eng.bcm_nll_slots([mk(1e-2), mk(0.0), mk(1e-2)])
