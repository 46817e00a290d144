"""The BCM objective's general path (LU) on the CPU: a mirror of its plan, and a blockwise fp64 oracle for experts too large
for `oracle.regression` (tests/test_gpu_bcm_general.py checks the GPU against both).

Plan (plan_objective, kLu, csrc/bcm_nll.cu).  The LU path serves every expert set whose largest expert (n_max) does not
fit the on-chip Cholesky, i.e. n_max >= 169.  gen_build_kernel writes each expert's K into an n_max x n_max block of a
global workspace, cuBLAS factors and inverts them, and gen_objective_kernel (one CTA per expert) reads y, alpha and
optionally the expert's rows from shared memory:
  - rows staged iff 8 (2 n + 33) + 8 n (d | 1) <= 200 KiB;
  - y and alpha in shared memory iff 8 (2 n + 33) <= 227 KiB (n <= 14511), else in the workspace;
  - workspace 16 E n^2 + 16 E n + E (16 + 4 (n + 1)) + 256 bytes;
  - refused (SGP_E_BADARG) above 46340 points: the kernel build indexes the n x n matrix in int;
  - SGP_E_NOMEM before allocating when the workspace exceeds free device memory plus what the context holds.

Blockwise oracle.  `regression_likelihood_and_gradient` forms one n x n derivative matrix per hyper-parameter; at
14512 points that is 1.7 GB each.  `blockwise_objective` builds the same K (each element by the oracle's expression),
takes log|det K| and K^-1 from `oracle.regression.log_det_and_inv`, and sums -1/2 dK_i o (alpha alpha' - K^-1) over row
blocks, never holding more than a block of any derivative.  It also returns `gradient_atol`'s bound, computed over the
same blocks, with the condition number from Lanczos iterations on K and K^-1 above 600 points.
"""
import os
import re

import numpy as np
import pytest
import scipy.linalg as sla

import oracle
import oracle.regression
from oracle.kernels import (ARDRBFKernel, ConstantTimesKernel, EyeKernel, RBFKernel, SumOfKernels,
                            TrainableScalarTimesKernel)
from test_host_logic import C_BOUND, EPS, EX_SUMS, SMEM_MAX, SMEM_STAGE_LU, bcm_variant, gradient_atol

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LU_MAX_POINTS = 46340
INT_MAX = 2 ** 31 - 1


# ---------------- plan mirror --------------------------------------------------------------------------------------------
def gen_objective_smem_bytes(n):
    return 8 * (2 * n + 8 + EX_SUMS)


def lu_workspace_bytes(E, n):
    return 2 * E * n * n * 8 + E * 2 * n * 8 + E * (2 * 8 + 4 * (1 + n)) + 256


def lu_plan(E, n_max, d):
    """plan_objective's LU plan: rows staged, y / alpha in the workspace, dynamic shared memory, workspace bytes."""
    base = gen_objective_smem_bytes(n_max)
    staged = base + 8 * n_max * (d | 1) <= SMEM_STAGE_LU
    smem = base + 8 * n_max * (d | 1) if staged else base
    ya_in_ws = smem > SMEM_MAX
    if ya_in_ws:
        smem = gen_objective_smem_bytes(0)
    return dict(staged=staged, ya_in_ws=ya_in_ws, smem=smem, workspace=lu_workspace_bytes(E, n_max))


def lu_outcome(E, n_max, d, free_bytes, held=0):
    """What sgp_bcm_nll returns on the LU path before its first launch: 'badarg', 'nomem' or 'ok'."""
    if n_max > LU_MAX_POINTS:
        return "badarg"
    if lu_plan(E, n_max, d)["workspace"] > free_bytes + held:
        return "nomem"
    return "ok"


def test_lu_plan_thresholds():
    assert min(n for n in range(1, 400) if bcm_variant(n, 1, 1) == "lu") == 169
    assert all(bcm_variant(169, t, d) == "lu" for t in (1, 2, 4) for d in (1, 64))
    for d, last in ((1, 8522), (16, 1345), (33, 730), (64, 381)):           # rows staged up to `last` points
        assert lu_plan(2, last, d)["staged"] and not lu_plan(2, last + 1, d)["staged"], d
    assert lu_plan(1, 14511, 2)["smem"] == gen_objective_smem_bytes(14511) <= SMEM_MAX
    assert gen_objective_smem_bytes(14512) > SMEM_MAX                        # what the launch used to request
    assert not lu_plan(1, 14511, 2)["ya_in_ws"] and lu_plan(1, 14512, 2)["ya_in_ws"]
    for n in list(range(169, 20000, 97)) + [14511, 14512, LU_MAX_POINTS]:    # every LU launch fits the opt-in limit
        for d in (1, 2, 71):
            p = lu_plan(3, n, d)
            assert p["smem"] <= SMEM_MAX and (p["ya_in_ws"] == (n > 14511)) and not (p["ya_in_ws"] and p["staged"])


def test_lu_size_limit_and_memory():
    n = LU_MAX_POINTS
    assert n * n <= INT_MAX < (n + 1) * (n + 1)
    assert (n - 1) * n + (n - 1) <= INT_MAX                   # ex_build_kernel's K[a * ld + b]
    assert n * n - 1 + 256 <= INT_MAX                         # gen_build_kernel's idx after its last step
    big = 1 << 62
    assert lu_outcome(1, n, 1, big) == "ok" and lu_outcome(1, n + 1, 1, big) == "badarg"
    assert lu_outcome(1, 75000, 1, big) == "badarg"           # the size refusal comes before the memory check
    assert lu_workspace_bytes(1, 75000) > 90 * 10 ** 9        # ... and 75 000 points cannot be allocated on 80 GB
    card = 80 * 2 ** 30
    assert lu_workspace_bytes(2600, 2000) > 160 * 10 ** 9 and lu_outcome(2600, 2000, 1, card) == "nomem"
    assert lu_outcome(6, 2000, 1, card) == "ok"
    ws = lu_workspace_bytes(2, 1000)
    assert lu_outcome(2, 1000, 1, ws - 1) == "nomem" and lu_outcome(2, 1000, 1, ws - 1, held=1) == "ok"


def test_lu_plan_mirror_matches_source():
    with open(os.path.join(ROOT, "spark_gp_b200", "csrc", "sgp_internal.h")) as f:
        internal = f.read()
    with open(os.path.join(ROOT, "spark_gp_b200", "csrc", "bcm_nll.cu")) as f:
        bcm = f.read()
    assert int(re.search(r"constexpr int kBcmLuMaxPoints = (\d+);", internal).group(1)) == LU_MAX_POINTS
    assert "return sizeof(double) * (2 * static_cast<size_t>(n_max) + 8 + EX_SUMS);" in bcm
    body = re.search(r"size_t bcm_general_workspace_bytes\(long long E, int n_max\) \{(.*?)\n\}", bcm, re.S).group(1)
    assert "2 * n_max * sizeof(double)" in body and "return 2 * mat + ya +" in body


# ---------------- blockwise oracle ---------------------------------------------------------------------------------------
def _rows_block(kernel, X, r0, r1):
    """(K[r0:r1, :], [dK_i[r0:r1, :]]) of an oracle kernel tree on the training rows X, each element by the expression
    its class's training_kernel_and_derivative uses."""
    A = X[r0:r1]
    if isinstance(kernel, EyeKernel):
        K = np.zeros((r1 - r0, len(X)))
        K[np.arange(r1 - r0), np.arange(r0, r1)] = 1.0
        return K, []
    if isinstance(kernel, ARDRBFKernel):
        K = kernel._kernel_elements(A, X)
        minus2K = -2.0 * K
        derivs = []
        for k in range(X.shape[1]):
            diff = A[:, k, None] - X[None, :, k]
            derivs.append(diff * diff * kernel.beta[k] * minus2K)
        return K, derivs
    if isinstance(kernel, RBFKernel):
        sqd = oracle.kernels._sqdist(A, X)
        K = np.exp(sqd / (-2.0 * kernel.sigma * kernel.sigma))
        return K, [sqd * K / (kernel.sigma ** 3)]
    if isinstance(kernel, TrainableScalarTimesKernel):
        K, d = _rows_block(kernel.kernel, X, r0, r1)
        return K * kernel.C, [K] + [x * kernel.C for x in d]
    if isinstance(kernel, ConstantTimesKernel):
        K, d = _rows_block(kernel.kernel, X, r0, r1)
        return K * kernel.C, [x * kernel.C for x in d]
    if isinstance(kernel, SumOfKernels):
        k1, d1 = _rows_block(kernel.kernel1, X, r0, r1)
        k2, d2 = _rows_block(kernel.kernel2, X, r0, r1)
        return k1 + k2, list(d1) + list(d2)
    raise TypeError("no blockwise form for %s" % type(kernel).__name__)


def _lanczos_top(M, steps=150):
    """Largest eigenvalue of a symmetric M from `steps` Lanczos steps with full reorthogonalisation (a Ritz value: never
    above the true one)."""
    n = len(M)
    steps = min(steps, n)
    Q, a, b = np.zeros((steps, n)), np.zeros(steps), np.zeros(steps)
    q = np.ones(n) / np.sqrt(n)
    m = steps
    last = None
    for j in range(steps):
        Q[j] = q
        w = M @ q
        a[j] = q @ w
        for _ in range(2):
            w -= Q[:j + 1].T @ (Q[:j + 1] @ w)
        b[j] = np.linalg.norm(w)
        if j == steps - 1 or b[j] <= 1e-14 * abs(a[j]):
            m = j + 1
            break
        if j % 10 == 9:                                       # stop once the Ritz value has settled
            top = sla.eigvalsh_tridiagonal(a[:j + 1], b[:j])[-1]
            if last is not None and abs(top - last) <= 1e-14 * abs(top):
                return float(top)
            last = top
        q = w / b[j]
    return float(sla.eigvalsh_tridiagonal(a[:m], b[:m - 1])[-1])


def spd_condition_number(K, Kinv):
    """2-norm condition number of a symmetric positive definite K, what np.linalg.cond returns: exactly up to 600
    points, above from Lanczos on K and K^-1 (at most 1e-3 low where K has a cluster of smallest eigenvalues)."""
    if len(K) <= 600:
        return float(np.linalg.cond(K))
    return _lanczos_top(K) * _lanczos_top(Kinv)


def cholesky_logdet_and_inv(K):
    """log|det K| and K^-1 of a symmetric positive definite K from its Cholesky factor (dpotrf + dpotri).  The LU of
    log_det_and_inv gives the same to rounding on an SPD matrix; at 14 512 points its dgetri takes minutes, this
    seconds."""
    c, lower = sla.cho_factor(K, lower=True)
    logdet = 2.0 * float(np.sum(np.log(np.diag(c))))
    potri, = sla.get_lapack_funcs(("potri",), (c,))
    inv, info = potri(c, lower=1, overwrite_c=1)
    assert info == 0
    inv = np.tril(inv)
    inv += np.tril(inv, -1).T
    return logdet, inv


def blockwise_objective(y, X, kernel_factory, theta, block=256, factor="lu"):
    """(nll, gradient, gradient_atol) of one expert, as oracle.regression.regression_likelihood_and_gradient and
    test_host_logic.gradient_atol compute them, over row blocks of `block` rows.  factor="cholesky" takes log|det K| and
    K^-1 from cholesky_logdet_and_inv instead of the oracle's LU (for experts of many thousand points)."""
    y, X = np.asarray(y, dtype=np.float64), np.asarray(X, dtype=np.float64)
    kernel = kernel_factory().set_hyperparameters(theta)
    n, nh = len(y), len(theta)
    K = np.empty((n, n))
    for r0 in range(0, n, block):
        r1 = min(n, r0 + block)
        K[r0:r1] = _rows_block(kernel, X, r0, r1)[0]
    if factor == "lu":
        _, logdet, kinv = oracle.regression.log_det_and_inv(K)
    else:
        logdet, kinv = cholesky_logdet_and_inv(K)
    alpha = kinv @ y
    nll = 0.5 * float(y @ alpha) + 0.5 * logdet
    abs_alpha = np.abs(alpha)
    grad, bound = np.zeros(nh), np.zeros(nh)
    for r0 in range(0, n, block):
        r1 = min(n, r0 + block)
        _, dK = _rows_block(kernel, X, r0, r1)
        assert len(dK) == nh
        W = np.outer(alpha[r0:r1], alpha) - kinv[r0:r1]
        absW = np.outer(abs_alpha[r0:r1], abs_alpha) + np.abs(kinv[r0:r1])
        for i, d in enumerate(dK):
            grad[i] += float(np.sum(d * W))
            bound[i] += float((np.abs(d) * absW).sum())
    scale = C_BOUND * EPS * (n + spd_condition_number(K, kinv))
    return nll, -0.5 * grad, scale * 0.5 * bound


FAMILIES = {
    "ard": lambda d, b: 1.3 * oracle.ARDRBFKernel(b) + oracle.const(1e-2) * oracle.EyeKernel(),
    "rbf": lambda d, b: (oracle.Scalar(1.5).between(0).and_(30) * oracle.RBFKernel(0.9 * np.sqrt(d), 1e-6, 100)
                         + oracle.WhiteNoiseKernel(0.3, 0, 1) + oracle.const(1e-3) * oracle.EyeKernel()),
    "nested": lambda d, b: (oracle.Scalar(0.7).between(0).and_(10) * (1.5 * oracle.ARDRBFKernel(b)
                                                                      + 0.4 * oracle.RBFKernel(0.9 * np.sqrt(d)))
                            + oracle.WhiteNoiseKernel(0.2, 0, 1) + oracle.const(1e-3) * oracle.EyeKernel()),
    "ard2": lambda d, b: (0.9 * oracle.ARDRBFKernel(b) + 0.6 * oracle.ARDRBFKernel(b[::-1].copy())
                          + oracle.const(1e-2) * oracle.EyeKernel()),
}


@pytest.mark.parametrize("kind,n,d,block", [("ard", 300, 3, 64), ("ard", 257, 17, 100), ("rbf", 300, 4, 37),
                                            ("nested", 280, 5, 256), ("ard2", 310, 2, 1000), ("ard", 1, 2, 8)])
def test_blockwise_oracle_matches_oracle(kind, n, d, block):
    rng = np.random.default_rng(n + d)
    X = rng.standard_normal((n, d))
    y = np.sin(X.sum(1)) + 0.3 * rng.standard_normal(n)
    ofac = lambda: FAMILIES[kind](d, rng_beta)       # noqa: E731
    rng_beta = rng.uniform(0.3, 3.0, d) / np.sqrt(d)
    theta = ofac().get_hyperparameters()
    l0, g0 = oracle.regression.regression_likelihood_and_gradient(y, ofac().set_training_vectors(X), theta)
    K, dK = ofac().set_hyperparameters(theta).set_training_vectors(X).training_kernel_and_derivative()
    atol0 = gradient_atol(K, dK, y)
    l, g, atol = blockwise_objective(y, X, ofac, theta, block)
    assert l == l0                                            # same K, same LU
    assert np.allclose(atol, atol0, rtol=1e-9, atol=0)
    # 1e-13 relative; a component that cancels to well below its terms differs by the rounding of its sum order, a
    # thousandth of the GPU gate (test_gpu_objectives: 1e-12 |g0| + atol)
    err = np.abs(g - g0)
    assert np.all(err <= 1e-13 * np.abs(g0) + 1e-3 * atol0), err / (1e-13 * np.abs(g0) + 1e-3 * atol0)


@pytest.mark.parametrize("kind,n,d", [("ard", 700, 2), ("nested", 400, 3)])
def test_cholesky_form_matches_lu_oracle(kind, n, d):
    """The Cholesky form the 14 511 / 14 512-point GPU cases use agrees with the LU oracle far inside the GPU gate."""
    rng = np.random.default_rng(n)
    X = rng.standard_normal((n, d))
    y = np.sin(X.sum(1)) + 0.3 * rng.standard_normal(n)
    b = rng.uniform(0.3, 3.0, d) / np.sqrt(d)
    ofac = lambda: FAMILIES[kind](d, b)                  # noqa: E731
    theta = ofac().get_hyperparameters()
    l0, g0, atol = blockwise_objective(y, X, ofac, theta)
    l, g, atol_c = blockwise_objective(y, X, ofac, theta, factor="cholesky")
    assert abs(l - l0) <= 1e-13 * abs(l0)
    assert np.all(np.abs(g - g0) <= 1e-13 * np.abs(g0) + 1e-3 * atol)
    assert np.allclose(atol_c, atol, rtol=1e-9, atol=0)


@pytest.mark.parametrize("n,d,lay", [(900, 2, "standardised"), (1500, 2, "clustered"), (1000, 17, "standardised")])
def test_condition_number_by_lanczos(n, d, lay):
    """Close to np.linalg.cond and never above it: the gate it sets is at most 1e-3 tighter than gradient_atol's."""
    rng = np.random.default_rng(n + d)
    if lay == "standardised":
        X = rng.standard_normal((n, d))
    else:
        X = rng.random((n, d)) + 300.0 * rng.integers(0, 4, (n, 1))
    K = (1.3 * oracle.ARDRBFKernel(rng.uniform(0.3, 1.2, d)) + oracle.const(1e-2) * oracle.EyeKernel()
         ).set_training_vectors(X).training_kernel()
    kappa, exact = spd_condition_number(K, np.linalg.inv(K)), np.linalg.cond(K)
    assert 1 - 1e-3 <= kappa / exact <= 1 + 1e-12, kappa / exact
