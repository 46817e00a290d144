"""The tail gate of tests/test_gpu_tail.py, checked without a GPU: a numpy restatement of the device tail passes it at the
GPU test's shapes (up to m = 1000), and each plausible bug of `kmm_build_kernel`, `axpby_kernel` or
`magic_matrix_kernel`, restated the same way, fails it.

The restatement follows the device: the active set is laid out as `[n_terms][m_pad][dpad]` rows of z * beta_t (zero
padded, m_pad a multiple of 128), K_mm[i][j] = sum_t C_t exp(-sum_k (z~_ti - z~_tj)^2) + eye_sum on the diagonal,
A = wn K_mm + G, both matrices by Cholesky (LU where it breaks down), M = inv(A) wn - inv(K_mm)."""
import numpy as np
import pytest
import scipy.linalg as sla

import oracle
import spark_gp_b200 as sg
from spark_gp_b200 import _native as N
from test_gpu_tail import CASES, case_id, gate, make_kernel, report, tail_case


def flat_terms(kernel, d):
    """(scales, betas, eye_sum) of the flattened kernel, with RBF as ARD with beta = 1 / (sqrt(2) sigma)."""
    scales, betas, eye = [], [], 0.0
    for t in kernel.flatten():
        if t["type"] == N.SGP_TERM_EYE:
            eye += t["scale"]
            continue
        scales.append(t["scale"])
        betas.append(np.asarray(t["beta"], dtype=np.float64) if t["type"] == N.SGP_TERM_ARD
                     else np.full(d, 1.0 / (np.sqrt(2.0) * t["sigma"])))
    return scales, betas, eye


def device_tail(c, kmm_f32=False, drop_term=None, drop_eye=False, wn=None, stride=None, no_wn_in_m=False, flip=False):
    """The device tail in numpy, with the listed bugs switchable: K_mm rounded to fp32, term `drop_term` left out, the Eye
    sum missing from the diagonal, `wn` in place of the Eye sum as the factor of K_mm in A and of inv(A) in M, active-set
    rows of term t read at t * stride + i instead of t * m_pad + i, inv(A) without wn, M with the wrong sign."""
    m, d = c["m"], c["d"]
    scales, betas, eye = flat_terms(make_kernel(sg, c["kernel"], d, c["sigma2"]), d)
    m_pad, dpad = (m + 127) // 128 * 128, (d + 3) & ~3
    Zs = np.zeros((max(len(scales), 1) * m_pad, dpad))
    for t, beta in enumerate(betas):
        Zs[t * m_pad:t * m_pad + m, :d] = c["Z"] * beta
    K = np.zeros((m, m))
    for t, C in enumerate(scales):
        if t == drop_term:
            continue
        rows = Zs[t * (m_pad if stride is None else stride) + np.arange(m)]
        q = np.zeros((m, m))
        for k in range(dpad):
            df = rows[:, None, k] - rows[None, :, k]
            q += df * df
        K += C * np.exp(-q)
    if not drop_eye:
        K += eye * np.eye(m)
    if kmm_f32:
        K = K.astype(np.float32).astype(np.float64)
    w = eye if wn is None else wn
    A = w * K + c["G"]
    v, inv_a = solve(A, c["b"])
    _, inv_k = solve(K, None)
    M = inv_a * (1.0 if no_wn_in_m else w) - inv_k
    return v, -M if flip else M


def solve(A, b):
    """(A \\ b, inv(A)) by Cholesky; by LU where Cholesky breaks down, as the device's slow path."""
    try:
        f = sla.cho_factor(A, lower=True)
        return (sla.cho_solve(f, b) if b is not None else None), sla.cho_solve(f, np.eye(len(A)))
    except np.linalg.LinAlgError:
        f = sla.lu_factor(A)
        return (sla.lu_solve(f, b) if b is not None else None), sla.lu_solve(f, np.eye(len(A)))


def errors(c, v, M):
    return oracle.tail_errors(c["k0"], c["G"], c["b"], v, M)


@pytest.mark.parametrize("spec", [s for s in CASES if s[0] <= 1000], ids=[case_id(s) for s in CASES if s[0] <= 1000])
def test_restated_tail_passes(spec):
    c = tail_case(*spec)
    e = errors(c, *device_tail(c))
    print(report(c["name"], e))
    assert gate(e), report(c["name"], e)


# each bug on shapes where it matters.  fp32 K_mm is not caught where sigma2 is so small that wn K_mm hardly enters A and
# wn inv(A) dominates M (the tiny-sigma2 regime: omega 13 u there)
@pytest.mark.parametrize("spec", [(300, 16, "bench", "unit", "tall"), (1000, 16, "bench", "unit", "wide"),
                                  (300, 16, "bench", "std", "wide"), (129, 3, "ard_rbf", "std", "tall")])
def test_fp32_kmm_fails(spec):
    c = tail_case(*spec)
    e = errors(c, *device_tail(c, kmm_f32=True))
    print(report(c["name"] + " fp32 K_mm", e))
    assert not gate(e)


@pytest.mark.parametrize("spec", [(129, 3, "ard_rbf", "std", "tall"), (200, 5, "ard_rbf", "unit", "wide"),
                                  (257, 5, "four", "unit", "tall")])
def test_dropped_term_fails(spec):
    c = tail_case(*spec)
    e = errors(c, *device_tail(c, drop_term=1))
    print(report(c["name"] + " term 1 dropped", e))
    assert not gate(e)


@pytest.mark.parametrize("spec", [(300, 16, "bench", "unit", "tall"), (129, 3, "rbf", "unit", "tall"),
                                  (257, 5, "four", "unit", "wide")])
def test_missing_eye_sum_fails(spec):
    c = tail_case(*spec)
    e = errors(c, *device_tail(c, drop_eye=True))
    print(report(c["name"] + " eye_sum missing", e))
    assert not gate(e)


@pytest.mark.parametrize("spec", [(300, 16, "bench", "unit", "tall"), (257, 5, "four", "unit", "tall"),
                                  (129, 3, "rbf", "unit", "wide")])
def test_wrong_wn_fails(spec):
    """wn = 1 instead of the Eye sum, and wn = the coefficient of one of the two Eye terms only."""
    c = tail_case(*spec)
    eyes = [t["scale"] for t in make_kernel(sg, c["kernel"], c["d"], c["sigma2"]).flatten() if t["type"] == N.SGP_TERM_EYE]
    for w in [1.0] + (eyes if len(eyes) == 2 else []):
        assert w != sum(eyes)
        e = errors(c, *device_tail(c, wn=w))
        print(report(c["name"] + " wn=%g" % w, e))
        assert not gate(e)


@pytest.mark.parametrize("m", [129, 200])
@pytest.mark.parametrize("kernel", ["ard_rbf", "four", "nested"])
def test_term_stride_m_fails(m, kernel):
    c = tail_case(m, 5, kernel)
    e = errors(c, *device_tail(c, stride=m))
    print(report(c["name"] + " stride m", e))
    assert not gate(e)


@pytest.mark.parametrize("spec", [(300, 16, "bench", "unit", "tall"), (129, 3, "ard_rbf", "std", "wide"),
                                  (200, 5, "ard_rbf", "unit", "tiny")])
def test_magic_matrix_bugs_fail(spec):
    c = tail_case(*spec)
    for bug in (dict(no_wn_in_m=True), dict(flip=True)):
        e = errors(c, *device_tail(c, **bug))
        print(report(c["name"] + " " + str(bug), e))
        assert not gate(e)
