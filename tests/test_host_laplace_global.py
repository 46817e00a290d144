"""Host-side checks of the global-memory Laplace path (csrc/laplace_global.cu); no GPU needed.

1. The plan: which kernel the any-size entries run (plan_objective), the workspace of one CTA and the persistent grid
   (laplace_global_grid), mirrored here from constants read out of the sources.
2. The blocked factorisation's tile schedule, replayed in numpy at the tile edges: every tile of every stage is visited
   exactly once, and the replay reproduces scipy.linalg.cholesky, the inverse of L and B^-1 = L^-T L^-1.
"""
import os
import re

import numpy as np
import pytest
import scipy.linalg

from test_host_logic import SMEM_MAX, laplace_smem_bytes, laplace_variant

CSRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "spark_gp_b200", "csrc")
NB, N_VECTORS = 32, 12
CAP_BYTES = 4 << 30
MAX_POINTS = 46336


def read(f):
    with open(os.path.join(CSRC, f)) as fh:
        return fh.read()


# ---- 1. plan mirror --------------------------------------------------------------------------------------------------
def any_size_variant(n_max, d):
    """'staged' / 'global' on chip (laplace_kernel, as sgp_laplace_nll), or 'lapglobal' (laplace_global_kernel)."""
    v = laplace_variant(n_max, d)
    return "lapglobal" if v is None else v


def ld_of(n_max):
    return (n_max + NB - 1) // NB * NB


def cta_bytes(n_max):
    ld = ld_of(n_max)
    return 8 * ld * (2 * ld + NB + N_VECTORS)


def grid(items, resident, cta, budget):
    return max(1, min(items, resident, budget // cta))


def test_mirror_constants_match_source():
    src, internal, bcm = read("laplace_global.cu"), read("sgp_internal.h"), read("bcm_nll.cu")
    assert int(re.search(r"constexpr int NB = (\d+);", src).group(1)) == NB
    assert int(re.search(r"constexpr int kLgVectors = (\d+);", src).group(1)) == N_VECTORS
    m = re.search(r"constexpr size_t kLaplaceGlobalCapBytes = size_t\((\d+)\) << (\d+);", internal)
    assert int(m.group(1)) << int(m.group(2)) == CAP_BYTES
    assert int(re.search(r"constexpr int kLaplaceGlobalMaxPoints = (\d+);", internal).group(1)) == MAX_POINTS
    # the workspace formula: K and M (ld x ld), the panel (NB x ld) and the vectors
    assert re.search(r"static_cast<size_t>\(ld\) \* \(2 \* static_cast<size_t>\(ld\) \+ NB \+ kLgVectors\)", src)
    # the grid: min(items, resident, budget / cta), at least one CTA
    body = re.search(r"long long laplace_global_grid\(.*?\n\}", src, re.S).group(0)
    assert "items < resident" in body and "budget / cta_bytes" in body and "g > 0 ? g : 1" in body
    # one rule: the any-size objective goes global exactly where the on-chip one is refused
    rule = re.search(r"if \(kind == Objective::kLaplace \|\| kind == Objective::kLaplaceAnySize\) \{(.*?)\n  \}", bcm,
                     re.S).group(1)
    assert "laplace_smem_bytes(ex.n_max) > kSmemOptInMax" in rule and "kLaplaceGlobal" in rule
    assert MAX_POINTS ** 2 < 2 ** 31 and ld_of(MAX_POINTS) == MAX_POINTS


def test_boundary_117_on_chip_118_global():
    assert laplace_smem_bytes(117) <= SMEM_MAX < laplace_smem_bytes(118)
    assert any_size_variant(117, 1) == "global" and any_size_variant(117, 784) == "global"
    assert any_size_variant(100, 20) == "staged"
    assert all(any_size_variant(n, 3) == "lapglobal" for n in (118, 128, 500, 2000, 40000))


def test_workspace_and_grid_at_the_cap():
    assert cta_bytes(118) == 8 * 128 * (2 * 128 + 44)
    assert cta_bytes(2000) == 8 * 2016 * (2 * 2016 + 44)            # 65.7 MB per CTA
    # the workspace grows with n_max^2 and the grid, not with the number of experts
    resident = 132
    assert grid(10 ** 6, resident, cta_bytes(500), CAP_BYTES) == resident
    assert grid(12, resident, cta_bytes(1000), CAP_BYTES) == 12           # mnist68 at n_e = 1000: 12 experts
    g = grid(10 ** 6, resident, cta_bytes(4000), CAP_BYTES)               # 257 MB per CTA: the cap binds
    assert g == CAP_BYTES // cta_bytes(4000) == 16 and g * cta_bytes(4000) <= CAP_BYTES
    assert grid(5, resident, cta_bytes(30000), CAP_BYTES) == 1             # one slice above the cap still runs
    assert cta_bytes(75000) > 80 * 10 ** 9                                 # above an 80 GB card: SGP_E_NOMEM


# ---- 2. tile schedule replay -----------------------------------------------------------------------------------------
def padded_b(n, seed):
    """B = I + sqrtW K sqrtW of n points, padded to np = n rounded up to NB with an identity block (the kernel's layout)."""
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, 3))
    K = 1.3 * np.exp(-0.5 * ((X[:, None, :] - X[None, :, :]) ** 2).sum(-1)) + 1e-2 * np.eye(n)
    sw = np.sqrt(rng.uniform(0.05, 0.25, n))
    np_ = ld_of(n)
    B = np.eye(np_)
    B[:n, :n] = np.eye(n) + sw[:, None] * K * sw[None, :]
    return B


def blocked_cholesky(B, visits):
    """lg_cholesky: per panel kb the diagonal block, the panel below (L21 = A21 L11^-T, one tile per warp) and the
    trailing update of the lower tiles (diagonal tiles: their lower triangle)."""
    M = np.tril(B).copy()
    nb = len(M) // NB
    t = lambda i: slice(i * NB, (i + 1) * NB)
    for kb in range(nb):
        L11 = np.linalg.cholesky(M[t(kb), t(kb)] + np.tril(M[t(kb), t(kb)], -1).T)
        M[t(kb), t(kb)] = L11
        visits["diag", kb, kb] += 1
        X11 = np.linalg.inv(L11)
        for I in range(kb + 1, nb):
            M[t(I), t(kb)] = M[t(I), t(kb)] @ X11.T
            visits["panel", I, kb] += 1
        for I in range(kb + 1, nb):                          # for_lower_tiles(kb + 1, nb)
            for J in range(kb + 1, I + 1):
                upd = M[t(I), t(J)] - M[t(I), t(kb)] @ M[t(J), t(kb)].T
                M[t(I), t(J)] = np.tril(upd) if I == J else upd
                visits["trail", kb, I, J] += 1
    return M


def blocked_invert_lower(L, visits):
    """lg_invert_lower: row block I top-down, T_IJ = sum_{K=J}^{I-1} L_IK X_KJ, X_IJ = -X_II T_IJ."""
    M = L.copy()
    nb = len(M) // NB
    t = lambda i: slice(i * NB, (i + 1) * NB)
    for I in range(nb):
        XII = np.linalg.inv(M[t(I), t(I)])
        P = {}
        for J in range(I):
            P[J] = sum(M[t(I), t(K)] @ M[t(K), t(J)] for K in range(J, I))
            visits["inv_T", I, J] += 1
        for J in range(I):
            M[t(I), t(J)] = -XII @ P[J]
            visits["inv_X", I, J] += 1
        M[t(I), t(I)] = np.tril(XII)
    return M


def blocked_ltl(X, visits):
    """lg_ltl: R_IJ = sum_{K>=I} X_KI^T X_KJ for J <= I, row block I top-down, written with its mirror."""
    M = X.copy()
    nb = len(M) // NB
    t = lambda i: slice(i * NB, (i + 1) * NB)
    for I in range(nb):
        P = {}
        for J in range(I + 1):
            P[J] = sum(M[t(K), t(I)].T @ M[t(K), t(J)] for K in range(I, nb))
            visits["ltl", I, J] += 1
        for J in range(I + 1):
            tile = np.tril(P[J]) if J == I else P[J]
            M[t(I), t(J)] = tile
            if J == I:
                M[t(I), t(I)] = tile + np.tril(tile, -1).T
            else:
                M[t(J), t(I)] = tile.T
    return M


@pytest.mark.parametrize("n", [1, 31, 32, 33, 63, 64, 65, 96, 129, 200])
def test_blocked_schedule_visits_every_tile_once_and_reproduces_scipy(n):
    from collections import Counter
    B = padded_b(n, seed=n)
    nb = len(B) // NB
    visits = Counter()
    L = blocked_cholesky(B, visits)
    X = blocked_invert_lower(L, visits)
    R = blocked_ltl(X, visits)
    # each stage visits each of its tiles exactly once
    assert all(v == 1 for v in visits.values())
    assert {k[1:] for k in visits if k[0] == "diag"} == {(kb, kb) for kb in range(nb)}
    assert {k[1:] for k in visits if k[0] == "panel"} == {(I, kb) for kb in range(nb) for I in range(kb + 1, nb)}
    assert {k[1:] for k in visits if k[0] == "trail"} == {(kb, I, J) for kb in range(nb) for I in range(kb + 1, nb)
                                                          for J in range(kb + 1, I + 1)}
    lower_strict = {(I, J) for I in range(nb) for J in range(I)}
    assert {k[1:] for k in visits if k[0] == "inv_T"} == lower_strict
    assert {k[1:] for k in visits if k[0] == "inv_X"} == lower_strict
    assert {k[1:] for k in visits if k[0] == "ltl"} == {(I, J) for I in range(nb) for J in range(I + 1)}
    # the replay reproduces scipy on the expert's block, and the padding stays an identity block
    Bn = B[:n, :n]
    L0 = scipy.linalg.cholesky(Bn, lower=True)
    assert np.abs(L[:n, :n] - L0).max() <= 1e-13 * np.abs(L0).max()
    assert np.abs(X[:n, :n] - scipy.linalg.inv(L0)).max() <= 1e-12 * np.abs(scipy.linalg.inv(L0)).max()
    Binv = scipy.linalg.inv(Bn)
    assert np.abs(R[:n, :n] - Binv).max() <= 1e-12 * np.abs(Binv).max()
    assert np.array_equal(R, R.T)
    assert np.array_equal(L[n:, n:], np.eye(len(B) - n)) and not np.any(L[n:, :n])
    # the sum of log diag L over the expert's rows: log det B / 2
    assert abs(np.log(np.diag(L)[:n]).sum() - 0.5 * np.linalg.slogdet(Bn)[1]) <= 1e-12 * max(1.0, abs(np.linalg.slogdet(Bn)[1]))
