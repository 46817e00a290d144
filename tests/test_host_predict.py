"""CPU mirror of the variance kernel's schedule (spark_gp_b200/csrc/predict.cu): the triangular packed form
B = triu(M + M^T, 1) + diag(M) and the (row tile, column tile) rasterisation, with the tile constants read from the source.

A CTA (R, C) accumulates W_RC = sum_{I <= C} K_RI B_IC over k chunks of kVarK and folds sum_c W_rc K_rc; the variance of a
point is selfKernel plus the sum of its column-tile partials.  Here the same loop runs in numpy: every (I <= C) block pair
must be visited exactly once per row tile, and the packed sum must equal k M k^T for an M that is not symmetric."""
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = open(os.path.join(ROOT, "spark_gp_b200", "csrc", "predict.cu")).read()


def const(name):
    return int(re.search(r"constexpr int %s = (\d+);" % name, SRC).group(1))


ROWS, COLS, KCH, GROUP = const("kVarRows"), const("kVarCols"), const("kVarK"), const("kVarGroup")
TILE = 128                                            # kTile: m_pad is a multiple of it (sgp_internal.h)
M_EDGES = [1, 63, 64, 65, 127, 128, 129, 1000, 2100, 4000]


def var_tile(b, n_rt, n_ct):
    """var_tile() of predict.cu."""
    g = b // (GROUP * n_ct)
    rows = min(GROUP, n_rt - g * GROUP)
    local = b - g * GROUP * n_ct
    return g * GROUP + local % rows, n_ct - 1 - local // rows


def pack(M, m_pad):
    m = len(M)
    B = np.zeros((m_pad, m_pad))
    B[:m, :m] = np.triu(M + M.T, 1) + np.diag(np.diag(M))
    return B


def schedule(m, n):
    """(row tile, column tile, k chunks) of every CTA of one launch, as launch_predict grids it."""
    n_ct = (m + COLS - 1) // COLS
    n_rt = (n + ROWS - 1) // ROWS
    for b in range(n_rt * n_ct):
        rt, ct = var_tile(b, n_rt, n_ct)
        yield rt, ct, range((ct + 1) * (COLS // KCH))


def test_constants_fit_the_layout():
    assert COLS % KCH == 0 and TILE % COLS == 0 and ROWS % 8 == 0 and KCH % 4 == 0


@pytest.mark.parametrize("m", M_EDGES)
@pytest.mark.parametrize("n", [1, 129, ROWS * GROUP * 2 + 5])
def test_every_block_pair_once(m, n):
    m_pad = (m + TILE - 1) // TILE * TILE
    n_ct = (m + COLS - 1) // COLS
    assert n_ct * COLS <= m_pad                       # the B and K columns a CTA stages exist
    seen = {}
    for rt, ct, chunks in schedule(m, n):
        for kc in chunks:
            blk = kc * KCH // COLS                    # the 64-wide block I this chunk belongs to
            assert blk <= ct
            seen[(rt, blk, ct)] = seen.get((rt, blk, ct), 0) + 1
    n_rt = (n + ROWS - 1) // ROWS
    expect = {(r, i, c): COLS // KCH for r in range(n_rt) for c in range(n_ct) for i in range(c + 1)}
    assert seen == expect                             # each (I <= C) pair once: COLS / KCH chunks of it, no more


@pytest.mark.parametrize("m", M_EDGES)
def test_packed_form_is_the_quadratic_form(m):
    rng = np.random.default_rng(m)
    n = 37
    m_pad = (m + TILE - 1) // TILE * TILE
    M = rng.standard_normal((m, m)) * 30.0            # not symmetric
    K = np.zeros((n, m_pad))
    K[:, :m] = rng.random((n, m))
    B = pack(M, m_pad)
    n_ct = (m + COLS - 1) // COLS
    part = np.zeros((n_ct, n))
    for ct in range(n_ct):
        c0 = ct * COLS
        W = np.zeros((n, COLS))
        for kc in range((ct + 1) * (COLS // KCH)):
            k0 = kc * KCH
            W += K[:, k0:k0 + KCH] @ B[k0:k0 + KCH, c0:c0 + COLS]
        part[ct] = (W * K[:, c0:c0 + COLS]).sum(1)
    var = part.sum(0)
    ref = np.einsum("ti,ij,tj->t", K[:, :m], M, K[:, :m])
    scale = np.einsum("ti,ij,tj->t", K[:, :m], np.abs(M), K[:, :m])
    assert float((np.abs(var - ref) / scale).max()) < 1e-13
