"""CPU-side checks of the device-resident fit: the ungroup permutation of `sgp_experts_get_f_rows_device` restated in
numpy against the grouping, the mode-store selector against the header, and the host side of the row helpers."""
import os
import re

import numpy as np
import pytest

from spark_gp_b200 import _native as N
from spark_gp_b200.engine import host_copy, rows_to_host, take_rows
from spark_gp_b200.hyperopt import group_for_experts, pack_experts

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def ungroup_source(n: int, E: int):
    """ungroup_experts_kernel: row i reads the packed position of expert i % E's (i / E)-th point; the first n % E
    experts own one point more."""
    i = np.arange(n)
    e, pos = i % E, i // E
    kq, r = divmod(n, E)
    return e * kq + np.minimum(e, r) + pos


@pytest.mark.parametrize("n,n_e", [(1, 1), (51, 100), (90, 100), (437, 40), (620, 150), (1000, 100), (1353, 100),
                                   (999, 7), (5, 2)])
def test_ungroup_is_the_inverse_of_the_grouping(n, n_e):
    order = np.concatenate(group_for_experts(n, n_e))       # packed position p holds row order[p]
    E = len(group_for_experts(n, n_e))
    src = ungroup_source(n, E)
    assert np.array_equal(order[src], np.arange(n))          # row i reads its own packed position
    rng = np.random.default_rng(n)
    X, y = rng.standard_normal((n, 2)), rng.standard_normal(n)
    _, yp, _ = pack_experts(X, y, n_e)
    assert np.array_equal(yp[src], y)                        # ungrouping the packed labels gives them back in row order
    latent = np.empty(n)
    latent[order] = yp                                       # the host reorder of laplace_fit
    assert np.array_equal(latent, yp[src])


def test_mode_store_selector_matches_header():
    src = open(os.path.join(ROOT, "include", "sgp.h")).read()
    m = re.search(r"enum\s*\{\s*SGP_MODES_BINARY\s*=\s*(\d+),\s*SGP_MODES_CLASS\s*=\s*(\d+),\s*SGP_MODES_SLOT\s*=\s*(\d+)", src)
    assert m is not None
    assert tuple(int(v) for v in m.groups()) == (N.SGP_MODES_BINARY, N.SGP_MODES_CLASS, N.SGP_MODES_SLOT)


def test_device_entries_are_bound():
    for name in ("sgp_experts_upload_grouped_device", "sgp_experts_upload_folds_device", "sgp_experts_get_f_rows_device",
                 "sgp_kmeans_device", "sgp_greedy_active_set_device"):
        assert name in N.EXPORTS


def test_row_helpers_on_host_arrays():
    X = np.arange(24, dtype=np.float32).reshape(8, 3)
    idx = np.array([5, 0, 5, 7])
    assert np.array_equal(take_rows(X, idx), X[idx]) and take_rows(X, idx).dtype == np.float32
    got = rows_to_host(X, idx)
    assert got.dtype == np.float64 and np.array_equal(got, X[idx].astype(np.float64))
    assert host_copy(X) is X
