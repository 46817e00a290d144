"""SGP_PREC_I8 on the device against the oracle at active-set sizes between the existing cases (m = 600: 5 tiles,
m = 1100: 9 tiles), where the producer splits the points into its own slices (52 and 29 on 132 SMs, two CTAs per SM)
and the Gram into others: b is summed over the producer's slices, G over the Gram's."""
import numpy as np
import pytest

import spark_gp_b200 as sg
from spark_gp_b200 import _native as N
from test_gpu_entry_points import TOL_STATS, TiledOracle, ard_pair, rel, stats_device, tiled, to_device

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    e = sg.ProjectedProcessEngine(0)
    yield e
    e.close()


@pytest.mark.parametrize("m", [600, 1100])
def test_i8_producer_split_vs_oracle(eng, m):
    d, n = 8, 250_000
    rng = np.random.default_rng(m)
    Xb = rng.random((4096, d), dtype=np.float32)
    yb = np.sin(Xb.astype(np.float64).sum(1)) + 0.1 * rng.standard_normal(len(Xb))
    Z = rng.random((m, d))
    k, ok = ard_pair(np.full(d, np.sqrt(18.0 / d)))
    G0, b0 = TiledOracle(ok, Xb, yb, Z).stats(n)
    G, b, path = stats_device(eng, k, to_device(tiled(Xb, n)), to_device(tiled(yb, n)), Z, N.SGP_PREC_I8)
    assert path == N.SGP_PREC_I8
    assert rel(G, G0) <= TOL_STATS and rel(b, b0) <= TOL_STATS
    assert np.array_equal(G, G.T)
