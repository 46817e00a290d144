"""`sgp_kmeans` (csrc/kmeans.cu) pinned bit for bit to its exact model (oracle/kmeans_model.py) on real-valued data, on
one H100 (`pytest -m gpu`).

Every case of oracle/kmeans_cases.py first checks, on the model's instrumentation, that it reaches the edge it names
(fp32 / fp64 flips, candidate counts and k-means++ segments, stream-101 draws, empty clusters, exact ties, chunks, the
prescale), then compares the centres, k_out, labels, iterations and cost with the model's, bit for bit, through the host
entry (fp64 and, where the case allows, fp32 X) and the device entry.  The refused cases must raise SGP_E_RANGE."""
import numpy as np
import pytest

from oracle import kmeans as okm
from oracle import kmeans_cases as kc
import spark_gp_b200 as sg
from spark_gp_b200.engine import OperandRangeError

pytestmark = pytest.mark.gpu
CASES = kc.catalogue()


@pytest.fixture(scope="module")
def eng():
    e = sg.ProjectedProcessEngine(0)
    yield e
    e.close()


def bits(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64)).view(np.int64)


def same(got, want, what):
    C, lab, it, cost = got
    Cm, labm, itm, costm = want
    assert C.shape == Cm.shape, "%s: k_out %d, model %d" % (what, len(C), len(Cm))
    assert np.array_equal(bits(C), bits(Cm)), "%s: centres differ in %d entries" % (what, int((bits(C) != bits(Cm)).sum()))
    assert np.array_equal(lab, labm), "%s: %d labels differ" % (what, int((lab != labm).sum()))
    assert it == itm, "%s: iterations %d, model %d" % (what, it, itm)
    assert bits(cost) == bits(costm), "%s: cost %r, model %r" % (what, cost, costm)


@pytest.mark.parametrize("name", list(CASES))
def test_kmeans_equals_its_model(eng, name):
    import torch
    case = CASES[name]()
    kw = dict(max_iter=case["max_iter"], tol=case["tol"], seed=case["seed"], init_centers=case["init"])
    for f32 in ([False, True] if case["f32"] else [False]):
        X = case["X"].astype(np.float32) if f32 else case["X"]
        want, info = kc.run_model(case, f32=f32)
        forms = [("host", X), ("device", torch.as_tensor(X, device="cuda:0"))]
        if case["refused"]:
            assert want is None
            for form, Xf in forms:
                with pytest.raises(OperandRangeError):
                    eng.kmeans(Xf, case["k"], **kw)
            continue
        kc.check_claims(case, info)
        for form, Xf in forms:
            same(eng.kmeans(Xf, case["k"], **kw), want, "%s %s" % (form, "fp32" if f32 else "fp64"))
        if name.startswith("near_tie") and not f32:
            # the pin is sharper than the fp64 restatement: it differs from the model on these cases
            o = okm.kmeans(X, case["k"], **kw)
            assert not (np.array_equal(o[1], want[1]) and np.array_equal(bits(o[0]), bits(want[0]))
                        and o[2] == want[2] and bits(o[3]) == bits(want[3]))

