"""CPU tests of the extended-precision kernel evaluation model (oracle/kernel_eval_model.py) that the GPU tests of
tests/test_gpu_kernel_eval_bounds.py judge every element by.  The model agrees with the oracle's fp64 kernels, and its
per-element bound is sharp: a float64 restatement of csrc/kernel_eval.cu's arithmetic stays inside it on every case, and
each planted bug of the kind the 1e-13-of-the-largest-entry tolerance lets through breaks it."""
import numpy as np
import pytest

import oracle
import spark_gp_b200 as sg
from oracle.kernel_eval_model import KernelEvalModel, bound_fraction, kernel_shapes
from spark_gp_b200 import _native as N

LD = np.longdouble
K_MAX_TERMS = 4          # sgp_internal.h: kMaxTerms


def oracle_eval(ok, A, B=None):
    """The oracle's (K, dK): trainingKernelAndDerivative on A, or for CROSS the A x B block of it on [A; B]."""
    if B is None:
        K, dK = ok.set_training_vectors(A).training_kernel_and_derivative()
        return K, np.array(dK).reshape(-1, len(A), len(A))
    n = len(A)
    K, dK = ok.set_training_vectors(np.vstack([A, B])).training_kernel_and_derivative()
    return K[:n, n:], np.array(dK).reshape(-1, len(K), len(K))[:, :n, n:]


@pytest.mark.parametrize("d", [1, 3, 33, 100])
def test_model_matches_oracle(d):
    rng = np.random.default_rng(100 + d)
    A, B = rng.random((23, d)), rng.random((41, d))
    for name, f in kernel_shapes(rng, d):
        ok = f(oracle)
        model = KernelEvalModel(ok)
        assert len(model.hypers) == ok.number_of_hyperparameters(), name
        for mode, args in (("training", (A,)), ("cross", (A, B))):
            K, _, dK, _ = model.evaluate(*args)
            K0, dK0 = oracle_eval(ok, *args)
            assert dK.shape == dK0.shape, (name, mode)
            for got, ref in zip([K] + list(dK), [K0] + list(dK0)):
                scale = max(np.abs(ref).max(), 1e-300)
                assert np.abs(got.astype(np.float64) - ref).max() <= 1e-13 * scale, (name, mode)


# ---- a float64 restatement of csrc/kernel_eval.cu, with planted bugs ------------------------------------------------

def fma(a, b, c):
    """fma in float64 through longdouble: within a 2^-11 fraction of an ulp of the fused result where nothing cancels
    by more than 2^11, far inside the model's bound elsewhere."""
    return (np.asarray(a, LD) * np.asarray(b, LD) + np.asarray(c, LD)).astype(np.float64)


BUGS = ["drop_chunk_dim", "ard_beta_squared", "neighbour_e", "rbf_no_scale", "eye_next_row", "rbf_sigma_squared",
        "scale_coef_of_next_term"]


def gpu_form(kernel, A, B=None, bug=None):
    """(K, dK) of a library kernel in float64 as kernel_eval_kernel computes them, from the flattened kernel and the
    hyper-parameter descriptors the library receives (kernel_eval_setup's tables rebuilt here)."""
    training = B is None
    B = A if training else B
    (n, d), m = A.shape, len(B)
    terms, hd = kernel.flatten(), kernel.hyper_descriptors()
    flat_of, flat = {}, []
    eye_sum = 0.0
    for i, t in enumerate(terms):
        if t["type"] == N.SGP_TERM_EYE:
            eye_sum += t["scale"]
        else:
            flat_of[i] = len(flat)
            flat.append(t)
    T = len(flat)
    betas = [np.asarray(t["beta"], np.float64) if t["type"] == N.SGP_TERM_ARD
             else np.full(d, 1.0 / (np.sqrt(2.0) * t["sigma"])) for t in flat]
    e, K = [], np.zeros((n, m))
    for t in range(T):
        beta, q = betas[t], np.zeros((n, m))
        for k in range(d):
            if bug == "drop_chunk_dim" and k == min(31, d - 1):
                continue
            a, b = A[:, k, None], B[None, :, k]
            df = a * beta[k] - b * beta[k] if training else fma(a, beta[k], -(b * beta[k]))
            q = fma(df, df, q)
        e.append(np.exp(-q))
        K = fma(flat[t]["scale"], e[t], K)
    diag = np.eye(n, m, k=-1 if bug == "eye_next_row" else 0, dtype=bool) & training
    K = np.where(diag, K + eye_sum, K)
    dsq = [(A[:, k, None] - B[None, :, k]) ** 2 for k in range(d)]
    s2 = np.zeros((n, m))
    for k in range(d):
        s2 = s2 + dsq[k]
    dK = np.empty((len(hd), n, m))
    for h, hp in enumerate(hd):
        if hp["kind"] == N.SGP_HYPER_SCALE:
            cf = np.zeros(K_MAX_TERMS + 1)
            for i, c in hp["coef"].items():
                cf[flat_of.get(i, K_MAX_TERMS)] += c
            v = np.zeros((n, m))
            for t in range(T):
                v = fma(cf[(t + 1) % T if bug == "scale_coef_of_next_term" else t], e[t], v)
            dK[h] = np.where(diag, v + cf[K_MAX_TERMS], v)
            continue
        t = flat_of[hp["term"]]
        C = flat[t]["scale"]
        if hp["kind"] == N.SGP_HYPER_ARD_BETA:
            k, bk = hp["dim"], betas[t][hp["dim"]]
            c2 = -2.0 * (bk * bk if bug == "ard_beta_squared" else bk)
            et = e[(t + 1) % T] if bug == "neighbour_e" else e[t]
            dK[h] = (c2 * dsq[k]) * (C * et)
        else:
            sig = flat[t]["sigma"]
            sig3 = sig * sig if bug == "rbf_sigma_squared" else sig * sig * sig
            dK[h] = (s2 * e[t] / sig3) * (1.0 if bug == "rbf_no_scale" else C)
    return K, dK


def cases():
    """(label, library kernel, model, A, B or None): every kernel shape in both modes at d = 5 and 33 on [0, 1), and
    the multi-term shapes with A and B offset by 1e3 / beta."""
    out = []
    for d in (5, 33):
        rng = np.random.default_rng(d)
        A, B = rng.random((19, d)), rng.random((26, d))
        for name, f in kernel_shapes(rng, d):
            model = KernelEvalModel(f(oracle))
            out += [("%s d=%d training" % (name, d), f(sg), model, A, None),
                    ("%s d=%d cross" % (name, d), f(sg), model, A, B)]
            if name in ("nested", "four", "scaled_sum"):
                off = 1e3 / max(float(np.max(model.beta(t, d))) for t in range(len(model.terms)))
                out.append(("%s d=%d cross at 1e3" % (name, d), f(sg), model, A + off, B + off))
    return out


CASES = cases()


def fractions(bug=None):
    """Largest fraction of the bound used per case, over K and every dK."""
    out = {}
    for label, k, model, A, B in CASES:
        K, bK, dK, bdK = model.evaluate(A, B)
        gK, gdK = gpu_form(k, A, B, bug)
        out[label] = max([bound_fraction(gK, K, bK)] + [bound_fraction(g, x, b) for g, x, b in zip(gdK, dK, bdK)])
    return out


def test_gpu_form_within_bound():
    fr = fractions()
    worst = max(fr, key=fr.get)
    print("\nclean float64 restatement: largest fraction of the bound %.3g (%s)" % (fr[worst], worst))
    assert fr[worst] <= 1.0, worst


@pytest.mark.parametrize("bug", BUGS)
def test_planted_bug_breaks_bound(bug):
    fr = fractions(bug)
    worst = max(fr, key=fr.get)
    print("\n%s: largest fraction of the bound %.3g (%s)" % (bug, fr[worst], worst))
    assert fr[worst] > 1.0
