"""CPU tests of the extended-precision model of prediction (oracle/predict_model.py) that tests/test_gpu_predict_bounds.py
judges every element, mean, variance and averaged probability by.  The arithmetic the model transcribes is read from
the kernel source, the model agrees with the oracle, and its bounds are sharp: a numpy restatement of the three
prediction kernels stays inside them on every case, and each planted bug below passes the gates of the existing GPU
tests (1e-11 of the summed magnitudes for the mean and variance, 3e-14 absolute for p) but breaks a bound.

Measured (each planted bug's error under the old gate, then its largest fraction of the new bound; the same case as
written stays at or below 0.45):
  * staging without the centre, 1e3 length scales out (d = 4, m = 150): mean 1.4e-14 and variance 4.2e-15 of the
    summed magnitudes; elements 286 and mean 6.2 times their bounds.
  * `exp` skipped past q = 60 (two clusters 10 length scales apart): mean 1.8e-16; elements 8e12 times their bound.
  * sigmoid as 1 - 1/(1 + exp(z)), means -40 .. -25: p off by 1.1e-16 absolute; 6e13 times its bound.
A variance-only bug the 1e-11 gate misses: the variance is judged per point against the same summed magnitudes,
selfKernel + (k + a)|B|(k + a)^T, with gamma(R_var) ~ (m + m/64 + 12) u in place of 1e-11 -- 2.4e-14 at m = 150, 420
times tighter.  Staging without the centre at 1e4 length scales in the variance's K only (the mean's K as written, as a
variance path that restaged the points would have it) moves the variance by 5.3e-14 of its scale: far under the gate,
2.1 times the bound.  At 1e3 length scales the same bug moves it by 4.2e-15, 0.17 of the bound: a variance-only error
below ~5e-15 of the summed magnitudes is rounding-sized and no per-point bound can tell it from rounding.
"""
import os
import re

import numpy as np
import pytest

import oracle
from oracle.gram_f64_model import centre
from oracle.integrator import averaged_probability
from oracle.predict_model import (ELEM_COLS, ELEM_PTS, LD, RSQRT_PI, VAR_COLS, VAR_ROWS, PredictModel, bound_fraction,
                                  fractions, m_padded, probability, probability_fraction, reference_share, rounding_counts,
                                  sample_points)
from spark_gp_b200 import _native as N
from test_gpu_predict import make_case, points

CSRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "spark_gp_b200", "csrc")
TOL, TOL_P = 1e-11, 3e-14
NODES = [1, 2, 100, 256]


def src(name):
    return open(os.path.join(CSRC, name)).read()


def const(text, name):
    return int(re.search(r"constexpr int %s = (\d+);" % name, text).group(1))


# ---- the arithmetic the model transcribes, read from the source -----------------------------------------------------
def test_mirrors_match_source():
    pred, api, misc, internal = src("predict.cu"), src("api.cu"), src("misc_kernels.cu"), src("sgp_internal.h")
    # staging: x~ centred and scaled in fp64, z~ from Zc (scale_rows_kernel), the centre after the betas in dBeta
    assert "const double* centre = p.beta + kMaxTerms * p.dpad;" in pred
    assert "xv = (x - centre[dim]) * bt[dim];" in pred
    assert "if (out_centred) out_centred[idx] = in_range ? (v - centre[k]) * beta[k] : 0.0;" in misc
    assert "ctr64[j] = sd > 0.0 ? std::nearbyint(ctr[j] / sd) * sd : ctr[j];" in api
    # q: one fma chain over dpad; each term folded with fma(C_t, exp(-q), acc)
    assert "const double d0 = x.x - z0, d1 = x.y - z1;" in pred
    assert "q[pp] = fma(d0, d0, q[pp]);\n" in pred and "q[pp] = fma(d1, d1, q[pp]);\n" in pred
    assert "e[pp] = p.kf.fold_term(e[pp], t, q[pp]);" in pred
    assert "return fma(term_scale(t), exp(-q), acc); }" in internal
    # mean: an fma chain over the column tiles, a butterfly over the warp, the warps in order
    assert "macc[pp] = fma(ev, vj, macc[pp]);" in pred
    assert "for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);" in pred
    assert "const double s = ((red[grp][0][col] + red[grp][1][col]) + red[grp][2][col]) + red[grp][3][col];" in pred
    # variance: the packed B, DMMA over the blocks I <= C, the epilogue, the partials in order, selfKernel once
    assert "if (i < j) v = M[static_cast<size_t>(i) * m + j] + M[static_cast<size_t>(j) * m + i];" in pred
    assert "else if (i == j) v = M[static_cast<size_t>(i) * m + i];" in pred
    assert "mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64" in pred
    assert "const int nk = (ct + 1) * (kVarCols / kVarK);" in pred
    assert "for (int j = 0; j < 4; ++j) {\n      const double2 kv" in pred
    assert "s = fma(acc[i][j][0], kv.x, s);" in pred and "s = fma(acc[i][j][1], kv.y, s);" in pred
    assert "s += __shfl_xor_sync(0xffffffffu, s, 1);" in pred and "s += __shfl_xor_sync(0xffffffffu, s, 2);" in pred
    assert "vpart[static_cast<size_t>(ct) * rows + r0 + tid] = red[0][tid] + red[1][tid];" in pred
    assert "for (int ct = 0; ct < n_ct; ++ct) s += vpart[static_cast<size_t>(ct) * rows + r];" in pred
    assert "const double v = self_k + s;" in pred
    assert "const int n_ct = (a.m + kVarCols - 1) / kVarCols;" in pred
    assert "kf.self_kernel += term.scale;" in api
    # probability
    assert "const double sd2 = sqrt(2.0 * (v < 0.0 ? 0.0 : v));" in pred
    assert "const double z = __dadd_rn(mu, __dmul_rn(sd2, rule[i]));" in pred
    assert "acc = fma(w[i], 1.0 / (1.0 + exp(-z)), acc);" in pred
    assert "prob[r] = acc * kRsqrtPi;" in pred
    assert float(re.search(r"constexpr double kRsqrtPi = ([0-9.]+);", pred).group(1)) == RSQRT_PI
    # the tile constants the rounding counts and the sample are computed from
    assert const(pred, "kElemCols") == ELEM_COLS == const(internal, "kTile")
    assert const(pred, "kElemPts") == ELEM_PTS
    assert const(pred, "kVarCols") == VAR_COLS and const(pred, "kVarRows") == VAR_ROWS
    assert const(pred, "kVarK") * 2 == VAR_COLS                # two k chunks per 64-wide block: 64 (C + 1) products
    assert "8 warps: 4 (rows) x 2 (columns), warp tile 32 x 32" in pred    # 8 columns per lane of a quad


def test_rounding_counts():
    assert rounding_counts(1) == (1 + 8, 64 + 11 + 1 + 1)
    assert rounding_counts(128) == (1 + 8, 128 + 11 + 2 + 1)
    assert rounding_counts(129) == (2 + 8, 192 + 11 + 3 + 1)
    assert rounding_counts(4000) == (32 + 8, 4032 + 11 + 63 + 1)
    assert m_padded(255) == m_padded(256) == 256 and m_padded(257) == 384


def test_sample_points():
    pts = set(sample_points(8193, np.random.default_rng(0), windows=[(0, 8192), (8192, 1)], count=10).tolist())
    assert {0, 15, 16, 31, 32, 63, 127, 128, 255, 8191, 8192} <= pts and max(pts) == 8192


# ---- the model against the oracle ------------------------------------------------------------------------------------
def test_model_matches_oracle():
    """In fp64 the model's mean and variance are the oracle predictor's (predict_many), and its p the oracle
    integrator's on the same rule, to the oracle's rounding."""
    for m, d, terms in ((65, 5, 1), (129, 33, 2), (200, 7, 4)):
        c = make_case(m, d, terms, seed=m)
        X = points(c, 120)
        st = PredictModel(c["k0"], c["Z"], c["v"], c["M"]).predict(X)
        m0, v0 = oracle.GaussianProjectedProcessRawPredictor(c["v"], c["M"], c["k0"]).predict_many(X)
        K0 = c["k0"].cross_kernel(X)
        assert np.all(np.abs(st["mean"].astype(np.float64) - m0) <= 1e-13 * (np.abs(K0) @ np.abs(c["v"])))
        scale = c["k0"].self_kernel(None) + np.einsum("ti,ti->t", np.abs(K0) @ np.abs(c["M"]), np.abs(K0))
        assert np.all(np.abs(st["var"].astype(np.float64) - v0) <= 1e-13 * scale)
    mean = np.linspace(-700, 40, 400)
    var = np.concatenate([np.zeros(100), np.geomspace(1e-6, 1e4, 300)])
    for n in NODES:
        x, w = np.polynomial.hermite.hermgauss(n)
        p, _, _ = probability(mean, var, x, w)
        p0 = averaged_probability(mean, var, n)
        assert np.all(np.abs(p.astype(np.float64) - p0) <= 1e-13 * p0 + 1e-300)


# ---- a numpy restatement of the prediction kernels, with planted bugs --------------------------------------------------
def fma(a, b, c):
    """fma through longdouble (the fp64 product and sum rounded once, to within the double rounding of the detour)."""
    return (np.asarray(a).astype(LD) * b + c).astype(np.float64)


def exp_1ulp(x, rng):
    """CUDA's exp: numpy's exp moved by a seeded random of up to half an ulp and rounded, within 1 ulp; 0 stays 0 or
    goes to the smallest subnormal, inf stays inf."""
    with np.errstate(over="ignore"):
        v = np.exp(x)
    fin = np.isfinite(v)
    moved = (v.astype(LD) + rng.uniform(-0.5, 0.5, v.shape) * np.spacing(np.where(fin, v, 0.0))).astype(np.float64)
    return np.where(fin, np.maximum(moved, 0.0), v)


def flat_terms(kernel, d):
    """(C_t, beta_t) of the library's flattened kernel and its selfKernel, as flatten_kernel builds them."""
    out, self_k = [], 0.0
    for t in kernel.flatten():
        self_k += t["scale"]
        if t["type"] == N.SGP_TERM_EYE:
            continue
        beta = (np.asarray(t["beta"], np.float64) if t["type"] == N.SGP_TERM_ARD
                else np.full(d, 1.0 / (np.sqrt(2.0) * t["sigma"])))
        out.append((t["scale"], beta))
    return out, self_k


def emul_elements(kernel, X, Z, rng, bug=None):
    """predict_elements_kernel's K[n][m]."""
    X = np.asarray(X, dtype=np.float64)
    (n, d), m = X.shape, len(Z)
    c = np.zeros(d) if bug == "uncentred" else centre(Z)
    K = np.zeros((n, m))
    for C, beta in flat_terms(kernel, d)[0]:
        zc = (Z - c) * beta                                              # scale_rows_kernel (Zc)
        xs = (X - c) * beta
        q = np.zeros((n, m))
        for k in range(d):
            df = xs[:, k, None] - zc[None, :, k]
            q = fma(df, df, q)
        ex = exp_1ulp(-q, rng)
        if bug == "flush_q60":
            ex = np.where(q > 60, 0.0, ex)
        K = fma(C, ex, K)
    return K


def emul_mean(K, v):
    """The mean: per lane an fma chain over the column tiles, a butterfly over the 32 lanes, the 4 warps in order."""
    n, m = K.shape
    mp = m_padded(m)
    Kp, vp = np.zeros((n, mp)), np.zeros(mp)
    Kp[:, :m], vp[:m] = K, v
    acc = np.zeros((n, ELEM_COLS))
    for ct in range(mp // ELEM_COLS):
        sl = slice(ct * ELEM_COLS, (ct + 1) * ELEM_COLS)
        acc = fma(Kp[:, sl], vp[sl], acc)
    s = acc.reshape(n, ELEM_COLS // 32, 32)
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        s = s + s[:, :, lanes ^ o]
    r = s[:, :, 0]
    return ((r[:, 0] + r[:, 1]) + r[:, 2]) + r[:, 3]


def emul_var(K, M, self_k):
    """The variance: B packed in fp64, W = K B by one rounding per product, the epilogue per column tile (two column
    warps, quads of lanes with 8 columns each), the partials in order, selfKernel last."""
    n, m = K.shape
    mp, n_ct = m_padded(m), (m + VAR_COLS - 1) // VAR_COLS
    B = np.zeros((mp, mp))
    B[:m, :m] = np.triu(M + M.T, 1) + np.diag(np.diag(M))
    Kp = np.zeros((n, mp))
    Kp[:, :m] = K
    W = np.zeros((n, mp))
    for i in range(VAR_COLS * n_ct):
        W = fma(Kp[:, i, None], B[None, i, :], W)
    s = np.zeros(n)
    for C in range(n_ct):
        red = []
        for wc in (0, 1):
            q = np.zeros((n, 4))
            for j in range(4):
                for h in (0, 1):
                    cols = C * VAR_COLS + wc * 32 + j * 8 + 2 * np.arange(4) + h
                    q = fma(W[:, cols], Kp[:, cols], q)
            q = q + q[:, [1, 0, 3, 2]]
            q = q + q[:, [2, 3, 0, 1]]
            red.append(q[:, 0])
        s = s + (red[0] + red[1])
    return self_k + s


def emul_prob(mean, var, x, w, rng, bug=None):
    """predict_var_reduce_kernel<true>'s p."""
    sd2 = np.sqrt(2.0 * np.where(var < 0.0, 0.0, var))
    acc = np.zeros(len(mean))
    with np.errstate(over="ignore"):
        for i in range(len(x)):
            z = mean + sd2 * x[i]
            if bug == "complement":
                sig = 1.0 - 1.0 / (1.0 + exp_1ulp(z, rng))
            else:
                sig = 1.0 / (1.0 + exp_1ulp(-z, rng))
            acc = fma(w[i], sig, acc)
    return acc * RSQRT_PI


def run(c, X, seed=0, bug=None, var_bug=None):
    """(elements, mean, var, model statistics) of the restated kernels; var_bug: a bug in the variance's K only."""
    rng = np.random.default_rng(seed)
    K = emul_elements(c["k"], X, c["Z"], rng, bug)
    Kv = emul_elements(c["k"], X, c["Z"], np.random.default_rng(seed), var_bug) if var_bug else K
    self_k = flat_terms(c["k"], c["d"])[1]
    st = PredictModel(c["k0"], c["Z"], c["v"], c["M"]).predict(X)
    return K, emul_mean(K, c["v"]), emul_var(Kv, c["M"], self_k), st


def element_fraction(K, st):
    return bound_fraction(K, st["K"], st["a"] + st["e"])


def gate(st, mean, var, c, X):
    """The existing GPU tests' gates: errors relative to |K0||v| and selfKernel + |K0||M||K0|^T."""
    A = np.abs(st["K"].astype(np.float64))
    em = float(np.max(np.abs(mean - st["mean"].astype(np.float64)) / np.maximum(A @ np.abs(c["v"]), 1e-300)))
    scale = c["k0"].self_kernel(None) + np.einsum("ti,ti->t", A @ np.abs(c["M"]), A)
    ev = float(np.max(np.abs(var - st["var"].astype(np.float64)) / scale))
    return em, ev


def shifted(c, X, frac=0.5):
    """The case with M + a 1 1^T, a chosen so that about `frac` of the variances at X are negative."""
    K0 = c["k0"].cross_kernel(X)
    a = -np.quantile(np.einsum("ti,ti->t", K0 @ c["M"], K0) / K0.sum(1) ** 2, frac)
    return dict(c, M=c["M"] + a)


def far(c, n, seed):
    """Points 6 to 60 length scales off the active set along dimension 0: elements from ~1e-5 through the subnormals to
    0."""
    rng = np.random.default_rng(seed)
    X = points(c, n, seed)
    X[:, 0] += rng.uniform(6.0, 60.0, n) * np.sqrt(c["d"]) * 1.5
    return X


def emulation_cases():
    """(label, case, X) on host-sized shapes."""
    out = []
    for m in (63, 64, 65, 127, 128, 129):
        c = make_case(m, 5, 1 + m % 4, seed=m)
        out.append(("m=%d" % m, c, points(c, 70)))
    for d in (1, 32, 33, 784):
        c = make_case(129 if d < 784 else 65, d, 1 + d % 4, seed=d)
        X = points(c, 40 if d == 784 else 70)
        out.append(("d=%d" % d, c, X))
        out.append(("d=%d fp32 input" % d, c, X.astype(np.float32).astype(np.float64)))
    for terms in (1, 2, 3, 4):
        c = make_case(100, 7, terms, seed=10 + terms)
        out.append(("%d terms" % terms, c, points(c, 70)))
    for where in ("0", "1e3", "-1e3", "1e3_one_dim"):
        d = 4
        off = np.zeros(d)
        if where == "1e3_one_dim":
            off[0] = 1e3 * np.sqrt(d)
        else:
            off[:] = float(where) * np.sqrt(d)
        c = make_case(150, d, 2, seed=21, offset=off)
        out.append(("placement %s" % where, c, points(c, 100)))
    c = make_case(130, 3, 2, seed=5)
    out.append(("far points", c, far(c, 100, 5)))
    c = make_case(140, 6, 2, seed=50)
    X = points(c, 100)
    out.append(("variances straddling 0", shifted(c, X), X))
    c = make_case(140, 6, 2, seed=77)
    E = np.random.default_rng(5).standard_normal(c["M"].shape) * 50.0
    out.append(("asymmetric M", dict(c, M=c["M"] + (E - E.T)), points(c, 100)))
    c = make_case(1, 1, 1, seed=1)
    out.append(("m=1 d=1", c, points(c, 20)))
    return out


def test_emulated_kernels_within_bound():
    worst, worst_label = 0.0, None
    for label, c, X in emulation_cases():
        K, mean, var, st = run(c, X)
        fe, (fm, fv) = element_fraction(K, st), fractions(st, mean, var)
        share = reference_share(st)
        print("%-28s elements %.3g  mean %.3g  var %.3g of the bound (reference %.1e of it)" % (label, fe, fm, fv, share))
        assert max(fe, fm, fv) <= 1.0, label
        assert share < 0.125, label
        if label == "far points":
            assert (K == 0).any() and ((K > 0) & (K < 2.3e-308)).any()    # zeros and subnormals both
        if label == "variances straddling 0":
            assert (var < 0).sum() > 20 and (var > 0).sum() > 20
        if max(fe, fm, fv) > worst:
            worst, worst_label = max(fe, fm, fv), label
    print("clean emulation: largest fraction of the bound %.3g (%s)" % (worst, worst_label))


def tail_inputs(rng, n=600):
    """Means from -740 to +40 and variances from 0 (and below) to 1e4."""
    mean = np.concatenate([np.linspace(-740.0, 40.0, n - 60), rng.uniform(-40, 40, 60)])
    var = np.concatenate([np.zeros(n // 4), -rng.random(n // 8), np.geomspace(1e-8, 1e4, n - n // 4 - n // 8)])
    return mean, rng.permutation(var)


@pytest.mark.parametrize("nodes", NODES)
def test_emulated_probability_within_bound(nodes):
    from spark_gp_b200.engine import ProjectedProcessEngine
    x, w = ProjectedProcessEngine.gauss_hermite_rule(nodes)
    rng = np.random.default_rng(nodes)
    mean, var = tail_inputs(rng)
    prob = probability(mean, var, x, w)
    worst = 0.0
    for seed in range(3):
        p = emul_prob(mean, var, x, w, np.random.default_rng(seed))
        worst = max(worst, probability_fraction(p, prob))
    share = float(np.max(prob[2] / prob[1]))
    print("%3d nodes: p %.3g of the bound (reference %.1e of it), p from %.1e" % (nodes, worst, share,
                                                                                  float(prob[0].min())))
    assert worst <= 1.0 and share < 0.125
    assert float(prob[0].min()) < 1e-300                     # the tails reach fp64's subnormal range


# ---- planted bugs -----------------------------------------------------------------------------------------------------
def placement_case(scale):
    d = 4
    off = np.full(d, scale * np.sqrt(d))
    c = make_case(150, d, 2, seed=21, offset=off)
    return c, points(c, 300)


def cluster_case():
    """Points in two clusters 10 length scales apart, the active set drawn from both: every point has near elements and
    far ones near exp(-100)."""
    rng = np.random.default_rng(3)
    c = make_case(128, 3, 1, seed=3)
    Z = rng.random((128, 3)) * 2.0
    Z[64:, 0] += 10.0 / c["k"].flatten()[0]["beta"][0]
    c = dict(c, Z=Z, k0=c["k0"].set_training_vectors(Z))
    X = Z[rng.integers(0, 128, 200)] + rng.standard_normal((200, 3)) * 0.3
    return c, X


@pytest.mark.parametrize("bug", ["uncentred", "flush_q60"])
def test_planted_element_bug(bug):
    c, X = placement_case(1e3) if bug == "uncentred" else cluster_case()
    K, mean, var, st = run(c, X, bug=bug)
    em, ev = gate(st, mean, var, c, X)
    fe, (fm, fv) = element_fraction(K, st), fractions(st, mean, var)
    K1, mean1, var1, _ = run(c, X)
    clean = (element_fraction(K1, st),) + fractions(st, mean1, var1)
    print("%-10s gate: mean %.1e var %.1e (gate %.0e); bound: elements %.3g mean %.3g var %.3g; as written: %.3g %.3g "
          "%.3g" % (bug, em, ev, TOL, fe, fm, fv, *clean))
    assert em < TOL and ev < TOL                  # the existing gate cannot see it ...
    assert fe > 1.0                               # ... the element bound can
    if bug == "uncentred":
        assert fm > 1.0                           # and the mean's
    assert max(clean) <= 1.0                      # and the same case as written passes


def test_planted_complement_sigmoid():
    """1 - 1/(1 + exp(z)) is sigmoid(z) in exact arithmetic, and loses every bit of p in the left tail."""
    from spark_gp_b200.engine import ProjectedProcessEngine
    x, w = ProjectedProcessEngine.gauss_hermite_rule(100)
    mean = np.linspace(-40.0, -25.0, 200)
    var = np.full(200, 1e-4)
    prob = probability(mean, var, x, w)
    p = emul_prob(mean, var, x, w, np.random.default_rng(0), bug="complement")
    p1 = emul_prob(mean, var, x, w, np.random.default_rng(0))
    err = float(np.max(np.abs(p - prob[0].astype(np.float64))))
    f, f1 = probability_fraction(p, prob), probability_fraction(p1, prob)
    print("complement sigmoid: gate %.1e (gate %.0e); bound %.3g; as written %.3g" % (err, TOL_P, f, f1))
    assert err < TOL_P and f > 1.0 and f1 <= 1.0


def test_variance_only_bug():
    """The variance's K staged without the centre at 1e4 length scales, the mean's K as written: the variance passes the
    1e-11 gate and breaks its bound; the mean is untouched."""
    c, X = placement_case(1e4)
    K, mean, var, st = run(c, X, var_bug="uncentred")
    em, ev = gate(st, mean, var, c, X)
    fm, fv = fractions(st, mean, var)
    _, mean1, var1, _ = run(c, X)
    print("variance-only uncentred 1e4: gate var %.1e (gate %.0e); bound: mean %.3g var %.3g; as written: var %.3g" % (
        ev, TOL, fm, fv, fractions(st, mean1, var1)[1]))
    assert ev < TOL and fv > 1.0 and fm <= 1.0
    assert fractions(st, mean1, var1)[1] <= 1.0
