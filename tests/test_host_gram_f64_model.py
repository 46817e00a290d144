"""CPU tests of the extended-precision model of the fp64 DMMA statistics kernel (oracle/gram_f64_model.py) that
tests/test_gpu_gram_f64_bounds.py judges every G and b element by.  The model agrees with the oracle, the arithmetic it
transcribes is read from the kernel source, and its per-element bound is sharp: a numpy restatement of each of the
kernel's four loops stays inside it on every case, and each planted bug below passes the normwise gate of the existing
GPU tests (max |G - G0| / max |G0| < 1e-6 in SGP_PREC_F64, < 1e-11 strict) but breaks the bound."""
import os
import re

import numpy as np
import pytest

import oracle
import spark_gp_b200 as sg
from oracle.gram_f64_model import (FLT_MIN, LD, SQRT_LOG2E, GramF64Model, centre, fractions, reference_share,
                                   sample_rows)
from spark_gp_b200 import _native as N
from test_host_logic import H100_SXM_SMS, f64_slices, host_chunks

CSRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "spark_gp_b200", "csrc")
TOL_STATS, TOL_STRICT = 1e-6, 1e-11
f32 = np.float32


def rounding_budget(launches, m, num_sms):
    """(R, R_b) of one begin..finish window whose fp64-kernel launches cover `launches` points each: the points of the
    fullest slice of any launch (one DMMA or fma rounding each), the most slices of any launch (gram_reduce_kernel adds
    them in order) and one G += / b += per launch."""
    pts = max(16 * max(f64_slices(m, n, num_sms)) for n in launches)
    slices = max(len(f64_slices(m, n, num_sms)) for n in launches)
    R = pts + slices + len(launches)
    return R, R


def rel(a, b):
    b = np.asarray(b, dtype=np.float64)
    return float(np.abs(np.asarray(a) - b).max() / max(np.abs(b).max(), 1e-300))


# ---- the arithmetic the model transcribes, read from the source -----------------------------------------------------
def test_mirrors_match_source():
    gram = open(os.path.join(CSRC, "gram_f64.cu")).read()
    api = open(os.path.join(CSRC, "api.cu")).read()
    misc = open(os.path.join(CSRC, "misc_kernels.cu")).read()
    internal = open(os.path.join(CSRC, "sgp_internal.h")).read()
    # staging: x~ in the pipelined loop (fetch_x) and the generic loops (load_x_chunk), z~ from Zc (load_z_chunk)
    assert "return static_cast<float>((v - ck) * bk * ElemOps<ET>::kPrescale);" in gram
    assert "const double sk = k_in ? p.beta[term * p.dpad + c0 + k] * ElemOps<ET>::kPrescale : 0.0;" in gram
    assert "v = (v - ck) * sk;" in gram and "xs[pp * DC + k] = static_cast<ET>(v);" in gram
    assert "static_cast<ET>(kZSign * ElemOps<ET>::kPrescale * src[k])" in gram
    assert "constexpr double kZSign = kPacked ? -1.0 : 1.0;" in gram
    assert "if (out_centred) out_centred[idx] = in_range ? (v - centre[k]) * beta[k] : 0.0;" in misc
    assert float.fromhex(re.search(r"constexpr double kSqrtLog2e = (0x[0-9a-f.p+]+);", internal).group(1)) == SQRT_LOG2E
    assert "static constexpr double kPrescale = kSqrtLog2e;" in gram and "static constexpr double kPrescale = 1.0;" in gram
    # the centre (stats_scales)
    assert "ctr64[j] = sd > 0.0 ? std::nearbyint(ctr[j] / sd) * sd : ctr[j];" in api
    assert "for (int j = 0; j < d; ++j) bt[j] = 1.0 / (std::sqrt(2.0) * term.sigma);" in api
    # the float2 lanes: dims 4k, 4k+2 in .x and 4k+1, 4k+3 in .y, one fma each, then one add
    assert gram.count("const float2 d01 = fadd2(make_float2(x.x, x.y), z01), d23 = fadd2(make_float2(x.z, x.w), z23);") == 2
    assert gram.count("q[pp] = ffma2(d01, d01, q[pp]);\n") == 2 and gram.count("q[pp] = ffma2(d23, d23, q[pp]);\n") == 2
    assert "if constexpr (kPacked) qq = q[pp].x + q[pp].y; else qq = q[pp];" in gram
    assert "ElemOps<ET>::ex(q[pp].x + q[pp].y)" in gram
    # strict: one fp64 fma chain, CUDA's exp
    assert "const ET df = x4[c] - z4[c];" in gram and "q[pp] = fma(df, df, q[pp]);" in gram
    assert "static __device__ __forceinline__ double ex(double q) { return exp(-q); }" in gram
    # the exponential of the fp32 loops
    assert 'asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(-q));' in gram
    # the term scale in fp64 after the exponential, the terms added in fp64
    assert "const double sc = p.scale[0];" in gram and "const double sc = p.scale[term];" in gram
    assert "static_cast<double>(ElemOps<ET>::ex(q[pp].x + q[pp].y)) * sc" in gram
    assert "static_cast<double>(ElemOps<ET>::ex(qq)) * sc" in gram
    assert "static_cast<float>(p.scale" not in gram and "static_cast<ET>(p.scale" not in gram
    assert "dst[pp * PS] = (term == 0) ? v : dst[pp * PS] + v;" in gram
    # accumulation: fp64 DMMA, b by an fp64 fma chain, slices added in order, one G += per launch
    assert "mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64" in gram
    assert gram.count("bacc = fma(p") == 2
    assert "for (int s = 0; s < n_slices; ++s) v += Gpart[s * stride + static_cast<size_t>(i) * m_pad + j];" in gram
    assert "G[static_cast<size_t>(i) * m + j] += v;" in gram and "b[j] += v;" in gram


def test_centre_and_rows():
    Z = np.array([[1.0, 5.0], [3.0, 5.0], [2.0, 5.0]])
    c = centre(Z)
    sd = np.sqrt(2.0 / 3.0)
    assert c[0] == np.rint(2.0 / sd) * sd and c[1] == 5.0
    rows = sample_rows(300, np.random.default_rng(0))
    assert {0, 63, 64, 127, 128, 191, 192, 255, 256, 299} <= set(rows.tolist()) and rows.max() < 300


# ---- kernels and data ------------------------------------------------------------------------------------------------
def kernel_of(n_terms, d, scales=(1.3, 0.4, 2.0, 0.7), width=1.0, seed=0):
    """(library kernel, oracle kernel): n_terms non-Eye terms alternating ARD and RBF, plus an Eye term."""
    rng = np.random.default_rng(seed)
    specs = [("ard", scales[t], rng.uniform(0.3, 1.5, d) * width / np.sqrt(d)) if t % 2 == 0 else
             ("rbf", scales[t], np.sqrt(d) * rng.uniform(0.7, 1.4) / width) for t in range(n_terms)]

    def make(S):
        body = None
        for kind, C, p in specs:
            term = C * (S.ARDRBFKernel(p) if kind == "ard" else S.RBFKernel(p))
            body = term if body is None else body + term
        return body + S.const(1e-2) * S.EyeKernel()
    return make(sg), make(oracle)


def test_model_matches_oracle():
    """In fp64 the model's K, G and b are the oracle's (get_matrix_kmn_knm_and_vector_kmny) to the oracle's rounding."""
    for terms, d in ((1, 5), (2, 33), (4, 3)):
        rng = np.random.default_rng(terms)
        X, Z = rng.standard_normal((300, d)), rng.standard_normal((40, d))
        Z[:10] = X[:10]
        y = rng.standard_normal(300)
        _, ok = kernel_of(terms, d, seed=terms)
        st = GramF64Model(ok, Z, strict=True).statistics(X, y, R=1, R_b=1)
        K0 = ok.set_training_vectors(X).cross_kernel(Z).T
        G0, b0 = oracle.get_matrix_kmn_knm_and_vector_kmny([(y, ok.set_training_vectors(X))], Z)
        assert np.all(np.abs(st["K"].astype(np.float64) - K0) <= 1e-12 * K0)
        assert np.all(np.abs(st["G"].astype(np.float64) - G0) <= 1e-12 * (K0.T @ K0))
        assert np.all(np.abs(st["b"].astype(np.float64) - b0) <= 1e-12 * (K0.T @ np.abs(y)))


# ---- a numpy restatement of the four loops of kmn_gram_f64_kernel, with planted bugs -----------------------------------
BUGS = ["uncentred", "flush_q60", "strict_flush_fp32_floor", "strict_b_fp32_tile", "fp32_term_scale"]


def flat_terms(kernel, d):
    """(C_t, beta_t) of the library's flattened kernel, as flatten_kernel builds them."""
    out = []
    for t in kernel.flatten():
        if t["type"] == N.SGP_TERM_EYE:
            continue
        beta = (np.asarray(t["beta"], np.float64) if t["type"] == N.SGP_TERM_ARD
                else np.full(d, 1.0 / (np.sqrt(2.0) * t["sigma"])))
        out.append((t["scale"], beta))
    return out


def fma32(a, b, c):
    """fmaf through float64: the fp32 product is exact in float64."""
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(f32)


def ex2_ftz(qq, rng):
    """ex2.approx.ftz.f32(-qq): the exact power, moved by a seeded random up to 1.5 ulp and rounded to fp32 (within 2
    ulp), results below 2^-126 flushed to 0."""
    v = np.exp2(-qq.astype(np.float64))
    ulp = np.spacing(v.astype(f32)).astype(np.float64)
    ex = (v + rng.uniform(-1.5, 1.5, v.shape) * ulp).astype(f32)
    return np.where((v < float(FLT_MIN)) | (ex < np.float32(FLT_MIN)), f32(0), ex)


def panel(kernel, X, Z, variant, rng, bug=None):
    """The kernel elements K[n][m] (fp64) as the loop `variant` computes them into its panels."""
    X = np.asarray(X, dtype=np.float64)
    (n, d), m = X.shape, len(Z)
    c = np.zeros(d) if bug == "uncentred" else centre(Z)
    K = np.zeros((n, m))
    for t, (C, beta) in enumerate(flat_terms(kernel, d)):
        zc = (Z - c) * beta                                               # scale_rows_kernel (Zc)
        if variant in ("pipelined", "generic"):
            if variant == "pipelined":
                xs = (((X - c) * beta) * SQRT_LOG2E).astype(f32)          # fetch_x
            else:
                xs = ((X - c) * (beta * SQRT_LOG2E)).astype(f32)          # load_x_chunk
            zs = ((-SQRT_LOG2E) * zc).astype(f32)                         # load_z_chunk, negated
            lanes = [np.zeros((n, m), f32), np.zeros((n, m), f32)]
            for k in range(d):
                dk = (xs[:, k, None] + zs[None, :, k]).astype(f32)
                lanes[k % 2] = fma32(dk, dk, lanes[k % 2])
            qq = (lanes[0] + lanes[1]).astype(f32)
            ex = ex2_ftz(qq, rng)
            if bug == "flush_q60":
                ex = np.where(qq > 60, f32(0), ex)
            v = (f32(C) * ex).astype(np.float64) if bug == "fp32_term_scale" else ex.astype(np.float64) * C
        else:
            xs = (X - c) * beta
            q = np.zeros((n, m))
            for k in range(d):                                            # one fma chain over dpad (resident or chunked)
                df = xs[:, k, None] - zc[None, :, k]
                q = (df.astype(LD) * df + q).astype(np.float64)
            ex = np.exp(-q)
            if bug == "strict_flush_fp32_floor":
                ex = np.where(ex < float(FLT_MIN), 0.0, ex)
            v = ex * C
        K = v if t == 0 else K + v
    return K


def accumulate(P, y, launches, num_sms, bug=None):
    """G, b of the panels P[n][m] over launches of the given point counts: per slice (f64_slices) one DMMA step of four
    points at a time into fp64 accumulators and an fp64 fma chain for b; slices added in order, G += per launch; the
    lower triangle mirrored."""
    n, m = P.shape
    G, b = np.zeros((m, m)), np.zeros(m)
    p0 = 0
    for cn in launches:
        Gl, bl = np.zeros((m, m)), np.zeros(m)
        off = p0
        for blocks in f64_slices(m, cn, num_sms):
            acc, bacc = np.zeros((m, m)), np.zeros(m)
            b32 = np.zeros(min(m, 256) - 128, f32) if m > 128 else None      # row tile 1 of the b bug
            for s0 in range(off, min(off + 16 * blocks, p0 + cn), 4):
                Pk = P[s0:min(s0 + 4, p0 + cn)]
                acc = acc + Pk.T @ Pk
                for p in range(s0, s0 + len(Pk)):
                    bacc = (P[p].astype(LD) * y[p] + bacc).astype(np.float64)
                    if bug == "strict_b_fp32_tile" and b32 is not None:
                        b32 = (P[p, 128:256].astype(f32).astype(np.float64) * f32(y[p]) + b32).astype(f32)
            if bug == "strict_b_fp32_tile" and b32 is not None:
                bacc[128:256] = b32
            Gl, bl = Gl + acc, bl + bacc
            off += 16 * blocks
        G, b = G + Gl, b + bl
        p0 += cn
    L = np.tril(G)
    return L + np.tril(L, -1).T, b


def far_clusters(d, n, m, q_far, rng):
    """Points in two clusters whose scaled squared distance is about q_far (natural units) under a unit ARD kernel, with
    the active set drawn from both: whole blocks of G sit near exp(-q_far)."""
    X = rng.standard_normal((n, d)) * 0.3
    X[n // 2:, 0] += np.sqrt(q_far)
    Z = X[rng.permutation(n)[:m]].copy()
    return X, Z


def unit_ard(d, C=1.0):
    beta = np.ones(d)
    return C * sg.ARDRBFKernel(beta) + sg.const(1e-2) * sg.EyeKernel(), C * oracle.ARDRBFKernel(beta) + oracle.const(
        1e-2) * oracle.EyeKernel()


def emulation_cases():
    """(label, variant, library kernel, oracle kernel, X, y, Z, launches) on host-sized shapes."""
    out = []
    for variant in ("pipelined", "generic", "resident", "chunked"):
        single = variant in ("pipelined", "resident")
        for i, terms in enumerate([1] if single else [2, 3, 4, 1]):
            d = 5 if single else (33, 7, 3, 36)[i]
            rng = np.random.default_rng(10 * i + len(variant))
            n, m = 700, 70
            X, Z = rng.standard_normal((n, d)), rng.standard_normal((m, d))
            Z[:20] = X[:20]                                                # coinciding points: k = 1 exactly
            k, ok = kernel_of(terms, d, seed=i)
            out.append(("%s %d terms d=%d" % (variant, terms, d), variant, k, ok, X, rng.standard_normal(n), Z, [n]))
        rng = np.random.default_rng(7)
        X, Z = far_clusters(4, 600, 40, 86.0 if single else 80.0, rng)    # far pairs near the fp32 floor (2^-126)
        k, ok = unit_ard(4)
        if not single:
            k, ok = (0.5 * sg.ARDRBFKernel(np.ones(4)) + 0.7 * sg.RBFKernel(1.0 / np.sqrt(2.0)),
                     0.5 * oracle.ARDRBFKernel(np.ones(4)) + 0.7 * oracle.RBFKernel(1.0 / np.sqrt(2.0)))
        out.append(("%s far pairs" % variant, variant, k, ok, X, rng.standard_normal(600), Z, [600]))
        rng = np.random.default_rng(8)
        X = rng.random((500, 5)) * 3.0 + 1e3                               # 1e3 length scales out
        Z = X[rng.permutation(500)[:50]].copy()
        k, ok = unit_ard(5)
        out.append(("%s placement 1e3, two launches" % variant, variant, k, ok, X, np.sin(X.sum(1)), Z, [300, 200]))
    return out


def run_case(variant, k, ok, X, y, Z, launches, bug=None, seed=0):
    P = panel(k, X, Z, variant, np.random.default_rng(seed), bug)
    G, b = accumulate(P, y, launches, H100_SXM_SMS, bug)
    R, R_b = rounding_budget(launches, len(Z), H100_SXM_SMS)
    st = GramF64Model(ok, Z, strict=variant in ("resident", "chunked")).statistics(X, y, R, R_b)
    return G, b, st


def test_emulated_loops_within_bound():
    worst, worst_label = 0.0, None
    for label, variant, k, ok, X, y, Z, launches in emulation_cases():
        G, b, st = run_case(variant, k, ok, X, y, Z, launches)
        fg, fb = fractions(G, b, st)
        share = reference_share(st)
        print("%-40s G %.3g  b %.3g  of the bound (reference %.1e of it)" % (label, fg, fb, share))
        assert np.array_equal(G, G.T)
        assert fg <= 1.0 and fb <= 1.0, label
        assert share < 0.125, label
        if max(fg, fb) > worst:
            worst, worst_label = max(fg, fb), label
    print("clean emulation: largest fraction of the bound %.3g (%s)" % (worst, worst_label))


def bug_case(bug):
    """(variant, library kernel, oracle kernel, X, y, Z, launches) on which the planted bug passes the normwise gate."""
    rng = np.random.default_rng(3)
    if bug == "uncentred":                       # 20 length scales out: each staged coordinate off by up to 2^-24 20
        X = rng.standard_normal((800, 4)) * 3.0 + 20.0
        Z = X[rng.permutation(800)[:60]].copy()
        k, ok = unit_ard(4)
        return "pipelined", k, ok, X, 1.0 + 0.1 * rng.standard_normal(800), Z, [800]
    if bug == "flush_q60":                       # the far block sits near exp(-50) = 2^-72
        X, Z = far_clusters(4, 800, 60, 50.0, rng)
        k, ok = unit_ard(4)
        return "pipelined", k, ok, X, rng.standard_normal(800), Z, [800]
    if bug == "strict_flush_fp32_floor":         # the far block sits near exp(-120), below fp32's range
        X, Z = far_clusters(4, 800, 60, 120.0, rng)
        k, ok = unit_ard(4)
        return "resident", k, ok, X, rng.standard_normal(800), Z, [800]
    if bug == "strict_b_fp32_tile":              # the second row tile of the active set is 6 length scales off the data
        X = rng.standard_normal((1200, 3)) * 0.5
        Z = np.vstack([X[:128], rng.standard_normal((72, 3)) * 0.5 + [6.0, 0.0, 0.0]])
        k, ok = unit_ard(3)
        return "resident", k, ok, X, rng.standard_normal(1200), Z, [1200]
    if bug == "fp32_term_scale":                 # C = 1e-30: products below 2^-126 C lose bits as fp32 subnormals
        X, Z = far_clusters(4, 800, 60, 30.0, rng)
        k, ok = unit_ard(4, C=1e-30)
        return "pipelined", k, ok, X, rng.standard_normal(800), Z, [800]
    raise ValueError(bug)


@pytest.mark.parametrize("bug", BUGS)
def test_planted_bug_passes_normwise_gate_and_breaks_bound(bug):
    variant, k, ok, X, y, Z, launches = bug_case(bug)
    G, b, st = run_case(variant, k, ok, X, y, Z, launches, bug=bug)
    tol = TOL_STRICT if variant in ("resident", "chunked") else TOL_STATS
    eg, eb = rel(G, st["G"].astype(np.float64)), rel(b, st["b"].astype(np.float64))
    fg, fb = fractions(G, b, st)
    G1, b1, _ = run_case(variant, k, ok, X, y, Z, launches)
    print("%-24s normwise dG %.1e db %.1e (gate %.0e); bound: G %.3g b %.3g; as written: G %.3g b %.3g" % (
        bug, eg, eb, tol, fg, fb, *fractions(G1, b1, st)))
    assert eg < tol and eb < tol                  # the existing gate cannot see it ...
    assert max(fg, fb) > 1.0                      # ... the bound can
    assert max(fractions(G1, b1, st)) <= 1.0      # and the same case as written passes


def test_fp32_term_scale_at_fp32_range_ends():
    """The term scale applied in fp32 (as the loops did before) at C = 1e-40 is an fp32 subnormal with 17 bits: every
    element is ~5e-6 off, which even the normwise gate sees; at C = 1e39 it overflows to inf.  In fp64 both are inside
    the bound."""
    rng = np.random.default_rng(4)
    X = rng.standard_normal((300, 3))
    Z = X[:30].copy()
    for C in (1e-40, 1e39):
        k, ok = unit_ard(3, C=C)
        G, b, st = run_case("pipelined", k, ok, X, rng.standard_normal(300), Z, [300])
        assert max(fractions(G, b, st)) <= 1.0
        with np.errstate(over="ignore", invalid="ignore"):
            Gb, bb, _ = run_case("pipelined", k, ok, X, rng.standard_normal(300), Z, [300], bug="fp32_term_scale")
        if C > 1.0:
            assert not np.all(np.isfinite(Gb))
        else:
            assert rel(Gb, st["G"].astype(np.float64)) > TOL_STATS


def test_rounding_budget_counts_launches():
    """R of the host entry over several chunks, and of several accumulate calls in one window."""
    chunks = host_chunks(100000, 64, True)
    assert len(chunks) == 2
    R, _ = rounding_budget(chunks, 64, H100_SXM_SMS)
    assert R == 16 * max(max(f64_slices(64, n, H100_SXM_SMS)) for n in chunks) + H100_SXM_SMS + 2
    assert rounding_budget([1], 2100, H100_SXM_SMS) == (16 + 1 + 1,) * 2
