"""Error model of the SIMT E-step (`estep_simt_kernel<D>`, csrc/kernels_simt.cuh), on the CPU: numpy only (the parameter
sets come from the project's builders and the CPU oracle).

The emulator restates the kernel's logits bit for bit:
  * the operand of build_epack (csrc/host_math.cpp): the means, the combined coefficients fl32(Rinv_ij + Rinv_ji) for
    i < j and Rinv_ii on the diagonal, and fl32(constant + logf(pi)) with glibc's logf (through ctypes: numpy's float32
    log may differ from it by an ulp);
  * dx = fl32(x - mu), the fmaf chains of the triangle in the kernel's order (t = fmaf(p, dx_j, t) over j >= i, then
    q = fmaf(dx_i, t, q)) and l = fmaf(-0.5, q, c).  fma32() rounds a float32 fma exactly: the product is exact in float64,
    TwoSum gives s = fl64(a b + c) with its exact error e, and fl32(s) is the answer except on a float32 midpoint, where
    the sign of e decides.
Everything after the logits is measured against gamma = exp(l - LSE(l)) and LSE(l) in float64 of the emulated logits.

The bar covers what is not emulated.  cuobjdump -sass of the kernel shows the logit operations as written and the online
update contracted to one FFMA, run_sum = fma(run_sum, expf(run_max - m2), expf(l - m2)), with run_max starting at
-FLT_MAX (a component with pi = 0 has the logit -inf and adds expf(-inf) = 0).  The error of run_sum is carried
through the K steps in the kernel's order (simt_bar), to first order in each step:
  * each expf: at most 2 ulp (2^-22 relative; the CUDA Math API, the build has no -use_fast_math), after the rounding of
    its argument (u |a|, u = 2^-24), and 2^-148 absolute for results in the subnormal range (no FTZ in this build);
  * the FFMA: u of the new running sum.
With eps = |run_sum - S| / S at the end, the log-density is held to
    |denom - LSE| <= dL (1 + 2^-23) + 2^-23 |ln S| + u (|LSE| + 2 dL),   dL = -ln(1 - eps)
(logf: at most 1 ulp; the FADD run_max + logf(run_sum)), and every responsibility to
    |gamma_gpu - gamma| <= gamma ((1 + 2^-22) e^r - 1) + 2^-146,   r = lbar + u (|l - LSE| + lbar)
(the FADD l - denom, then expf; the absolute term covers subnormal results and the 0 below about -103.9).

The module asserts, on the shapes of tests/test_gpu_simt.py:
  1. a faithful FP32 emulation (expf / logf as float32 roundings of float64 values, the online log-sum-exp with the FFMA
     in the kernel's order, the FADDs and the second sweep) stays within FAITHFUL_MAX = 0.9 of the bar.  It cannot stay
     below a quarter: the bar is rigorous, and the faithful run carries the same IEEE roundings the kernel does.  The FADD
     denom = run_max + logf(run_sum) alone is off by up to half an ulp of denom, u |denom|, which is more than half of
     the log-density bar; the FADD l - denom is the same for the responsibilities of far clusters.  Measured over the
     shapes: 0.80 on responsibilities and 0.83 on log-densities;
  2. each of these kernel faults exceeds the bar at one shape at least: the off-diagonal coefficient not combined
     (Rinv_ij only), the last partial 16-cluster chunk iterating over all 16 staged records (stale records of the previous
     chunk in the denominator), the online rescale factor dropped, ln pi dropped from the constant, the second sweep
     using run_max instead of denom, and coordinate 0 read from the next SoA row;
  3. the emulated logits agree with a float64 evaluation of -1/2 (x - mu)^T Rinv (x - mu) + constant + ln pi within the
     a-priori bound of the FP32 triangle, so the emulator computes the same mathematics.
  4. with components at pi = 0 (the first, the last, a whole 16-cluster chunk, the first chunk) the faithful emulation gives
     them a responsibility of exactly 0, and the others and the log-densities stay within FAITHFUL_MAX of the bar.
Run it as a script (python tests/test_simt_error_model.py) for the table of worst error / bar per shape.
"""
import ctypes
import os
import sys
from fractions import Fraction

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from conftest import entry, fitted_params, random_spd_params  # noqa: E402

U = 2.0 ** -24
EXP_REL = 2.0 ** -22          # expf: 2 ulp
LOG_ULP = 2.0 ** -23          # logf: 1 ulp
EXP_SUB = 2.0 ** -148         # expf: 2 ulp of a subnormal result
FLOOR = 2.0 ** -146           # absolute part of the responsibility bar
CHUNK = 16                    # kEstepClusterChunk
FLT_MAX = float(np.finfo(np.float32).max)
FAITHFUL_MAX = 0.9            # the faithful FP32 emulation's share of the bar (module docstring, item 1)
FAULTS = ("uncombined", "stale_chunk", "no_rescale", "no_ln_pi", "sweep_run_max", "next_row")

_libm = ctypes.CDLL("libm.so.6")
_libm.logf.restype = ctypes.c_float
_libm.logf.argtypes = [ctypes.c_float]


def logf_c(a):
    """glibc's logf, element by element (the host's build_epack calls it)."""
    return np.array([_libm.logf(float(v)) for v in np.ravel(a)], np.float32).reshape(np.shape(a))


def f32(a):
    return np.asarray(a, np.float64).astype(np.float32).astype(np.float64)


def fma32(a, b, c):
    """fmaf of float32 values (held in float64 arrays), correctly rounded to float32, as float64."""
    a, b, c = np.broadcast_arrays(*(np.asarray(t, np.float64) for t in (a, b, c)))
    p = a * b                                   # exact: 24 + 24 significant bits
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)               # TwoSum: s + e == p + c exactly
    r = f32(s)
    d = np.abs(s - r)                           # exact (Sterbenz)
    ulp = np.spacing(np.abs(r).astype(np.float32)).astype(np.float64)
    cand = ((2 * d == ulp) | (4 * d == ulp)) & (e != 0)
    if cand.any():                              # s on a float32 midpoint: the sign of e decides
        rc, sc, ec = r[cand], s[cand], e[cand]
        nb = np.nextafter(rc.astype(np.float32), np.where(sc > rc, np.float32(np.inf), np.float32(-np.inf))).astype(np.float64)
        mid = (rc + nb) * 0.5 == sc
        fix = np.where(ec > 0, np.maximum(rc, nb), np.minimum(rc, nb))
        r = r.copy()
        r[cand] = np.where(mid, fix, rc)
    return r


# ---- the operand (build_epack) and the logits ----------------------------------------------------------------------------
def epack(cl, K, combine=True, ln_pi=True):
    """(means [K][D], coefficients [NCOEF][K] in the kernel's order, c [K]) as float64 values of the kernel's floats."""
    D = cl.means.shape[1]
    Ri = np.asarray(cl.Rinv[:K], np.float32)
    coef = []
    for i in range(D):
        for j in range(i, D):
            coef.append(Ri[:, i, i] if i == j else (Ri[:, i, j] + Ri[:, j, i] if combine else Ri[:, i, j]))
    const = np.asarray(cl.constant[:K], np.float32)
    c = const + logf_c(np.asarray(cl.pi[:K], np.float32)) if ln_pi else const
    return (np.asarray(cl.means[:K], np.float32).astype(np.float64), np.array(coef, np.float32).astype(np.float64),
            np.asarray(c, np.float32).astype(np.float64))


def logits(x, ep, block=1 << 22):
    """The kernel's float32 logits [n][K] (float64 values) of events x [n][D] under the operand ep."""
    mu, coef, c = ep
    x = np.asarray(x, np.float32)
    n, D = x.shape
    K = mu.shape[0]
    out = np.empty((n, K))
    step = max(1, block // max(1, K * D))
    for e0 in range(0, n, step):
        xs = x[e0:e0 + step]
        dx = (xs[:, None, :] - mu.astype(np.float32)[None]).astype(np.float64)        # fl32(x - mu)
        q = np.zeros(dx.shape[:2])
        idx = 0
        for i in range(D):
            t = np.zeros(dx.shape[:2])
            for j in range(i, D):
                t = fma32(coef[idx][None], dx[:, :, j], t)
                idx += 1
            q = fma32(dx[:, :, i], t, q)
        out[e0:e0 + step] = fma32(-0.5, q, c[None])
    return out


def lse64(l):
    M = l.max(1)
    S = np.exp(l - M[:, None]).sum(1)
    return M + np.log(S)


# ---- the bar ---------------------------------------------------------------------------------------------------------------
def simt_bar(l):
    """gamma, LSE (float64 of the emulated logits [n][K]) and the per-(event, cluster) / per-event bars."""
    n, K = l.shape
    Mx = np.full(n, -FLT_MAX)                    # the kernel's start: a -inf logit (pi = 0) ahead of every finite one adds 0
    Sx = np.zeros(n)
    B = np.zeros(n)

    def rel(a):                                  # relative error of expf(fl32(a)) against exp(a)
        # expf(-inf) and expf(-FLT_MAX - l) (the start of the running maximum, a < -FLT_MAX / 2 for any logit l of the
        # kernel's range) are exactly 0 and carry no error
        fa = np.isfinite(a) & (a > -0.5 * FLT_MAX)
        return np.where(fa, EXP_REL + np.expm1(U * np.abs(np.where(fa, a, 0.0))) * (1 + EXP_REL), 0.0)

    for k in range(K):
        lk = l[:, k]
        m2 = np.maximum(Mx, lk)
        a1, a2 = Mx - m2, lk - m2
        E1, E2 = np.exp(a1), np.exp(a2)
        S1 = Sx * E1 + E2
        Bp = (np.where(E1 > 0, (B * (1 + rel(a1)) + Sx * rel(a1)) * E1, 0.0) + np.where(E2 > 0, E2 * rel(a2), 0.0)
              + 2 * EXP_SUB)                     # (a factor that underflows to 0 carries no error)
        B = Bp * (1 + U) + U * S1
        Sx, Mx = S1, m2
    eps = B / Sx
    lnS = np.log(Sx)
    lse = Mx + lnS
    dL = -np.log1p(-eps)
    lbar = dL * (1 + LOG_ULP) + LOG_ULP * np.abs(lnS) + U * (np.abs(lse) + 2 * dL)
    a = l - lse[:, None]
    gamma = np.exp(a)
    r = np.minimum(lbar[:, None] + U * (np.abs(a) + lbar[:, None]), 700.0)
    gbar = gamma * ((1 + EXP_REL) * np.exp(r) - 1) + FLOOR
    return gamma, lse, gbar, lbar


def faithful(l):
    """The kernel's FP32 sequence after the logits, expf / logf as float32 roundings of float64: (gamma, denom)."""
    n, K = l.shape
    l32 = l.astype(np.float32)
    run_max = np.full(n, -FLT_MAX, np.float32)
    run_sum = np.zeros(n)
    for k in range(K):
        m2 = np.maximum(run_max, l32[:, k])
        E1 = f32(np.exp((run_max - m2).astype(np.float64)))
        E2 = f32(np.exp((l32[:, k] - m2).astype(np.float64)))
        run_sum = fma32(run_sum, E1, E2)
        run_max = m2
    denom = run_max + f32(np.log(run_sum)).astype(np.float32)
    g = f32(np.exp((l32 - denom[:, None]).astype(np.float64)))
    return g, denom.astype(np.float64)


def fault_gamma(v, x, cl, K, l):
    """Responsibilities [n][K] of the kernel fault v (float64 after the faulted logits or sums)."""
    if v == "uncombined":
        l2 = logits(x, epack(cl, K, combine=False))
        return np.exp(l2 - lse64(l2)[:, None])
    if v == "no_ln_pi":
        l2 = logits(x, epack(cl, K, ln_pi=False))
        return np.exp(l2 - lse64(l2)[:, None])
    if v == "next_row":
        if x.shape[1] < 2:
            return np.exp(l - lse64(l)[:, None])
        x2 = np.array(x, np.float32)
        x2[:, 0] = x2[:, 1]
        l2 = logits(x2, epack(cl, K))
        return np.exp(l2 - lse64(l2)[:, None])
    if v == "stale_chunk":                        # slots kc..15 of the last chunk still hold the previous chunk's records
        k0 = (K - 1) // CHUNK * CHUNK
        extra = [k0 - CHUNK + kk for kk in range(K - k0, CHUNK)] if k0 >= CHUNK else []
        full = np.concatenate([l, l[:, extra]], 1) if extra else l
        return np.exp(l - lse64(full)[:, None])
    if v == "no_rescale":                         # run_sum = run_sum + exp(l - m2)
        M = np.full(l.shape[0], -np.inf)
        S = np.zeros(l.shape[0])
        for k in range(K):
            m2 = np.maximum(M, l[:, k])
            S = S + np.exp(l[:, k] - m2)
            M = m2
        return np.exp(l - (M + np.log(S))[:, None])
    if v == "sweep_run_max":
        return np.exp(l - l.max(1)[:, None])
    raise ValueError(v)


def triangle_ratio(x, cl, K, l):
    """Worst |l_emu - l64| over the a-priori bound of the FP32 triangle; l64 = -1/2 (x-mu)^T Rinv (x-mu) + constant + ln pi
    in float64."""
    D = x.shape[1]
    Ri = np.asarray(cl.Rinv[:K], np.float32).astype(np.float64)
    xm = np.asarray(x, np.float32).astype(np.float64)[:, None, :] - np.asarray(cl.means[:K], np.float32).astype(np.float64)[None]
    q = np.einsum("nki,kij,nkj->nk", xm, Ri, xm)
    A = np.einsum("nki,kij,nkj->nk", np.abs(xm), np.abs(Ri), np.abs(xm))
    const = np.asarray(cl.constant[:K], np.float32).astype(np.float64)
    lnpi = np.log(np.asarray(cl.pi[:K], np.float32).astype(np.float64))
    l64 = -0.5 * q + const + lnpi
    m = 2 * D + 3
    gam = m * U / (1 - m * U)
    bound = (0.5 * gam * A * (1 + U) ** 2 + U * np.abs(l) + U * np.abs(const + lnpi) + 2 * LOG_ULP * np.abs(lnpi)
             + 2.0 ** -50 * (np.abs(l64) + A))
    return float((np.abs(l - l64) / bound).max())


# ---- shapes (shared with tests/test_gpu_simt.py) --------------------------------------------------------------------------
KS = (1, 15, 16, 17, 33, 130)
N_SMALL_K, N_LARGE_K = 20_011, 4_097      # resident shard: a partial last 128-event block (4 097: one event in it)


def estep_cases():
    """(kind, D, K, n): every D from 1 to 32 at two K of KS each, K = 512 (32 staging chunks) and a random SPD set."""
    cases = []
    for D in range(1, 33):
        for K in (KS[(D - 1) % 6], KS[(D + 2) % 6]):
            cases.append(("fitted", D, K, N_SMALL_K if K <= 17 else N_LARGE_K))
    return cases + [("fitted", 7, 512, N_LARGE_K), ("spd", 19, 33, N_LARGE_K)]


def blobs(n, D, K):
    return entry.load_package().synth.make_blobs(n, D, min(K, 16), seed=900 + D)


N_FIT = 4_000


def param_set(pkg, oracle, kind, D, K, ev):
    """fitted: the oracle's seeding + 2 EM iterations on the first 4 000 events (near and far clusters); spd: random SPD
    parameters spread over +-6 (Mahalanobis distances in the hundreds)."""
    if kind == "spd":
        cl = random_spd_params(pkg, K, D, np.random.default_rng(D * 31 + K), spread=6.0)
        oracle.constants(cl, K)
        return cl
    return fitted_params(pkg, oracle, np.ascontiguousarray(ev[:N_FIT]), K)


N_CPU = 600
_cache = {}


def shape_result(kind, D, K, n):
    key = (kind, D, K, n)
    if key not in _cache:
        pkg = entry.load_package()
        oracle = entry.load_oracle("f64")
        ev = blobs(n, D, K)
        cl = param_set(pkg, oracle, kind, D, K, ev)
        x = np.ascontiguousarray(ev[:N_CPU])
        l = logits(x, epack(cl, K))
        gamma, lse, gbar, lbar = simt_bar(l)
        g, den = faithful(l)
        res = {"faithful": float((np.abs(g - gamma) / gbar).max()), "faithful_logp": float((np.abs(den - lse) / lbar).max()),
               "triangle": triangle_ratio(x, cl, K, l)}
        for v in FAULTS:
            gf = fault_gamma(v, x, cl, K, l)
            res[v] = float((np.abs(gf - gamma) / gbar).max())
            res[v + "_old_bar_passes"] = bool((np.abs(gf - gamma) <= 1e-4 * gamma + 1e-6).all())
        _cache[key] = res
    return _cache[key]


def _fmt(key, r):
    return (f"{key[0]:6s} D={key[1]:2d} K={key[2]:3d}  faithful {r['faithful']:.3f}  logp {r['faithful_logp']:.3f}  "
            f"triangle {r['triangle']:.3f}  " + "  ".join(f"{v} {r[v]:.3g}{'*' if r[v + '_old_bar_passes'] else ''}" for v in FAULTS))


SHAPES = estep_cases()


@pytest.mark.parametrize("kind,D,K,n", SHAPES)
def test_faithful_fp32_within_the_bar(kind, D, K, n):
    r = shape_result(kind, D, K, n)
    print("\n" + _fmt((kind, D, K), r))
    assert r["faithful"] <= FAITHFUL_MAX and r["faithful_logp"] <= FAITHFUL_MAX, r
    assert r["triangle"] <= 1.0, r


def test_each_kernel_fault_exceeds_the_bar():
    res = {s: shape_result(*s) for s in SHAPES}
    worst = {v: max(r[v] for r in res.values()) for v in FAULTS}
    print("\nworst error / bar over the shapes: " + ", ".join(f"{v} {w:.3g}" for v, w in worst.items()))
    for v in FAULTS:
        caught = [s for s, r in res.items() if r[v] > 1.0]
        old = [s for s, r in res.items() if r[v] > 1.0 and r[v + "_old_bar_passes"]]
        print(f"  {v}: above the bar at {len(caught)} of {len(res)} shapes, {len(old)} of them pass the old 1e-4 / 1e-6 bar")
        assert worst[v] > 1.0, (v, worst[v])


ZERO_PI = {"first": (7, [0]), "last": (7, [6]), "chunk1": (40, list(range(16, 32))), "chunk0": (40, list(range(16)))}


@pytest.mark.parametrize("case", list(ZERO_PI))
@pytest.mark.parametrize("D", (5, 24))
def test_zero_pi_components(case, D):
    K, zero = ZERO_PI[case]
    pkg = entry.load_package()
    oracle = entry.load_oracle("f64")
    ev = blobs(N_LARGE_K, D, K)
    cl = param_set(pkg, oracle, "fitted", D, K, ev)
    cl.pi[zero] = 0.0
    with np.errstate(invalid="ignore"):          # fma32's TwoSum tail is NaN for c = -inf; the rounded -inf is kept
        l = logits(np.ascontiguousarray(ev[:N_CPU]), epack(cl, K))
    assert np.all(l[:, zero] == -np.inf) and np.isfinite(np.delete(l, zero, 1)).all()
    with np.errstate(invalid="ignore"):          # (-inf) - (-FLT_MAX) etc. inside the bar; its results are checked below
        gamma, lse, gbar, lbar = simt_bar(l)
    g, den = faithful(l)
    for a in (gamma, lse, gbar, lbar, g, den):
        assert not np.isnan(a).any(), case
    assert np.all(g[:, zero] == 0.0) and np.all(gamma[:, zero] == 0.0)
    np.testing.assert_allclose(lse, lse64(np.delete(l, zero, 1)), rtol=1e-15, atol=0)
    assert (np.abs(g - gamma) / gbar).max() <= FAITHFUL_MAX and (np.abs(den - lse) / lbar).max() <= FAITHFUL_MAX


def _exact_fma32(a, b, c):
    """Round a * b + c (float32 inputs) to float32 with exact rationals: nearest, ties to even."""
    v = Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c))
    r = np.float32(float(v))
    cands = [np.nextafter(r, np.float32(-np.inf)), r, np.nextafter(r, np.float32(np.inf))]
    best = min(cands, key=lambda t: (abs(Fraction(float(t)) - v), int(np.float32(t).view(np.uint32)) & 1))
    return float(best)


def test_fma32_emulation_is_exact():
    rng = np.random.default_rng(5)
    n = 4000
    a = (rng.standard_normal(n) * 2.0 ** rng.integers(-20, 20, n)).astype(np.float32)
    b = (rng.standard_normal(n) * 2.0 ** rng.integers(-20, 20, n)).astype(np.float32)
    c = (rng.standard_normal(n) * 2.0 ** rng.integers(-30, 30, n)).astype(np.float32)
    c[::7] = -(a[::7].astype(np.float64) * b[::7]).astype(np.float32)           # heavy cancellation
    got = fma32(a, b, c)
    want = np.array([_exact_fma32(*t) for t in zip(a, b, c)])
    np.testing.assert_array_equal(got, want)
    # float32 midpoints that fl64(a b + c) lands on exactly, with the sign of the lost tail deciding: (1 - 2^-23)(1 + 2^-23)
    # = 1 - 2^-46, plus 2^24 + 2 sits just below the midpoint 2^24 + 3 (ties-to-even would round up to 2^24 + 4)
    a0, b0, c0 = np.float32(1 - 2.0 ** -23), np.float32(1 + 2.0 ** -23), np.float32(2.0 ** 24 + 2)
    mids = []
    for k in range(-40, 40, 3):
        for sa, sc in ((1, 1), (-1, -1)):
            mids.append((np.float32(sa * a0 * 2.0 ** k), b0, np.float32(sc * c0 * 2.0 ** k)))
            mids.append((np.float32(sa * b0 * 2.0 ** k), b0, np.float32(sc * (2.0 ** 24 + 1) * 2.0 ** k)))
    ma, mb, mc = (np.array(t, np.float32) for t in zip(*mids))
    got = fma32(ma, mb, mc)
    want = np.array([_exact_fma32(*t) for t in mids])
    np.testing.assert_array_equal(got, want)
    naive = f32(ma.astype(np.float64) * mb + mc)
    assert (naive != want).any()                                                # the midpoint path is exercised


if __name__ == "__main__":
    for s in SHAPES:
        print(_fmt(s, shape_result(*s)))
