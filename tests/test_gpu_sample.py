"""gmm_sample: drawing events from a fitted mixture (run with -m gpu on an H100).

Labels must equal the numpy restatement (tests/_sample_ref.py) bit for bit, and events must agree with its float64
arithmetic within 4e-6 (|mu_d| + sum_j |U_dj z_j|); the worst observed on an H100 is 5.0e-7 (D = 32, K = 3), and each case
prints its own as SAMPLE-DEV.  The output must not
depend on the chunking, the split into calls, the path option or the context; its distribution must pass goodness-of-fit
tests; a fit -> sample -> gmm_score_stats round trip must give back the fitted weights and means; sampling must leave the
EM state alone; and every error of gmm.h must be reported."""
import ctypes as C

import numpy as np
import pytest
from scipy import stats

import _sample_ref as ref
from conftest import random_spd_params

pytestmark = pytest.mark.gpu

ERR_ARG, ERR_STATE = 1, 6
EV_TOL = 4e-6


def model(pkg, K, D, seed, spread=4.0):
    """A consistent parameter set: random SPD R with its inverse and constant, pi = N / sum N."""
    cl = random_spd_params(pkg, K, D, np.random.default_rng(seed), spread=spread)
    for k in range(K):
        R64 = cl.R[k].astype(np.float64)
        cl.Rinv[k] = np.linalg.inv(R64).astype(np.float32)
        cl.constant[k] = np.float32(-0.5 * D * np.log(2 * np.pi) - 0.5 * np.linalg.slogdet(R64)[1])
    cl.pi[...] = (cl.N / cl.N.sum()).astype(np.float32)
    return cl


def engine_with(pkg, cl, K, Kmax=None, n=4096):
    ev = pkg.synth.make_blobs(n, cl.D, 4, seed=5)
    eng = pkg.Engine(ev, Kmax or K)
    eng.set_clusters(K, cl)
    return eng


def raw_sample(eng, K, n, seed, first, out, labels=None):
    ptr = lambda a: a.ctypes.data if a is not None else None  # noqa: E731
    return eng.lib.gmm_sample(eng.h, K, n, C.c_ulonglong(seed), first, ptr(out), ptr(labels))


def check_restatement(cl, K, seed, first, x, lab, what):
    xr, lr, scale = ref.sample(cl, K, seed, first, x.shape[0])
    np.testing.assert_array_equal(lab, lr, err_msg=what)
    dev = np.abs(x.astype(np.float64) - xr) / scale
    print(f"\nSAMPLE-DEV {what}: max |dx| / (|mu| + sum |U z|) = {dev.max():.2e}")
    assert dev.max() <= EV_TOL, (what, float(dev.max()))
    return float(dev.max())


# ---- 1. restatement ---------------------------------------------------------------------------------------------------------
RESTATE = [(D, K) for D in (1, 2, 3, 8, 16, 24, 31, 32) for K in (1, 3, 64, 65)] + [(4, 512)]


@pytest.mark.parametrize("D,K", RESTATE)
def test_matches_restatement(pkg, D, K):
    cl = model(pkg, K, D, seed=D * 1000 + K)
    if K >= 3:
        cl.pi[1] = 0.0                                          # never drawn
    n, seed = 5003, 0x9E3779B97F4A7C15 ^ (D * K)
    with engine_with(pkg, cl, K) as eng:
        for first in (0, (1 << 32) + 5):
            x, lab = eng.sample(K, n, seed=seed, first=first)
            check_restatement(cl, K, seed, first, x, lab, f"D={D} K={K} first={first}")
            if K >= 3:
                assert not np.any(lab == 1)
            assert lab.min() >= 0 and lab.max() < K


# ---- 2. invariance ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D,K", [(24, 64), (32, 512)])      # parameters staged in shared memory / read through L1
def test_invariance(pkg, D, K):
    cl = model(pkg, K, D, seed=7)
    n, seed = 50_000, 1234
    with engine_with(pkg, cl, K) as eng, engine_with(pkg, cl, K) as eng2:
        x, lab = eng.sample(K, 2 * n, seed=seed)
        for chunk in (1000, 1 << 20):
            eng.set_option("score_chunk", chunk)
            x2, lab2 = eng.sample(K, 2 * n, seed=seed)
            np.testing.assert_array_equal(x2, x)
            np.testing.assert_array_equal(lab2, lab)
        eng.set_option("score_chunk", 777)
        a, la = eng.sample(K, 12_345, seed=seed)
        b, lb = eng.sample(K, 2 * n - 12_345, seed=seed, first=12_345)
        np.testing.assert_array_equal(np.concatenate([a, b]), x)
        np.testing.assert_array_equal(np.concatenate([la, lb]), lab)
        eng.set_option("path", pkg.PATH_SIMT)
        x3, _ = eng.sample(K, 2 * n, seed=seed)
        np.testing.assert_array_equal(x3, x)
        # two contexts on one GPU, as two ranks would split the sample
        p, lp = eng.sample(K, n, seed=seed)
        q, lq = eng2.sample(K, n, seed=seed, first=n)
        np.testing.assert_array_equal(np.concatenate([p, q]), x)
        np.testing.assert_array_equal(np.concatenate([lp, lq]), lab)
        again, _ = eng2.sample(K, 2 * n, seed=seed)
        np.testing.assert_array_equal(again, x)
        other, lo = eng2.sample(K, 2 * n, seed=seed + 1)
        assert np.mean(np.all(other != x, axis=1)) > 0.99 and np.mean(lo != lab) > 0.5
        _, none = eng2.sample(K, 10, seed=seed, labels=False)
        assert none is None
        prof = eng2.sample_profile(reset=True)
        assert prof["kernel_ms"] > 0 and prof["wall_ms"] >= prof["kernel_ms"]
        assert eng2.sample_profile() == dict(kernel_ms=0.0, wall_ms=0.0)


# ---- 3. distribution --------------------------------------------------------------------------------------------------------
def test_distribution(pkg):
    K, D, n = 8, 16, 4_000_000
    cl = model(pkg, K, D, seed=2024)
    with engine_with(pkg, cl, K) as eng:
        x, lab = eng.sample(K, n, seed=99)
    p = cl.pi[:K].astype(np.float64) / cl.pi[:K].astype(np.float64).sum()
    counts = np.bincount(lab, minlength=K)
    chi = stats.chisquare(counts, p * n)
    assert chi.pvalue > 1e-4, chi
    x64 = x.astype(np.float64)
    for k in range(K):
        sel = lab == k
        se = np.sqrt(np.diag(cl.R[k]).astype(np.float64) / sel.sum())
        z = (x64[sel].mean(0) - cl.means[k]) / se
        assert np.abs(z).max() < 5.0, (k, z)
    sub, ls = x64[:1_000_000], lab[:1_000_000]
    d2 = np.empty(len(sub))
    for k in range(K):
        sel = ls == k
        d = sub[sel] - cl.means[k]
        d2[sel] = np.einsum("ni,ni->n", d @ np.linalg.inv(cl.R[k].astype(np.float64)), d)
    ks = stats.kstest(d2, stats.chi2(D).cdf)
    print(f"\nSAMPLE-DIST chi2 p = {chi.pvalue:.3g}, KS p = {ks.pvalue:.3g}")
    assert ks.pvalue > 1e-4, ks


# ---- 4. round trip ----------------------------------------------------------------------------------------------------------
def test_fit_sample_score_stats_round_trip(pkg):
    n, D, K = 1_000_000, 16, 32
    ev = pkg.synth.make_blobs(n, D, K, seed=31)
    with pkg.Engine(ev, K) as eng:
        eng.seed(K)
        eng.em(K, 20, 20)
        fit = eng.get_clusters(K)
        x, _ = eng.sample(K, n, seed=5)
        st, sh, _ = eng.score_stats(K, x)
    got = pkg.Clusters(K, D)                                    # avgvar 0: the sample's own covariances
    pkg.host_finalize(st, sh, got, K)
    pi = fit.pi[:K].astype(np.float64) / fit.pi[:K].astype(np.float64).sum()
    live = pi * n >= 50
    assert live.sum() >= K // 2
    frac = got.N[:K].astype(np.float64) / n
    sigma = np.sqrt(pi * (1 - pi) / n)
    assert np.all(np.abs(frac - pi)[live] <= 4 * sigma[live] + 1e-6), np.max((np.abs(frac - pi) / sigma)[live])
    for k in np.nonzero(live)[0]:
        se = np.sqrt(np.diag(fit.R[k]).astype(np.float64) / (pi[k] * n))
        dz = (got.means[k].astype(np.float64) - fit.means[k]) / se
        assert np.abs(dz).max() < 6.0, (k, dz)


# ---- 5. no interference -----------------------------------------------------------------------------------------------------
def test_no_interference(pkg):
    n, D, K = 200_000, 16, 16
    ev = pkg.synth.make_blobs(n, D, K, seed=8)
    runs = []
    for interleave in (False, True):
        with pkg.Engine(ev, K) as eng:
            eng.seed(K)
            ll0, _ = eng.em(K, 3, 3)
            if interleave:
                sp, prof = eng.score_profile(), eng.profile()
                eng.sample(K, 100_000, seed=1)
                assert eng.score_profile() == sp and eng.profile() == prof
            ll1 = eng.em_iterations(K, 3)                       # device finalisation: the host copy is refreshed after it
            if interleave:
                cur = eng.get_clusters(K)
                x, lab = eng.sample(K, 20_000, seed=2)
                check_restatement(cur, K, 2, 0, x, lab, "after gmm_em_iterations")
            ll2 = eng.em_iterations(K, 2)
            got = eng.get_clusters(K, with_memberships=True)
            runs.append((ll0, ll1, ll2, got))
    (a0, a1, a2, A), (b0, b1, b2, B) = runs
    assert (a0, a1, a2) == (b0, b1, b2)
    for f in ("N", "pi", "constant", "means", "R", "Rinv", "memberships"):
        np.testing.assert_array_equal(getattr(A, f), getattr(B, f), err_msg=f)


# ---- 6. errors --------------------------------------------------------------------------------------------------------------
def test_errors(pkg):
    D, K, Kmax = 4, 4, 8
    good = model(pkg, K, D, seed=3)
    out = np.full((16, D), 7.0, np.float32)
    with engine_with(pkg, good, K, Kmax=Kmax) as eng:
        def err(fn):
            with pytest.raises(pkg.GmmError) as e:
                fn()
            return e.value.code, str(e.value)
        assert err(lambda: eng.sample(0, 10))[0] == ERR_ARG
        assert err(lambda: eng.sample(Kmax + 1, 10))[0] == ERR_ARG
        assert err(lambda: eng.sample(K, -1))[0] == ERR_ARG
        assert err(lambda: eng.sample(K, 10, first=-1))[0] == ERR_ARG
        assert err(lambda: eng.sample(K, 10, first=(1 << 62) - 9))[0] == ERR_ARG
        assert raw_sample(eng, K, 10, 0, 0, None) == ERR_ARG
        x, _ = eng.sample(K, 10, first=(1 << 62) - 10)        # the last events of the range
        assert np.all(np.isfinite(x))
        assert raw_sample(eng, K, 0, 0, 0, out) == 0 and np.all(out == 7.0)   # n = 0 writes nothing
        assert err(lambda: eng.sample(K + 1, 10))[0] == ERR_STATE            # not the current K
        eng.estep(K)
        eng.mstep(K)
        assert err(lambda: eng.sample(K, 10))[0] == ERR_STATE               # between gmm_mstep and gmm_constants
        eng.constants(K)
        eng.sample(K, 10)
        bad = good.copy()
        bad.R[2] = np.diag([1.0, -1.0, 1.0, 1.0]).astype(np.float32)      # indefinite
        eng.set_clusters(K, bad)
        code, msg = err(lambda: eng.sample(K, 10))
        assert code == ERR_STATE and "cluster 2" in msg, msg
        for k, v in ((1, -0.1), (3, np.nan), (0, np.inf)):
            bad = good.copy()
            bad.pi[k] = v
            eng.set_clusters(K, bad)
            code, msg = err(lambda: eng.sample(K, 10))
            assert code == ERR_STATE and f"cluster {k}" in msg, msg
        bad = good.copy()
        bad.pi[:] = 0.0
        eng.set_clusters(K, bad)
        assert err(lambda: eng.sample(K, 10))[0] == ERR_STATE               # T = 0
        eng.set_clusters(K, good)
        eng.sample(K, 10)
