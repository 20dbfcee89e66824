"""gmm_condition: scoring events measured on a subset of the dimensions, and imputing the others (run with -m gpu on an H100).

With every dimension observed the outputs are gmm_score's SIMT kernel's bit for bit; the imputing kernel's labels, max_resp
and logp are the marginal-only kernel's bit for bit; everything is held against the float64 restatement of gmm.h
(tests/_condition_ref.py) and against the textbook formulas on R; the variance must stay accurate on raw intensities; the
imputations must be calibrated on data drawn from the mixture; the output must not depend on the chunking; the EM state
must stay untouched; and every error of gmm.h must be reported.

FP32 bars of the imputations (each case prints its worst as COND-DEV):
  mean  |d| <= 2e-6 A + (1e-4 + 1e-6 |l_max|) sqrt(var)
        A = sum_k r_k (|mu_kM| + sum_j |G_kj dx_j|) is the magnitude the float sums run over; a float carries 6e-8 of it per
        operation and the running mean adds a few of those per cluster.  The logits carry ~1e-7 |l| of rounding (the bar
        of test_gpu_score.py), which moves the posterior weights by that relative amount and the mean by at most that
        times the spread sqrt(var) of the component means.
  var   |d| <= 2e-4 var + 4 sqrt(var) tol_mean
        (m_k - mean)^2 inherits twice the relative error of m_k - mean; the weights move var as they move the mean."""
import ctypes as C

import numpy as np
import pytest
from scipy import stats
from scipy.special import logsumexp

import _condition_ref as ref
from conftest import random_spd_params

pytestmark = pytest.mark.gpu

ERR_ARG, ERR_STATE = 1, 6


def model(pkg, K, D, seed, spread=4.0, offset=0.0):
    """A consistent parameter set: random SPD R with its inverse and constant, pi = N / sum N."""
    cl = random_spd_params(pkg, K, D, np.random.default_rng(seed), spread=spread)
    cl.means[...] += np.float32(offset)
    for k in range(K):
        R64 = cl.R[k].astype(np.float64)
        cl.Rinv[k] = np.linalg.inv(R64).astype(np.float32)
        cl.constant[k] = np.float32(-0.5 * D * np.log(2 * np.pi) - 0.5 * np.linalg.slogdet(R64)[1])
    cl.pi[...] = (cl.N / cl.N.sum()).astype(np.float32)
    return cl


def engine_with(pkg, cl, K, Kmax=None, n=4096, path=None):
    ev = pkg.synth.make_blobs(n, cl.D, 4, seed=5)
    eng = pkg.Engine(ev, Kmax or K)
    if path is not None:
        eng.set_option("estep_path", path)
    eng.set_clusters(K, cl)
    return eng


def events(cl, K, n, seed, far=0.2):
    """Events around the clusters, a fraction `far` of them well outside."""
    rng = np.random.default_rng(seed)
    D = cl.D
    k = rng.integers(0, K, n)
    x = cl.means[:K][k].astype(np.float64) + rng.standard_normal((n, D)) * 1.5
    out = rng.random(n) < far
    x[out] += rng.standard_normal((out.sum(), D)) * 12.0
    return x.astype(np.float32)


def subsets(D):
    """A single dimension, all but one, interleaved, prefix and suffix."""
    s = {(D // 2,), tuple(d for d in range(D) if d != D // 3), tuple(range(0, D, 2)), tuple(range((D + 1) // 2)),
         tuple(range(D // 2, D))}
    return sorted(t for t in s if 0 < len(t) <= D)


def top_two_gap(a):
    s = np.sort(a, axis=1)
    return s[:, -1] - s[:, -2]


def check_ref(cl, K, obs, xo, out, what):
    lab, mr, lp, mean, var, ll = out
    L, rlp, rmean, rvar, A = ref.condition(cl, K, obs, xo)
    dlp = np.abs(lp.astype(np.float64) - rlp) / (1.0 + np.abs(rlp))
    assert dlp.max() <= 1e-4, (what, float(dlp.max()))
    sure = top_two_gap(L) > 1e-3 if K > 1 else np.ones(len(xo), bool)
    np.testing.assert_array_equal(lab[sure], L.argmax(1)[sure], err_msg=what)
    assert abs(ll - float(np.sum(lp, dtype=np.float64))) <= 1e-9 * (1 + abs(ll)), what
    worst = (0.0, 0.0)
    if mean is not None:
        lmax = np.abs(L.max(1))[:, None]
        tol_m = 2e-6 * A + (1e-4 + 1e-6 * lmax) * np.sqrt(rvar)
        dm = np.abs(mean.astype(np.float64) - rmean)
        assert np.all(dm <= tol_m), (what, float((dm / tol_m).max()))
        tol_v = 2e-4 * rvar + 4.0 * np.sqrt(rvar) * tol_m
        dv = np.abs(var.astype(np.float64) - rvar)
        assert np.all(dv <= tol_v), (what, float((dv / tol_v).max()))
        worst = (float((dm / tol_m).max()), float((dv / tol_v).max()))
        print(f"\nCOND-DEV {what}: logp {dlp.max():.2e}, mean {worst[0]:.3f} of the bar, var {worst[1]:.3f} of the bar")
    return worst


# ---- 1. every dimension observed = gmm_score's SIMT kernel -----------------------------------------------------------------
@pytest.mark.parametrize("D,K", [(D, K) for D in (5, 24, 32) for K in (1, 7, 64, 130)])
def test_full_set_is_score(pkg, D, K):
    cl = model(pkg, K, D, seed=D * 100 + K)
    x = events(cl, K, 20_011, seed=K)
    with engine_with(pkg, cl, K, path=pkg.PATH_SIMT) as eng:
        lab, mr, lp, sll = eng.score(K, x)
        out = eng.condition(K, np.arange(D), x, mean=True, var=True)
        assert out[3] is None and out[4] is None
        np.testing.assert_array_equal(out[0], lab)
        np.testing.assert_array_equal(out[1], mr)
        np.testing.assert_array_equal(out[2], lp)
        assert abs(out[5] - sll) <= 1e-12 * abs(sll)            # (the block sums are added by atomics)


def test_full_set_after_device_finalisation(pkg):
    n, D, K = 200_000, 24, 32
    ev = pkg.synth.make_blobs(n, D, K, seed=8)
    with pkg.Engine(ev, K) as eng:
        eng.set_option("path", pkg.PATH_TENSOR)
        eng.seed(K)
        eng.em(K, 2, 2)
        eng.em_iterations(K, 3)                              # device finalisation: the host copy is refreshed after it
        got = eng.condition(K, np.arange(D), ev[:50_000])
        cur = eng.get_clusters(K)
    with engine_with(pkg, cur, K, path=pkg.PATH_SIMT) as simt:
        lab, mr, lp, sll = simt.score(K, ev[:50_000])
    np.testing.assert_array_equal(got[0], lab)
    np.testing.assert_array_equal(got[1], mr)
    np.testing.assert_array_equal(got[2], lp)
    assert abs(got[5] - sll) <= 1e-12 * abs(sll)


# ---- 2. the imputing kernel scores as the marginal-only kernel --------------------------------------------------------------
@pytest.mark.parametrize("n_obs,nm", [(o, m) for o in (1, 2, 3, 4, 5, 6, 7, 8) for m in (1, 2, 3, 4) if o + m <= 12] + [(21, 11), (31, 1), (1, 31)])
def test_paths_agree(pkg, n_obs, nm):
    D, K = n_obs + nm, 37
    cl = model(pkg, K, D, seed=n_obs * 64 + nm)
    obs = np.sort(np.random.default_rng(nm).choice(D, n_obs, replace=False))
    x = events(cl, K, 9_001, seed=3)[:, obs]
    x[5, 0] = np.nan                                         # a row that is not finite
    with engine_with(pkg, cl, K) as eng:
        a = eng.condition(K, obs, x, mean=False)
        b = eng.condition(K, obs, x, mean=True, var=True)
    for i in range(3):
        np.testing.assert_array_equal(a[i], b[i])
    assert np.isnan(a[5]) and np.isnan(b[5])                # the NaN row
    assert b[0][5] == -1 and np.isnan(b[1][5]) and np.isnan(b[2][5])
    assert np.all(np.isnan(b[3][5])) and np.all(np.isnan(b[4][5]))
    fin = np.ones(len(x), bool)
    fin[5] = False
    assert np.all(np.isfinite(b[3][fin])) and np.all(b[4][fin] > 0)


# ---- 3. float64 restatement -------------------------------------------------------------------------------------------------
RESTATE = [(D, K) for D in (2, 3, 8, 16, 24, 31, 32) for K in (1, 3, 64, 65)] + [(4, 512)]


@pytest.mark.parametrize("D,K", RESTATE)
def test_matches_restatement(pkg, D, K):
    cl = model(pkg, K, D, seed=D * 1000 + K)
    x = events(cl, K, 3001, seed=D + K)
    with engine_with(pkg, cl, K) as eng:
        for obs in subsets(D):
            obs = np.asarray(obs)
            out = eng.condition(K, obs, x[:, obs], var=True)
            check_ref(cl, K, obs, x[:, obs], out, f"D={D} K={K} obs={obs.tolist()}")


# ---- 4. the math from R -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D,K", [(6, 1), (12, 4)])
def test_textbook(pkg, D, K):
    cl = model(pkg, K, D, seed=77 + K)
    x = events(cl, K, 2000, seed=1)
    obs = np.array([0, 2, 3, D - 1])
    mis = np.setdiff1d(np.arange(D), obs)
    with engine_with(pkg, cl, K) as eng:
        lab, mr, lp, mean, var, _ = eng.condition(K, obs, x[:, obs], var=True)
    xo = x[:, obs].astype(np.float64)
    dens, ms, vs = [], [], []
    for k in range(K):
        R = cl.R[k].astype(np.float64)
        mu = cl.means[k].astype(np.float64)
        Roo, Rmo, Rmm = R[np.ix_(obs, obs)], R[np.ix_(mis, obs)], R[np.ix_(mis, mis)]
        dens.append(np.log(float(cl.pi[k])) + stats.multivariate_normal(mu[obs], Roo).logpdf(xo).reshape(-1))
        W = Rmo @ np.linalg.inv(Roo)
        ms.append(mu[mis] + (xo - mu[obs]) @ W.T)
        vs.append(np.diag(Rmm - W @ Rmo.T))
    Lk = np.stack(dens, 1)
    rlp = logsumexp(Lk, axis=1)
    r = np.exp(Lk - rlp[:, None])
    M = np.stack(ms, 0)
    rmean = np.einsum("nk,knd->nd", r, M)
    rvar = np.einsum("nk,knd->nd", r, np.stack(vs, 0)[:, None, :] + (M - rmean[None]) ** 2)
    # float Rinv against inv(R): a relative perturbation of 6e-8 cond(R) in the precision
    cond = max(np.linalg.cond(cl.R[k].astype(np.float64)) for k in range(K))
    e = 1e-4 + 1e-7 * cond
    np.testing.assert_allclose(lp, rlp, rtol=e, atol=e)
    np.testing.assert_allclose(mean, rmean, rtol=0, atol=e * (1 + np.abs(rmean).max()))
    np.testing.assert_allclose(var, rvar, rtol=10 * e, atol=10 * e * rvar.max())


# ---- 5. stable variance on raw intensities ----------------------------------------------------------------------------------
@pytest.mark.parametrize("spread", [40.0, 1.0])           # separated, overlapping
def test_variance_at_large_means(pkg, spread):
    D, K = 8, 12
    cl = random_spd_params(pkg, K, D, np.random.default_rng(5), spread=spread)
    cl.means[...] += np.float32(1e4)
    for k in range(K):
        cl.R[k] = np.eye(D, dtype=np.float32)
        cl.Rinv[k] = np.eye(D, dtype=np.float32)
        cl.constant[k] = np.float32(-0.5 * D * np.log(2 * np.pi))
    cl.pi[...] = (cl.N / cl.N.sum()).astype(np.float32)
    x = events(cl, K, 20_000, seed=2, far=0.0)
    obs = np.array([0, 1, 2, 5])
    with engine_with(pkg, cl, K) as eng:
        out = eng.condition(K, obs, x[:, obs], var=True)
    check_ref(cl, K, obs, x[:, obs], out, f"means 1e4 spread={spread}")
    _, rlp, rmean, rvar, _ = ref.condition(cl, K, obs, x[:, obs])
    # the naive sum_k r_k (c_k + m_k^2) - mean^2 in float: off by units at 1e4 (float carries 1e8 * 6e-8 = 6 of m^2)
    assert np.abs(out[4].astype(np.float64) - rvar).max() < 0.05 * rvar.min()


# ---- 6. calibration on events drawn from the mixture ------------------------------------------------------------------------
def test_calibration(pkg):
    n, D, K = 400_000, 12, 8
    ev = pkg.synth.make_blobs(n, D, K, seed=21)
    obs = np.array([0, 1, 3, 4, 6, 8, 9])
    mis = np.setdiff1d(np.arange(D), obs)
    with pkg.Engine(ev, K) as eng:
        eng.seed(K)
        eng.em(K, 10, 10)
        x, _ = eng.sample(K, 1_000_000, seed=4)
        _, _, _, mean, var, _ = eng.condition(K, obs, x[:, obs], labels=False, max_resp=False, logp=False, var=True)
    z2 = (x[:, mis].astype(np.float64) - mean) ** 2 / var
    m = z2.mean(0)
    print(f"\nCOND-CALIBRATION mean z^2 per missing dimension: {np.round(m, 4).tolist()}")
    assert np.all(np.abs(m - 1.0) <= 0.02), m


# ---- 7. chunking ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D,K", [(24, 64), (16, 5)])
def test_chunking(pkg, D, K):
    cl = model(pkg, K, D, seed=9)
    x = events(cl, K, 20_000, seed=4)
    obs = np.arange(0, D, 3)
    with engine_with(pkg, cl, K) as eng:
        base = eng.condition(K, obs, x[:, obs], var=True)
        for chunk in (1, 33, 4097, 1 << 20):
            if chunk == 1:
                xs = x[:300]
                b = eng.condition(K, obs, xs[:, obs], var=True)
                eng.set_option("score_chunk", 1)
                o = eng.condition(K, obs, xs[:, obs], var=True)
                for i in range(5):
                    np.testing.assert_array_equal(o[i], b[i])
                continue
            eng.set_option("score_chunk", chunk)
            o = eng.condition(K, obs, x[:, obs], var=True)
            for i in range(5):
                np.testing.assert_array_equal(o[i], base[i])
            assert abs(o[5] - base[5]) <= 1e-12 * abs(base[5])
        a = eng.condition(K, obs, x[:7_777, obs], var=True)
        b = eng.condition(K, obs, x[7_777:, obs], var=True)
        for i in range(5):
            np.testing.assert_array_equal(np.concatenate([a[i], b[i]]), base[i])
        prof = eng.condition_profile(reset=True)
        assert prof["kernel_ms"] > 0 and prof["wall_ms"] >= prof["kernel_ms"]
        assert eng.condition_profile() == dict(kernel_ms=0.0, wall_ms=0.0)


# ---- 8. EM state untouched --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("path", ["simt", "tensor"])
def test_no_interference(pkg, path):
    n, D, K = 200_000, 16, 16
    ev = pkg.synth.make_blobs(n, D, K, seed=8)
    runs = []
    for interleave in (False, True):
        with pkg.Engine(ev, K) as eng:
            if path == "simt":
                eng.set_option("path", pkg.PATH_SIMT)
            eng.seed(K)
            ll0, _ = eng.em(K, 3, 3)
            if interleave:
                profs = (eng.profile(), eng.score_profile(), eng.score_stats_profile(), eng.sample_profile())
                eng.condition(K, [1, 4, 5], ev[:50_000, [1, 4, 5]], var=True)
                eng.condition(K, np.arange(D), ev[:50_000])
                assert (eng.profile(), eng.score_profile(), eng.score_stats_profile(), eng.sample_profile()) == profs
            ll1 = eng.em_iterations(K, 3)
            if interleave:
                eng.condition(K, [0, 15], ev[:10_000, [0, 15]])
            ll2 = eng.em_iterations(K, 2)
            lab, mr, lp, _ = eng.score(K, ev[:10_000])
            got = eng.get_clusters(K, with_memberships=True)
            runs.append((ll0, ll1, ll2, got, lab, mr, lp))
    (a0, a1, a2, A, *sa), (b0, b1, b2, B, *sb) = runs
    assert (a0, a1, a2) == (b0, b1, b2)
    for f in ("N", "pi", "constant", "means", "R", "Rinv", "memberships"):
        np.testing.assert_array_equal(getattr(A, f), getattr(B, f), err_msg=f)
    for u, v in zip(sa, sb):
        np.testing.assert_array_equal(u, v)


# ---- 9. errors --------------------------------------------------------------------------------------------------------------
def raw(eng, K, obs, n_obs, x, n, lab=None, mean=None, ll=None):
    ptr = lambda a: a.ctypes.data if a is not None else None  # noqa: E731
    return eng.lib.gmm_condition(eng.h, K, ptr(obs), n_obs, ptr(x), n, ptr(lab), None, None, ptr(mean), None,
                                 C.byref(ll) if ll is not None else None)


def test_errors(pkg):
    D, K, Kmax = 4, 4, 8
    good = model(pkg, K, D, seed=3)
    x = np.ones((16, 2), np.float32)
    with engine_with(pkg, good, K, Kmax=Kmax) as eng:
        def err(fn):
            with pytest.raises(pkg.GmmError) as e:
                fn()
            return e.value.code, str(e.value)
        obs = np.array([0, 2], np.int32)
        assert err(lambda: eng.condition(0, obs, x))[0] == ERR_ARG
        assert err(lambda: eng.condition(Kmax + 1, obs, x))[0] == ERR_ARG
        assert raw(eng, K, obs, 2, x, -1) == ERR_ARG
        assert raw(eng, K, obs, 2, None, 16) == ERR_ARG                        # no rows
        assert raw(eng, K, None, 2, x, 16) == ERR_ARG                          # no obs_dims
        assert raw(eng, K, obs, 0, x, 16) == ERR_ARG
        assert raw(eng, K, np.arange(5, dtype=np.int32), 5, np.ones((16, 5), np.float32), 16) == ERR_ARG   # n_obs > D
        for bad in ([2, 0], [1, 1], [0, 4], [-1, 2]):
            assert err(lambda: eng.condition(K, bad, x))[0] == ERR_ARG, bad
        lab = np.full(16, 7, np.int32)
        mean = np.full((16, 2), 7.0, np.float32)
        ll = C.c_double(7.0)
        assert raw(eng, K, obs, 2, x, 0, lab, mean, ll) == 0                   # n = 0 writes nothing
        assert np.all(lab == 7) and np.all(mean == 7.0) and ll.value == 7.0
        assert err(lambda: eng.condition(K + 1, obs, x))[0] == ERR_STATE        # not the current K
        eng.estep(K)
        eng.mstep(K)
        assert err(lambda: eng.condition(K, obs, x))[0] == ERR_STATE            # between gmm_mstep and gmm_constants
        eng.constants(K)
        eng.condition(K, obs, x)
        bad = good.copy()
        bad.Rinv[2] = np.diag([1.0, -1.0, 1.0, 1.0]).astype(np.float32)       # P_MM indefinite for M = {1, 3}
        eng.set_clusters(K, bad)
        code, msg = err(lambda: eng.condition(K, obs, x))
        assert code == ERR_STATE and "cluster 2" in msg, msg
        eng.condition(K, [1, 2], x)                                             # M = {0, 3}: positive definite
        eng.set_clusters(K, good)
        eng.condition(K, obs, x)
