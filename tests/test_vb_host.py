"""gmm_vb_em's host side, no GPU needed: the float64 restatement (_vb_ref.py) against sklearn's BayesianGaussianMixture,
gmm_host_vb_finalize against the restatement, the library's digamma, and the prior's argument errors."""
import ctypes as C

import numpy as np
import pytest
from scipy.special import digamma

import _vb_ref as vb

DS = (1, 2, 5, 24, 32)
KS = (1, 3, 64, 130)


def _case(D, K, seed, n=None):
    rng = np.random.default_rng(seed)
    n = n or max(3 * K, 200)
    X = rng.standard_normal((n, D)) * rng.uniform(0.5, 3.0, D) + rng.uniform(-5, 5, D)
    resp = rng.dirichlet(np.full(K, 0.3), size=n)
    if K > 1:                                               # all-zero columns, some components nearly empty
        resp[:, rng.choice(K, size=max(1, K // 4), replace=False)] = 0.0
        resp[:, -1] *= 1e-9
        resp /= resp.sum(1, keepdims=True)
    return X, resp


def _prior(X, K, ptype, rng):
    m0, psi0 = vb.default_moments(X)
    if ptype == vb.DP:
        return vb.prior(K, X.shape[1], ptype, m0=m0, psi0=psi0)
    D = X.shape[1]
    return vb.prior(K, D, ptype, gamma0=0.7, beta0=0.3, nu0=D + 1.5, m0=m0 + 0.1, psi0=psi0 * 1.3, reg=1e-5)


def _close(a, b, rtol, what):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    scale = max(1e-300, float(np.abs(b).max()))
    err = float(np.abs(a - b).max()) / scale
    assert err <= rtol, f"{what}: {err:.3g} > {rtol}"


@pytest.mark.parametrize("ptype", [vb.DP, vb.DIRICHLET])
@pytest.mark.parametrize("D", DS)
@pytest.mark.parametrize("K", KS)
def test_restatement_matches_sklearn(D, K, ptype):
    mixture = pytest.importorskip("sklearn.mixture")
    X, resp = _case(D, K, 100 * D + K + ptype)
    pr = _prior(X, K, ptype, None)
    bgm = mixture.BayesianGaussianMixture(
        n_components=K, covariance_type="full", reg_covar=pr["reg"], mean_prior=pr["m0"], covariance_prior=pr["psi0"],
        weight_concentration_prior_type="dirichlet_process" if ptype == vb.DP else "dirichlet_distribution",
        weight_concentration_prior=pr["gamma0"], mean_precision_prior=pr["beta0"], degrees_of_freedom_prior=pr["nu0"])
    bgm._check_parameters(X)
    with np.errstate(divide="ignore"):                     # exp(-1e300) = 0 and 0 * -1e300 = 0: sklearn's terms of empty columns
        log_resp = np.where(resp > 0, np.log(resp), -1e300)
    bgm._m_step(X, log_resp)
    p = vb.m_step_resp(X, resp, pr, rounding=False)
    tol = 1e-12
    _close(p["weight_concentration"], np.array(bgm.weight_concentration_), tol, "weight_concentration")
    _close(p["beta"], bgm.mean_precision_, tol, "mean_precision")
    _close(p["m"], bgm.means_, tol, "means")
    _close(p["nu"], bgm.degrees_of_freedom_, tol, "dof")
    _close(p["C"], bgm.covariances_, tol, "covariances")
    _close(p["elog"], bgm._estimate_log_weights(), tol, "log weights")
    ref_lp = bgm._estimate_log_prob(X) + bgm._estimate_log_weights()
    _close(vb.log_prob(X, p), ref_lp, tol, "weighted log prob")
    lb = bgm._compute_lower_bound(log_resp, None)
    got_lb = -vb.entropy_sum(resp) + p["bound_par"]
    assert abs(got_lb - lb) <= tol * max(1.0, abs(lb)), (got_lb, lb)
    bgm._set_parameters(bgm._get_parameters())
    _close(p["weights"], bgm.weights_, tol, "weights_")
    # the statistics route (packed S0 / S1 / S2 about a centre) gives the same M-step
    shift = X.mean(0) + 0.25
    q = vb.m_step(vb.stats_from_resp(X, resp, shift), shift, K, D, pr, rounding=False)
    for key in ("beta", "m", "nu", "C", "weights", "elog"):
        _close(q[key], p[key], 1e-10, key)


def _host(pkg, stats, shift, K, D, pr):
    cl = pkg.Clusters(K, D)
    cl.avgvar[...] = 0.125
    post, bound = pkg.host_vb_finalize(stats, shift, cl, K, pr["m0"], pr["psi0"], prior_type=pr["type"], weight_concentration=pr["gamma0"],
                                       mean_precision=pr["beta0"], dof=pr["nu0"], reg_covar=pr["reg"])
    return cl, post, bound


def _ulp_close(a, b, what, extra=0.0):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    ulp = np.spacing(np.abs(b).astype(np.float32))
    bad = np.abs(a.astype(np.float64) - b.astype(np.float64)) > ulp.astype(np.float64) + extra
    assert not bad.any(), f"{what}: {int(bad.sum())} entries beyond one ulp, max diff {np.abs(a - b).max():.3g}"


@pytest.mark.parametrize("ptype", [vb.DP, vb.DIRICHLET])
@pytest.mark.parametrize("D", DS)
@pytest.mark.parametrize("K", KS)
def test_host_vb_finalize_matches_restatement(pkg, D, K, ptype):
    X, resp = _case(D, K, 7 * D + K + ptype)
    pr = _prior(X, K, ptype, None)
    shift = X.mean(0).astype(np.float32).astype(np.float64)
    stats = vb.stats_from_resp(X, resp, shift)
    cl, post, bound = _host(pkg, stats, shift, K, D, pr)
    p = vb.m_step(stats, shift, K, D, pr, rounding=True)
    _ulp_close(cl.N[:K], p["N"], "N")
    _ulp_close(cl.means[:K], p["means"], "means")
    _ulp_close(cl.R[:K], p["R"], "R")
    _ulp_close(cl.pi[:K], p["pi"], "pi")
    for k in range(K):                                      # the inverse: one ulp plus the conditioning of the float R
        cond = np.linalg.cond(p["R"][k].astype(np.float64))
        _ulp_close(cl.Rinv[k], p["Rinv"][k], f"Rinv[{k}]", extra=cond * 1e-15 * float(np.abs(p["Rinv"][k]).max()))
    _ulp_close(cl.constant[:K], p["constant"], "constant", extra=1e-12 * float(np.abs(p["constant"]).max()))
    assert (cl.avgvar == np.float32(0.125)).all()
    for key, ref in (("weights", p["weights"]), ("weight_concentration", p["weight_concentration"]), ("mean_precision", p["beta"]),
                     ("dof", p["nu"]), ("mean_prior", pr["m0"]), ("covariance_prior", pr["psi0"])):
        np.testing.assert_allclose(post[key], ref, rtol=1e-13, atol=1e-300, err_msg=key)
    assert abs(bound - p["bound_par"]) <= 1e-13 * max(1.0, abs(p["bound_par"])), (bound, p["bound_par"])


def test_digamma_matches_scipy(pkg):
    x = np.concatenate([np.geomspace(1e-3, 1e9, 20001), np.linspace(0.5, 30.0, 5001), [1.4616321449683622]])
    got = pkg.host_digamma(x)
    ref = digamma(x)
    err = np.abs(got - ref)
    # a few ulps of max(|psi|, 1): relative where |psi| is large, absolute around the root at 1.4616
    assert (err <= 2e-15 * np.maximum(np.abs(ref), 1.0)).all(), float((err / np.maximum(np.abs(ref), 1.0)).max())


def _call(pkg, D, K=3, **kw):
    X, resp = _case(D, K, 5)
    m0, psi0 = vb.default_moments(X)
    shift = np.zeros(D)
    stats = vb.stats_from_resp(X, resp, shift)
    args = dict(mean=m0, covariance=psi0)
    args.update(kw)
    cl = pkg.Clusters(K, D)
    return pkg.host_vb_finalize(stats, shift, cl, K, **args)


@pytest.mark.parametrize("kw", [
    dict(prior_type=2), dict(weight_concentration=np.inf), dict(weight_concentration=np.nan), dict(mean_precision=np.nan),
    dict(mean_precision=-np.inf), dict(dof=2.0), dict(dof=3.9), dict(dof=np.nan), dict(dof=np.inf), dict(reg_covar=np.nan),
    dict(covariance="asym"), dict(covariance="indef"), dict(covariance="nan"), dict(mean="nan"), dict(mean=None), dict(covariance=None)])
def test_prior_errors(pkg, kw):
    D = 5
    kw = dict(kw)
    if isinstance(kw.get("covariance"), str):
        c = np.eye(D) * 2.0
        if kw["covariance"] == "asym":
            c[0, 1] = 0.5
        elif kw["covariance"] == "indef":
            c[2, 2] = -1.0
        else:
            c[1, 1] = np.nan
        kw["covariance"] = c
    if isinstance(kw.get("mean"), str):
        kw["mean"] = np.full(D, np.nan)
    with pytest.raises(pkg.GmmError) as e:
        _call(pkg, D, **kw)
    assert e.value.code == 1


def test_prior_defaults(pkg):
    """<= 0 selects gamma0 = 1/K, beta0 = 1, nu0 = D; reg_covar < 0 selects 1e-6."""
    D, K = 5, 3
    X, resp = _case(D, K, 5)
    m0, psi0 = vb.default_moments(X)
    shift = np.zeros(D)
    stats = vb.stats_from_resp(X, resp, shift)
    cl = pkg.Clusters(K, D)
    post, bound = pkg.host_vb_finalize(stats, shift, cl, K, m0, psi0, weight_concentration=0.0, mean_precision=-1.0, dof=0.0, reg_covar=-1.0)
    p = vb.m_step(stats, shift, K, D, vb.prior(K, D, vb.DP, m0=m0, psi0=psi0), rounding=True)
    np.testing.assert_allclose(post["weight_concentration"], p["weight_concentration"], rtol=1e-13)
    np.testing.assert_allclose(post["dof"], p["nu"], rtol=1e-13)
    assert abs(bound - p["bound_par"]) <= 1e-13 * abs(p["bound_par"])


def test_dof_at_the_bound_is_accepted(pkg):
    D = 5
    post, _ = _call(pkg, D, dof=D - 1 + 1e-9)
    assert np.isfinite(post["dof"]).all()


def test_host_vb_finalize_null_arguments(pkg):
    L = pkg.load_library()
    rc = L.gmm_host_vb_finalize(None, None, 3, 2, None, None, None, None)
    assert rc == 1
    assert L.gmm_host_digamma(None, None, C.c_longlong(0)) == 0
