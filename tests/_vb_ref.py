"""float64 numpy restatement of gmm_vb_em / gmm_host_vb_finalize (include/gmm.h): sklearn's BayesianGaussianMixture with
covariance_type='full', driven by the library's packed statistics and parameter set.

``rounding=True`` adds the library's float rounding points (N, means, R, pi, constant and Rinv stored as float32; the E-step
and the constant use the float R), ``rounding=False`` is sklearn's arithmetic throughout."""
import numpy as np
from scipy.special import digamma, gammaln

DP, DIRICHLET = 0, 1
EPS10 = 10 * np.finfo(np.float64).eps
FLT_MIN = np.float32(np.finfo(np.float32).tiny)


def feat_index(D):
    """(i, j) of the packed second-moment features, i >= j row by row."""
    return [(i, j) for i in range(D) for j in range(i + 1)]


def default_moments(X, w=None):
    """The default m0 / Psi0: the (weighted) mean and np.cov(X.T) (denominator sum w - 1)."""
    X = np.asarray(X, np.float64)
    w = np.ones(len(X)) if w is None else np.asarray(w, np.float64)
    W = w.sum()
    m = (w[:, None] * X).sum(0) / W
    d = X - m
    return m, np.atleast_2d((w[:, None] * d).T @ d / (W - 1.0))


def prior(K, D, prior_type=DP, gamma0=None, beta0=None, nu0=None, m0=None, psi0=None, reg=None):
    return dict(type=prior_type, gamma0=1.0 / K if gamma0 is None else gamma0, beta0=1.0 if beta0 is None else beta0,
                nu0=float(D) if nu0 is None else nu0, m0=np.asarray(m0, np.float64), psi0=np.asarray(psi0, np.float64),
                reg=1e-6 if reg is None else reg)


def stats_from_resp(X, resp, shift, w=None):
    """The packed statistics [K*F + 1] about `shift` in float64 (resp [n][K]; the last slot 0)."""
    X = np.asarray(X, np.float64)
    n, D = X.shape
    K = resp.shape[1]
    g = resp * (1.0 if w is None else np.asarray(w, np.float64)[:, None])
    y = X - shift
    F = 1 + D + D * (D + 1) // 2
    st = np.zeros(K * F + 1)
    ii, jj = np.array(feat_index(D), dtype=np.int64).reshape(-1, 2).T
    for k in range(K):
        row = st[k * F:(k + 1) * F]
        row[0] = g[:, k].sum()
        row[1:1 + D] = g[:, k] @ y
        row[1 + D:] = ((g[:, k, None] * y).T @ y)[ii, jj]
    return st


def m_step(stats, shift, K, D, pr, rounding=True):
    """The VB M-step from packed statistics: the posterior, the parameter set and the bound without its entropy."""
    F = 1 + D + D * (D + 1) // 2
    shift = np.asarray(shift, np.float64)
    st = np.asarray(stats, np.float64)[:K * F].reshape(K, F)
    S0, S1 = st[:, 0], st[:, 1:1 + D]
    S2 = np.zeros((K, D, D))
    for f, (i, j) in enumerate(feat_index(D)):
        S2[:, i, j] = S2[:, j, i] = st[:, 1 + D + f]
    nk = S0 + EPS10
    xk = (S0[:, None] * shift + S1) / nk[:, None]
    dd = xk - shift
    Q = S2 - S1[:, :, None] * dd[:, None, :] - dd[:, :, None] * S1[:, None, :] + S0[:, None, None] * dd[:, :, None] * dd[:, None, :]
    nksk = Q + nk[:, None, None] * pr["reg"] * np.eye(D)
    return posterior(nk, xk, nksk, D, pr, rounding)


def m_step_resp(X, resp, pr, w=None, rounding=False):
    """The same from events and responsibilities, in sklearn's own form (_estimate_gaussian_parameters)."""
    X = np.asarray(X, np.float64)
    g = resp * (1.0 if w is None else np.asarray(w, np.float64)[:, None])
    nk = g.sum(0) + EPS10
    xk = (g.T @ X) / nk[:, None]
    D = X.shape[1]
    sk = np.empty((len(nk), D, D))
    for k in range(len(nk)):
        d = X - xk[k]
        sk[k] = (g[:, k] * d.T) @ d / nk[k]
        sk[k].flat[::D + 1] += pr["reg"]
    return posterior(nk, xk, nk[:, None, None] * sk, D, pr, rounding)


def posterior(nk, xk, nksk, D, pr, rounding):
    K = len(nk)
    beta = pr["beta0"] + nk
    m = (pr["beta0"] * pr["m0"] + nk[:, None] * xk) / beta[:, None]
    nu = pr["nu0"] + nk
    diff = xk - pr["m0"]
    C = (pr["psi0"] + nksk + (nk * pr["beta0"] / beta)[:, None, None] * diff[:, :, None] * diff[:, None, :]) / nu[:, None, None]
    if pr["type"] == DP:
        a = 1.0 + nk
        b = pr["gamma0"] + np.hstack((np.cumsum(nk[::-1])[-2::-1], 0))
        ds = digamma(a + b)
        elog = digamma(a) - ds + np.hstack((0, np.cumsum(digamma(b) - ds)[:-1]))
        wts = a / (a + b) * np.hstack((1, np.cumprod(b / (a + b))[:-1]))
        log_norm_weight = -np.sum(gammaln(a) + gammaln(b) - gammaln(a + b))
        wc = np.stack([a, b])
    else:
        a = pr["gamma0"] + nk
        elog = digamma(a) - digamma(a.sum())
        wts = a.copy()
        log_norm_weight = gammaln(a.sum()) - gammaln(a).sum()
        wc = a
    wts = wts / wts.sum()
    i = np.arange(D)[:, None]
    sum_psi = digamma(0.5 * (nu - i)).sum(0)
    sum_lg = gammaln(0.5 * (nu - i)).sum(0)
    half_ld = np.array([np.linalg.slogdet(C[k])[1] / 2 for k in range(K)])
    log_wishart = -(nu * (-half_ld - 0.5 * D * np.log(nu)) + nu * D * 0.5 * np.log(2.0) + sum_lg)
    bound_par = -log_wishart.sum() - log_norm_weight - 0.5 * D * np.log(beta).sum()
    p = dict(nk=nk, xk=xk, beta=beta, m=m, nu=nu, C=C, weight_concentration=wc, weights=wts, elog=elog, bound_par=bound_par,
             type=pr["type"])
    if rounding:
        R = C.astype(np.float32)
        Rd = R.astype(np.float64)
        Rd = 0.5 * (Rd + np.swapaxes(Rd, 1, 2))
        half_ld_R = np.array([np.linalg.slogdet(Rd[k])[1] / 2 for k in range(K)])
        pi = np.maximum(wts.astype(np.float32), FLT_MIN)
        p.update(R=R, Rinv=np.linalg.inv(Rd).astype(np.float32), means=m.astype(np.float32), N=nk.astype(np.float32), pi=pi)
        Rq, ldq, mq = Rd, half_ld_R, m.astype(np.float32).astype(np.float64)
    else:
        pi = wts
        Rq, ldq, mq = C, half_ld, m
    offset = -0.5 * D * np.log(2 * np.pi) - ldq - 0.5 * D * np.log(nu) + 0.5 * (D * np.log(2.0) + sum_psi) - 0.5 * D / beta
    p["log_weight"] = offset + elog                       # constant + ln pi of the E-step
    p["constant"] = (p["log_weight"] - np.log(np.asarray(pi, np.float64))).astype(np.float32 if rounding else np.float64)
    p["Pq"], p["mq"] = np.linalg.inv(Rq), mq
    return p


def log_prob(X, p):
    """sklearn's _estimate_weighted_log_prob under the parameter set: [n][K]."""
    X = np.asarray(X, np.float64)
    q = np.empty((len(X), len(p["mq"])))
    for k in range(len(p["mq"])):
        d = X - p["mq"][k]
        q[:, k] = ((d @ p["Pq"][k]) * d).sum(1)
    return p["log_weight"][None] - 0.5 * q


def e_step(X, p):
    """(log_resp [n][K], log_prob_norm [n])."""
    lp = log_prob(X, p)
    mx = lp.max(1, keepdims=True)
    norm = mx[:, 0] + np.log(np.exp(lp - mx).sum(1))
    return lp - norm[:, None], norm


def entropy_sum(resp, w=None):
    """sum_n w_n sum_k g ln g (0 ln 0 = 0), resp [n][K]."""
    r = np.asarray(resp, np.float64)
    t = np.where(r > 0, r * np.log(np.where(r > 0, r, 1.0)), 0.0).sum(1)
    return float(t.sum() if w is None else (np.asarray(w, np.float64) * t).sum())


def fit(X, resp0, pr, min_iters, max_iters, tol, w=None, rounding=True):
    """gmm_vb_em's loop from the responsibilities resp0 [n][K] of the first E-step.
    Returns (params, lower bound, bounds, iters, converged, final resp [n][K])."""
    shift = np.zeros(X.shape[1])
    K, D = resp0.shape[1], X.shape[1]
    p = m_step(stats_from_resp(X, resp0, shift, w), shift, K, D, pr, rounding)
    lb, lbs, conv, it = -np.inf, [], False, 0
    for i in range(1, max_iters + 1):
        log_resp, _ = e_step(X, p)
        resp = np.exp(log_resp)
        p = m_step(stats_from_resp(X, resp, shift, w), shift, K, D, pr, rounding)
        prev, lb = lb, -entropy_sum(resp, w) + p["bound_par"]
        lbs.append(lb)
        it = i
        if i >= min_iters and abs(lb - prev) < tol:
            conv = True
            break
    log_resp, _ = e_step(X, p)
    return p, lb, np.array(lbs), it, conv, np.exp(log_resp)
