"""float64 numpy restatement of gmm_modes / gmm_mode_labels (include/gmm.h): the parameters, the step-form fixed point of
Carreira-Perpinan (2000), the stop rule, the dedup of gmm_modes and the label rule of gmm_mode_labels."""
import numpy as np

CONVERGED, UNCONVERGED, NOT_FINITE = 1, 2, 3


def params(means, Rinv, R, constant, pi):
    """The derived parameters of the components with pi > 0, in double: centre c (rounded through float), mu - c, S,
    const + ln pi, 1 / sigma."""
    pi = np.asarray(pi, np.float64)
    live = np.nonzero(pi > 0)[0]
    means = np.asarray(means, np.float64)[live]
    P = np.asarray(Rinv, np.float64)[live]
    Rd = np.asarray(R, np.float64)[live]
    w = pi[live]
    c = (w[:, None] * means).sum(0).astype(np.float32).astype(np.float64)
    sigma = np.sqrt((w[:, None] * np.diagonal(Rd, axis1=1, axis2=2)).sum(0))
    return dict(live=live, c=c, mu=means - c, S=0.5 * (P + np.swapaxes(P, 1, 2)),
                lc=np.asarray(constant, np.float64)[live] + np.log(w), inv_sigma=1.0 / sigma)


def _terms(p, x):
    dx = x[:, None, :] - p["mu"][None]                            # [n][K][D]
    v = np.einsum("kij,nkj->nki", p["S"], dx)
    l = p["lc"][None] - 0.5 * np.einsum("nki,nki->nk", dx, v)
    m = l.max(1, keepdims=True)
    lp = m[:, 0] + np.log(np.exp(l - m).sum(1))
    r = np.exp(l - lp[:, None])
    return v, r, lp


def logp(p, x):
    return _terms(p, np.atleast_2d(x))[2]


def grad_hess(p, x):
    """Gradient [n][D] and Hessian [n][D][D] of ln p at x (relative coordinates)."""
    v, r, _ = _terms(p, np.atleast_2d(x))
    g = -np.einsum("nk,nki->ni", r, v)
    H = np.einsum("nk,nki,nkj->nij", r, v, v) - np.einsum("nk,kij->nij", r, p["S"]) - g[:, :, None] * g[:, None, :]
    return g, H


def is_max(p, x):
    _, H = grad_hess(p, x)
    return np.array([np.all(np.linalg.eigvalsh(-h) > 0) for h in H])


def step(p, x):
    v, r, lp = _terms(p, x)
    g = -np.einsum("nk,nki->ni", r, v)
    A = np.einsum("nk,kij->nij", r, p["S"])
    return np.linalg.solve(A, g[..., None])[..., 0], lp


def climb(p, x0, max_iter=500, tol=1e-5, trace=False):
    """Each point's ascent: (endpoints, iters, status[, logp per iteration of each point as a list of arrays])."""
    x = np.array(x0, np.float64)
    n = len(x)
    it = np.zeros(n, np.int64)
    st = np.where(np.all(np.isfinite(x), 1), 0, NOT_FINITE)
    hist = [logp(p, np.nan_to_num(x))] if trace else None
    for _ in range(max_iter):
        a = np.nonzero(st == 0)[0]
        if a.size == 0:
            break
        d, _ = step(p, x[a])
        # below tol sigma_d, or within 2 float ulps of the coordinate (relative to the centre) before the step
        done = np.all(np.abs(d) * p["inv_sigma"] < np.maximum(tol, np.abs(x[a]) * 2.0 ** -22 * p["inv_sigma"]), 1)
        x[a] += d
        it[a] += 1
        st[a[done]] = CONVERGED
        st[a[~done & (it[a] >= max_iter)]] = UNCONVERGED
        if trace:
            hist.append(logp(p, np.nan_to_num(x)))
    x[st == NOT_FINITE] = np.nan
    return (x, it, st, hist) if trace else (x, it, st)


def rho(p, a, b):
    return np.max(np.abs(np.asarray(a) - np.asarray(b)) * p["inv_sigma"], -1)


def dedup(p, ends, st, merge_tol):
    """gmm_modes' dedup in start order: (modes [M][D] relative, mode of each start (-1 unconverged))."""
    modes, cm = [], np.full(len(ends), -1)
    for i, (e, s) in enumerate(zip(ends, st)):
        if s != CONVERGED:
            continue
        j = next((j for j, m in enumerate(modes) if rho(p, e, m) <= merge_tol), None)
        if j is None:
            modes.append(np.array(e))
            j = len(modes) - 1
        cm[i] = j
    return np.array(modes).reshape(-1, len(p["c"])), cm


def labels(p, ends, st, modes, merge_tol):
    """gmm_mode_labels' rule: the listed mode of smallest rho <= merge_tol (ties to the lower index), -2 none, -1 not
    converged."""
    out = np.full(len(ends), -1)
    for i, (e, s) in enumerate(zip(ends, st)):
        if s != CONVERGED:
            continue
        r = rho(p, e[None], modes)
        ok = np.nonzero(r <= merge_tol)[0]
        out[i] = -2 if ok.size == 0 else ok[np.argmin(r[ok])]
    return out
