"""float64 numpy restatement of gmm_condition (include/gmm.h): the marginal and conditional parameters derived from the
float Rinv, constant, means and pi, rounded to float as the library rounds them, then the marginal log-sum-exp and the
moments of the conditional mixture in float64."""
import numpy as np
from scipy.special import logsumexp

LN2PI = np.log(2.0 * np.pi)


def split(D, obs):
    obs = np.asarray(obs, np.int64)
    return obs, np.setdiff1d(np.arange(D), obs)


def params(cl, K, obs):
    """Per cluster (mu_O, P_O, constant_O, mu_M, G, c) as float64 arrays holding float32 values."""
    D = cl.means.shape[1]
    obs, mis = split(D, obs)
    f32 = lambda a: np.asarray(a, np.float32).astype(np.float64)  # noqa: E731
    out = []
    for k in range(K):
        P = cl.Rinv[k].astype(np.float64)
        mu = cl.means[k].astype(np.float64)
        if mis.size == 0:
            out.append((mu, P, float(cl.constant[k]), np.zeros(0), np.zeros((0, D)), np.zeros(0)))
            continue
        S = 0.5 * (P + P.T)
        Smm, Smo, Soo = S[np.ix_(mis, mis)], S[np.ix_(mis, obs)], S[np.ix_(obs, obs)]
        L = np.linalg.cholesky(Smm)
        Z = np.linalg.solve(Smm, Smo)
        Po = Soo - Smo.T @ Z
        const = float(cl.constant[k]) + 0.5 * mis.size * LN2PI - np.sum(np.log(np.diag(L)))
        c = np.diag(np.linalg.inv(Smm))
        out.append((mu[obs], f32(0.5 * (Po + Po.T)), float(np.float32(const)), mu[mis], f32(-Z), f32(c)))
    return out


def condition(cl, K, obs, xo):
    """(logits [n][K], logp [n], mean [n][NM], var [n][NM], A [n][NM]) in float64; A = sum_k r_k (|mu_kM| + sum_j |G_kj dx_j|),
    the magnitude the float sums of the conditional means run over."""
    xo = np.asarray(xo, np.float64)
    n = xo.shape[0]
    pr = params(cl, K, obs)
    nm = pr[0][3].size
    L = np.empty((n, K))
    M = np.empty((K, n, nm))
    Ab = np.empty((K, n, nm))
    C = np.empty((K, nm))
    for k, (mo, Po, co, mm, G, c) in enumerate(pr):
        dx = xo - mo
        L[:, k] = np.log(np.float64(cl.pi[k])) + co - 0.5 * np.einsum("ni,ni->n", dx @ Po, dx)
        M[k] = mm + dx @ G.T
        Ab[k] = np.abs(mm) + np.abs(dx) @ np.abs(G).T
        C[k] = c
    lp = logsumexp(L, axis=1)
    r = np.exp(L - lp[:, None]).T                                  # [K][n]
    mean = np.einsum("kn,knd->nd", r, M)
    var = np.einsum("kn,knd->nd", r, C[:, None, :] + (M - mean[None]) ** 2)
    A = np.einsum("kn,knd->nd", r, Ab)
    return L, lp, mean, var, A
