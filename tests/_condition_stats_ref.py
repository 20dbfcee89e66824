"""float64 numpy restatement of gmm_condition_stats (include/gmm.h): the expected full-D M-step statistics of events measured
on the dimensions O, from the per-cluster moments T0, T1, T2 of the observed coordinates about the centre and the
per-cluster regression of the missing dimensions on the observed ones, derived in double from the float Rinv."""
import numpy as np

import _condition_ref as cref


def regression(cl, K, obs):
    """Per cluster (G [NM][n_obs], C [NM][NM]) in float64: G = -S_MM^-1 S_MO, C = S_MM^-1, S = (P + P^T) / 2."""
    D = cl.means.shape[1]
    obs, mis = cref.split(D, obs)
    out = []
    for k in range(K):
        P = cl.Rinv[k].astype(np.float64)
        S = 0.5 * (P + P.T)
        Smm, Smo = S[np.ix_(mis, mis)], S[np.ix_(mis, obs)]
        C = np.linalg.inv(Smm)
        out.append((-C @ Smo, 0.5 * (C + C.T)))
    return out


def marginal_posterior(cl, K, obs, xo):
    """(memberships [K][n], logp [n]) under the marginal mixture of gmm_condition, in float64."""
    L, lp, _, _, _ = cref.condition(cl, K, obs, xo)
    return np.exp(L - lp[:, None]).T, lp


def pack(S0, S1, S2, ll=0.0):
    """Packed statistics [K * F + 1] from S0 [K], S1 [K][D], S2 [K][D][D] (host_math.h feat2 order)."""
    D = S1.shape[1]
    i, j = np.tril_indices(D)
    rows = [np.concatenate([[S0[k]], S1[k], S2[k][i, j]]) for k in range(len(S0))]
    return np.concatenate(rows + [[ll]])


def expected_stats(cl, K, obs, xo, memb, shift, ll=0.0):
    """The packed statistics gmm_condition_stats returns for the rows xo [n][n_obs] weighted by memb [K][n], about shift, by
    the identity of gmm.h: T0, T1 and T2 of y = x_O - s_O, then per cluster
      S1_M = b T0 + G T1,  S2_MO = b T1^T + G T2,  S2_MM = T0 (b b^T + C) + b u^T + u b^T + G T2 G^T,  u = G T1,
    with b = (mu_M - s_M) - G (mu_O - s_O)."""
    D = cl.means.shape[1]
    obs, mis = cref.split(D, obs)
    shift = np.asarray(shift, np.float64)
    y = np.asarray(xo, np.float32).astype(np.float64) - shift[obs]
    g = np.asarray(memb, np.float32).astype(np.float64)
    S0 = np.zeros(K)
    S1 = np.zeros((K, D))
    S2 = np.zeros((K, D, D))
    reg = regression(cl, K, obs) if mis.size else None
    for k in range(K):
        T0 = g[k].sum()
        T1 = g[k] @ y
        T2 = (g[k][:, None] * y).T @ y
        S0[k] = T0
        S1[k, obs] = T1
        S2[k][np.ix_(obs, obs)] = T2
        if mis.size == 0:
            continue
        G, C = reg[k]
        mu = cl.means[k].astype(np.float64)
        b = (mu[mis] - shift[mis]) - G @ (mu[obs] - shift[obs])
        u = G @ T1
        S1[k, mis] = b * T0 + u
        smo = np.outer(b, T1) + G @ T2
        S2[k][np.ix_(mis, obs)] = smo
        S2[k][np.ix_(obs, mis)] = smo.T
        S2[k][np.ix_(mis, mis)] = T0 * (np.outer(b, b) + C) + np.outer(b, u) + np.outer(u, b) + G @ T2 @ G.T
    return pack(S0, S1, S2, ll)


def brute_force_stats(cl, K, obs, xo, memb, shift):
    """The same statistics event by event: each event completed per cluster by E[x_M | x_O, k], and C_k added to the
    second moment of its missing block."""
    D = cl.means.shape[1]
    obs, mis = cref.split(D, obs)
    shift = np.asarray(shift, np.float64)
    x = np.asarray(xo, np.float32).astype(np.float64)
    g = np.asarray(memb, np.float32).astype(np.float64)
    reg = regression(cl, K, obs) if mis.size else None
    S0 = np.zeros(K)
    S1 = np.zeros((K, D))
    S2 = np.zeros((K, D, D))
    for k in range(K):
        mu = cl.means[k].astype(np.float64)
        for e in range(len(x)):
            full = np.empty(D)
            full[obs] = x[e]
            extra = np.zeros((D, D))
            if mis.size:
                G, C = reg[k]
                full[mis] = mu[mis] + G @ (x[e] - mu[obs])
                extra[np.ix_(mis, mis)] = C
            d = full - shift
            S0[k] += g[k, e]
            S1[k] += g[k, e] * d
            S2[k] += g[k, e] * (np.outer(d, d) + extra)
    return pack(S0, S1, S2)
