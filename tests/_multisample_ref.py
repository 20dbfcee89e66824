"""numpy restatement of gmm_em_multisample (include/gmm.h): EM over samples with shared components and per-sample mixing
weights pi_{s,k}.  The E-step with per-sample log-weights is float64; the reweight of the pooled memberships is the
library's float32 arithmetic bit for bit; the shared update is the library's own host finalisation (gmm_host_finalize,
no GPU needed)."""
import numpy as np

from _vb_ref import stats_from_resp

PI_FLOOR = 1e-10


def sample_of(offsets, n):
    """The sample index of each of the n events: [n] int."""
    off = np.asarray(offsets, np.int64)
    return np.repeat(np.arange(off.size - 1), np.diff(off))[:n]


def log_dens(X, cl, K):
    """constant_k - 1/2 (x - mu_k)^T Rinv_k (x - mu_k) in float64 from the stored float parameters: [n][K]."""
    X = np.asarray(X, np.float64)
    out = np.empty((len(X), K))
    for k in range(K):
        d = X - np.asarray(cl.means[k], np.float64)
        out[:, k] = float(cl.constant[k]) - 0.5 * ((d @ np.asarray(cl.Rinv[k], np.float64)) * d).sum(1)
    return out


def estep(X, cl, K, logw):
    """E-step with log-weights logw ([K] or [n][K]): (resp [n][K], ln p [n])."""
    lp = log_dens(X, cl, K) + logw
    mx = lp.max(1, keepdims=True)
    norm = mx[:, 0] + np.log(np.exp(lp - mx).sum(1))
    return np.exp(lp - norm[:, None]), norm


def estep_multi(X, cl, K, offsets, pi):
    """The model's E-step: sample s's events under ln pi[s] (pi [S][K] float64)."""
    with np.errstate(divide="ignore"):
        logw = np.log(np.asarray(pi, np.float64))[sample_of(offsets, len(X))]
    return estep(X, cl, K, logw)


def reweight64(resp, rho, offsets):
    """float64 reweight of pooled responsibilities resp [n][K]: (r' [n][K], ln S [n])."""
    t = resp * np.asarray(rho, np.float64)[sample_of(offsets, len(resp))]
    S = t.sum(1)
    return t / S[:, None], np.log(S)


def rho_of(pi, pooled_pi):
    """rho_{s,k} = (float)(pi_{s,k} / (double)pi_k), 0 where pi_k = 0: [S][K] float32."""
    p = np.asarray(pooled_pi, np.float32).astype(np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.asarray(pi, np.float64) / p[None, :]
    return np.where(p[None, :] > 0, r, 0.0).astype(np.float32)


def reweight32(memb, rho, offsets, w=None):
    """The reweight pass on the stored memberships memb [>= K][n] float32 (K = rho's columns), bit for bit:
    t_k = r_k rho_{s,k}, S = t_0 + t_1 + ... in increasing k, r'_k = t_k / S, all float32 with one rounding each.
    Returns (r' [K][n] float32, S [n] float32, sum_n w_n log((double)S))."""
    rho = np.asarray(rho, np.float32)
    K = rho.shape[1]
    n = memb.shape[1]
    r = np.asarray(memb[:K], np.float32)
    rs = rho[sample_of(offsets, n)].T                       # [K][n]
    t = r * rs
    S = t[0].copy()
    for k in range(1, K):
        S = S + t[k]
    out = t / S[None, :]
    wd = np.ones(n) if w is None else np.asarray(w, np.float64)
    with np.errstate(divide="ignore"):
        corr = float((wd * np.log(S.astype(np.float64))).sum())
    return out, S, corr


def masses(memb, offsets, K, w=None):
    """M [S][K] = sum_{n in s} w_n memb[k][n] and n_s [S] = sum_{n in s} w_n, in float64."""
    off = np.asarray(offsets, np.int64)
    S = off.size - 1
    wd = np.ones(memb.shape[1]) if w is None else np.asarray(w, np.float64)
    g = np.asarray(memb[:K], np.float64) * wd[None, :]
    M = np.stack([g[:, off[s]:off[s + 1]].sum(1) for s in range(S)])
    ns = np.array([wd[off[s]:off[s + 1]].sum() for s in range(S)])
    return M, ns


def update_pi(M, ns):
    """pi_{s,k} = max(M_{s,k} / n_s, 1e-10): floored, not renormalised."""
    return np.maximum(M / ns[:, None], PI_FLOOR)


def em(pkg, X, cl, K, offsets, pi0, iters, w=None):
    """`iters` iterations of the model's EM in float64 from the parameter set cl (a pkg.Clusters, updated in place through
    gmm_host_finalize) and the weights pi0 [S][K] of the start (None: the pooled pi).
    Returns (pi [S][K] of the last E-step, n_s, log-likelihoods [iters + 1], r' [n][K] of the last E-step)."""
    off = np.asarray(offsets, np.int64)
    S = off.size - 1
    pi = np.tile(np.asarray(cl.pi[:K], np.float64), (S, 1)) if pi0 is None else np.asarray(pi0, np.float64) / np.sum(pi0, 1, keepdims=True)
    wd = np.ones(len(X)) if w is None else np.asarray(w, np.float64)
    resp, lp = estep_multi(X, cl, K, off, pi)
    lls = [float((wd * lp).sum())]
    shift = np.zeros(cl.D)
    for _ in range(iters):
        M, ns = masses(resp.T, off, K, w)
        pkg.host_finalize(stats_from_resp(X, resp, shift, w), shift, cl, K)
        pi = update_pi(M, ns)
        resp, lp = estep_multi(X, cl, K, off, pi)
        lls.append(float((wd * lp).sum()))
    _, ns = masses(resp.T, off, K, w)
    return pi, ns, np.array(lls), resp
