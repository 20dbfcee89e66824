"""Restatement of gmm_combine's semantics (include/gmm.h) in numpy: group sums in float32 (left to right in increasing
component order, as the kernels add them), phi in float64, events summed in float64, the greedy entropy hierarchy with its
tie rule, the entropy and mass columns, the labels of a grouping, the groups of a level and the elbow.

tau is float32 [K][n] (the engine's own memberships), w float [n] or None."""
import numpy as np


def group_sum(tau, members):
    """Float32 sum of the rows `members` (increasing), added left to right; an empty group is 0."""
    if len(members) == 0:
        return np.zeros(tau.shape[1], np.float32)
    v = tau[members[0]].astype(np.float32, copy=True)
    for k in members[1:]:
        v = (v + tau[k]).astype(np.float32)
    return v


def phi(a, b):
    """(a+b) ln(a+b) - a ln a - b ln b in float64 of float inputs, as M h(m / M) (no cancellation); 0 where m = 0."""
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    M, m = np.maximum(a, b), np.minimum(a, b)
    out = np.zeros(np.broadcast(a, b).shape)
    pos = m > 0
    r = m[pos] / M[pos]
    out[pos] = M[pos] * ((1.0 + r) * np.log1p(r) - r * np.log(r))
    return out


def phi_direct(a, b):
    """The defining formula, float64, 0 ln 0 = 0 (cancels where one argument dominates: for checking only)."""
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    return xlogx(a + b) - xlogx(a) - xlogx(b)


def xlogx(x):
    x = np.asarray(x, np.float64)
    out = np.zeros_like(x)
    pos = x > 0
    out[pos] = x[pos] * np.log(x[pos])
    return out


def _weights(w, n):
    return np.ones(n) if w is None else np.asarray(w, np.float64)


def gain(ta, tb, w=None, chunk=1 << 20):
    """sum_n w_n phi(ta, tb), chunked."""
    wv = _weights(w, ta.shape[0])
    s = 0.0
    for i in range(0, ta.shape[0], chunk):
        s += float(np.dot(wv[i:i + chunk], phi(ta[i:i + chunk], tb[i:i + chunk])))
    return s


def entropy(tau, w=None, chunk=1 << 18):
    """-sum_n w_n sum_k tau ln tau in float64 (0 ln 0 = 0)."""
    K, n = tau.shape
    wv = _weights(w, n)
    s = 0.0
    for i in range(0, n, chunk):
        s += float(np.dot(xlogx(tau[:, i:i + chunk]).sum(axis=0), wv[i:i + chunk]))
    return -s


def combine(tau, w=None):
    """The hierarchy: dict(merges [K-1][2], gain [K-1], entropy [K], mass [K-1], gap [K-1]) where gap[s] is the relative
    distance (g1 - g2) / g1 between the two largest live gains of step s (inf when there is one pair, nan when g1 = 0)."""
    tau = np.asarray(tau, np.float32)
    K, n = tau.shape
    wv = _weights(w, n)
    mk = np.array([float(np.dot(wv, tau[k].astype(np.float64))) for k in range(K)])
    members = {k: [k] for k in range(K)}
    rows = {k: tau[k] for k in range(K)}
    g = {}
    for a in range(K):
        for b in range(a + 1, K):
            g[(a, b)] = gain(rows[a], rows[b], w)
    live = list(range(K))
    merges, gains, mass, gaps = [], [], [], []
    for s in range(K - 1):
        best, second = None, None
        for i, a in enumerate(live):
            for b in live[i + 1:]:
                v = g[(a, b)]
                if best is None or v > best[0]:
                    best, second = (v, a, b), best
                elif second is None or v > second[0]:
                    second = (v, a, b)
        v, a, b = best
        merges.append((a, b))
        gains.append(v)
        if second is None:
            gaps.append(np.inf)
        else:
            gaps.append((v - second[0]) / v if v > 0 else np.nan)
        mass.append(sum(mk[k] for k in members[a]) + sum(mk[k] for k in members[b]))
        members[a] = sorted(members[a] + members[b])
        del members[b], rows[b]
        live.remove(b)
        rows[a] = group_sum(tau, members[a])
        if s < K - 2:
            for h in live:
                if h != a:
                    g[(min(a, h), max(a, h))] = gain(rows[a], rows[h], w)
    ent = np.zeros(K)
    ent[K - 1] = entropy(tau, w)
    for L in range(K, 1, -1):
        ent[L - 2] = ent[L - 1] - gains[K - L]
    return dict(merges=np.array(merges, np.int32).reshape(-1, 2), gain=np.array(gains), entropy=ent, mass=np.array(mass),
                gap=np.array(gaps))


def groups(merges, K, L):
    """Cluster of each component at level L: the first K-L merges applied, clusters numbered by smallest component."""
    rep = list(range(K))
    for a, b in np.asarray(merges).reshape(-1, 2)[:K - L]:
        rep[int(b)] = int(a)

    def root(k):
        while rep[k] != k:
            k = rep[k]
        return k
    label, out = {}, np.empty(K, np.int32)
    for k in range(K):
        r = root(k)
        label.setdefault(r, len(label))
        out[k] = label[r]
    return out


def labels(tau, group, G):
    """argmax over g of the float32 group sums (lowest g on ties, NaN sums skipped, -1 when all are NaN) and that sum."""
    tau = np.asarray(tau, np.float32)
    n = tau.shape[1]
    sums = np.stack([group_sum(tau, [k for k in range(len(group)) if group[k] == g]) for g in range(G)])
    lab = np.full(n, -1, np.int32)
    best = np.full(n, np.nan, np.float32)
    for g in range(G):
        v = sums[g]
        take = ~np.isnan(v) & ((lab < 0) | (v > best))
        lab[take] = g
        best[take] = v[take]
    return lab, best


def _sse(x, y):
    """Residual sum of squares of the least-squares line (the mean when every x is equal): centred sums in index order."""
    m = len(x)
    sx = sy = 0.0
    for i in range(m):
        sx += x[i]
        sy += y[i]
    mx, my = sx / m, sy / m
    sxx = sxy = 0.0
    for i in range(m):
        sxx += (x[i] - mx) * (x[i] - mx)
        sxy += (x[i] - mx) * (y[i] - my)
    beta = sxy / sxx if sxx > 0.0 else 0.0
    sse = 0.0
    for i in range(m):
        r = (y[i] - my) - beta * (x[i] - mx)
        sse += r * r
    return sse


def elbow_sse(entropy_, x=None):
    """Total SSE per change point c = 2 .. K-1 (index c - 2)."""
    y = [float(v) for v in entropy_]
    K = len(y)
    xs = [float(i + 1) for i in range(K)] if x is None else [float(v) for v in x]
    return np.array([_sse(xs[:c], y[:c]) + _sse(xs[c - 1:], y[c - 1:]) for c in range(2, K)])


def elbow(entropy_, x=None):
    """The change point: the c of the smallest total SSE, the smaller c on ties."""
    s = elbow_sse(entropy_, x)
    best = 0
    for i in range(1, len(s)):
        if s[i] < s[best]:
            best = i
    return best + 2
