"""gmm_combine's host side (no GPU needed): the restatement tests/_combine_ref.py against the defining formulas in float64,
gmm_host_combine_groups and gmm_host_combine_elbow against the restatement (and the elbow against np.polyfit), and every
argument error of the host calls."""
import ctypes as C

import numpy as np
import pytest

import _combine_ref as cr


def _tau(K, n, seed, w=False):
    rng = np.random.default_rng(seed)
    tau = rng.dirichlet(np.full(K, 0.3), size=n).T.astype(np.float32)
    tau[:, rng.random(n) < 0.1] = 0.0                                      # some events without memberships
    k = rng.integers(0, K)                                                   # exact zeros in a row that still sums to 1
    tau[k, :7] = 0.0
    tau[(k + 1) % K, :7] = 1.0 - (tau[:, :7].sum(axis=0) - tau[(k + 1) % K, :7])
    wv = rng.integers(0, 4, size=n).astype(np.float32) if w else None
    return tau, wv


@pytest.mark.parametrize("K,weighted", [(2, False), (5, False), (9, True), (12, False)])
def test_restatement_against_direct_formulas(K, weighted):
    tau, w = _tau(K, 700, 10 + K, weighted)
    n = tau.shape[1]
    wv = np.ones(n) if w is None else w.astype(np.float64)
    r = cr.combine(tau, w)
    members = {k: [k] for k in range(K)}
    for s in range(K - 1):
        live = sorted(members)
        rows = {a: cr.group_sum(tau, members[a]) for a in live}
        # every live pair by the direct formula; the chosen pair has the largest gain
        direct = {(a, b): float(np.sum(wv * cr.phi_direct(rows[a], rows[b]))) for i, a in enumerate(live) for b in live[i + 1:]}
        a, b = (int(v) for v in r["merges"][s])
        assert a < b and (a, b) in direct
        assert abs(r["gain"][s] - direct[(a, b)]) <= 1e-9 * max(1.0, abs(direct[(a, b)]))
        assert direct[(a, b)] >= max(direct.values()) - 1e-9 * max(1.0, max(direct.values()))
        assert r["mass"][s] == pytest.approx(float(np.sum(wv * (rows[a].astype(np.float64) + rows[b]))), rel=1e-6)
        # the entropy column at L = K - s clusters is the classification entropy of the grouping
        ent = -sum(float(np.sum(wv * cr.xlogx(rows[g]))) for g in live)
        assert r["entropy"][K - 1 - s] == pytest.approx(ent, rel=1e-5, abs=1e-6 * n)
        members[a] = sorted(members[a] + members.pop(b))
    assert abs(r["entropy"][0]) <= 1e-5 * n


def test_phi_is_cancellation_free():
    """phi's M h(m / M) form against the direct formula where it does not cancel, and its limits."""
    a = np.array([1.0, 0.5, 1e-3, 1e-20, 0.0, 0.3], np.float32)
    b = np.array([1.0, 0.25, 0.9, 0.999, 0.7, 0.0], np.float32)
    np.testing.assert_allclose(cr.phi(a[:3], b[:3]), cr.phi_direct(a[:3], b[:3]), rtol=1e-12)
    x = 1e-20
    assert cr.phi(a[3:4], b[3:4])[0] == pytest.approx(0.999 * float(np.float32(x) / np.float32(0.999)) * (1 - np.log(
        float(np.float32(x)) / float(np.float32(0.999)))), rel=1e-6)
    assert cr.phi(a[4:], b[4:]).tolist() == [0.0, 0.0]
    assert cr.phi(np.float32(1.0), np.float32(1.0)) == pytest.approx(2 * np.log(2.0), rel=1e-15)


def _merges(K, rng):
    """A random valid hierarchy."""
    live = list(range(K))
    out = []
    while len(live) > 1:
        i, j = sorted(rng.choice(len(live), 2, replace=False))
        a, b = live[i], live[j]
        out.append((a, b))
        live.remove(b)
    return np.array(out, np.int32).reshape(-1, 2)


@pytest.mark.parametrize("K", [1, 2, 3, 8, 65])
def test_groups_against_restatement(pkg, K):
    rng = np.random.default_rng(K)
    m = _merges(K, rng)
    for L in range(1, K + 1):
        got = pkg.host_combine_groups(m, K, L)
        ref = cr.groups(m, K, L)
        np.testing.assert_array_equal(got, ref)
        assert sorted(set(got.tolist())) == list(range(L))
        first = [int(np.flatnonzero(got == g)[0]) for g in range(L)]
        assert first == sorted(first)


def _polyfit_sse(x, y):
    x, y = np.asarray(x, np.float64), np.asarray(y, np.float64)
    if np.all(x == x[0]):
        return float(np.sum((y - y.mean()) ** 2))
    p = np.polyfit(x, y, 1)
    return float(np.sum((y - np.polyval(p, x)) ** 2))


@pytest.mark.parametrize("K,seed,with_x", [(3, 0, False), (4, 1, True), (10, 2, False), (40, 3, True), (130, 4, False)])
def test_elbow_against_restatement_and_polyfit(pkg, K, seed, with_x):
    rng = np.random.default_rng(seed)
    knee = int(rng.integers(2, K)) if K > 3 else 2
    L = np.arange(1, K + 1, dtype=np.float64)
    ent = np.where(L <= knee, 50.0 * (L - 1), 50.0 * (knee - 1) + 2.0 * (L - knee)) + rng.normal(0, 0.5, K)
    x = np.cumsum(rng.uniform(0.5, 2.0, K)) if with_x else None
    got = pkg.host_combine_elbow(ent, x)
    assert got == cr.elbow(ent, x)
    xs = L if x is None else x
    sse = [_polyfit_sse(xs[:c], ent[:c]) + _polyfit_sse(xs[c - 1:], ent[c - 1:]) for c in range(2, K)]
    tol = 1e-12 * K * float(np.max(ent ** 2))
    np.testing.assert_allclose(cr.elbow_sse(ent, x), sse, rtol=1e-7, atol=tol)
    assert abs(sse[got - 2] - min(sse)) <= tol
    if K > 4 and not with_x:                      # the knee is one in L, not in a random x
        assert abs(got - knee) <= 1


def test_elbow_ties_and_equal_x(pkg):
    # constant entropy: every change point fits exactly, the smallest c wins
    assert pkg.host_combine_elbow(np.full(6, 3.25)) == 2
    # two exact lines meeting at L = 4: c = 4 is the unique zero
    e = np.array([0.0, 4.0, 8.0, 12.0, 13.0, 14.0, 15.0])
    assert pkg.host_combine_elbow(e) == 4 == cr.elbow(e)
    # equal x on a segment: that segment uses its mean
    x = np.array([1.0, 1.0, 1.0, 2.0, 3.0, 4.0, 4.0])
    e = np.array([5.0, 6.0, 5.5, 4.0, 3.0, 2.5, 1.5])
    sse = [_polyfit_sse(x[:c], e[:c]) + _polyfit_sse(x[c - 1:], e[c - 1:]) for c in range(2, 7)]
    np.testing.assert_allclose(cr.elbow_sse(e, x), sse, atol=1e-12)
    assert sorted(sse)[1] - min(sse) > 0.01
    assert pkg.host_combine_elbow(e, x) == cr.elbow(e, x) == 2 + int(np.argmin(sse))
    # symmetric data: a tie between c = 3 and c = 4 within exact arithmetic goes to the smaller c
    e = np.array([0.0, 1.0, 2.0, 2.0, 1.0, 0.0])
    s = cr.elbow_sse(e)
    assert pkg.host_combine_elbow(e) == cr.elbow(e) == 2 + int(np.argmin(s))


def test_host_argument_errors(pkg):
    L = pkg.load_library()
    ARG = 1
    m = np.array([[0, 1], [0, 2]], np.int32)
    out = np.zeros(3, np.int32)
    p = lambda a: a.ctypes.data  # noqa: E731
    assert L.gmm_host_combine_groups(p(m), 3, 1, p(out)) == 0
    assert L.gmm_host_combine_groups(p(m), 3, 0, p(out)) == ARG                  # L < 1
    assert L.gmm_host_combine_groups(p(m), 3, 4, p(out)) == ARG                  # L > K
    assert L.gmm_host_combine_groups(p(m), 0, 1, p(out)) == ARG                  # K < 1
    assert L.gmm_host_combine_groups(p(m), 513, 1, p(out)) == ARG                # K > 512
    assert L.gmm_host_combine_groups(None, 3, 1, p(out)) == ARG                  # NULL merges, K >= 2
    assert L.gmm_host_combine_groups(None, 1, 1, p(out)) == 0                    # K = 1 needs none
    assert L.gmm_host_combine_groups(p(m), 3, 1, None) == ARG                    # NULL output
    for bad in ([[1, 0], [0, 2]], [[0, 1], [1, 2]], [[0, 0], [0, 2]], [[0, 3], [0, 1]], [[-1, 1], [0, 2]], [[0, 1], [0, 1]]):
        b = np.array(bad, np.int32)
        assert L.gmm_host_combine_groups(p(b), 3, 2, p(out)) == ARG, bad
    assert "merge" in L.gmm_last_error().decode()
    e = np.array([3.0, 1.0, 0.5, 0.2])
    Lo = C.c_int()
    assert L.gmm_host_combine_elbow(p(e), None, 4, C.byref(Lo)) == 0
    assert L.gmm_host_combine_elbow(p(e), None, 2, C.byref(Lo)) == ARG          # K < 3
    assert L.gmm_host_combine_elbow(None, None, 4, C.byref(Lo)) == ARG
    assert L.gmm_host_combine_elbow(p(e), None, 4, None) == ARG
    for v in (np.nan, np.inf):
        e2 = e.copy()
        e2[1] = v
        assert L.gmm_host_combine_elbow(p(e2), None, 4, C.byref(Lo)) == ARG
        x = np.arange(4.0)
        x[2] = v
        assert L.gmm_host_combine_elbow(p(e), p(x), 4, C.byref(Lo)) == ARG
    with pytest.raises(pkg.GmmError):
        pkg.host_combine_elbow([1.0, 0.0])
    with pytest.raises(pkg.GmmError):
        pkg.host_combine_groups(m, 3, 5)
