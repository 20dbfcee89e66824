"""The restatement of gmm_em_multisample (tests/_multisample_ref.py) checked without a GPU: the reweight identity in float64,
the reduction to the pooled EM, and the float32 reweight against hand-computed cases."""
import numpy as np
import pytest

import _multisample_ref as ms
from conftest import random_spd_params


def _params(pkg, K, D, seed):
    """Random well-conditioned parameters with Rinv and constant formed by the host finalisation's rules."""
    rng = np.random.default_rng(seed)
    cl = random_spd_params(pkg, K, D, rng, spread=2.0)
    for k in range(K):
        R = cl.R[k].astype(np.float64)
        cl.Rinv[k] = np.linalg.inv(R).astype(np.float32)
        cl.constant[k] = np.float32(-0.5 * D * np.log(2 * np.pi) - 0.5 * np.linalg.slogdet(R)[1])
    cl.pi[:K] = (cl.N[:K] / cl.N[:K].sum()).astype(np.float32)
    X = rng.uniform(-3, 3, size=(3000, D))
    return cl, X, rng


@pytest.mark.parametrize("K,D,S", [(1, 3, 2), (5, 4, 3), (12, 6, 7)])
def test_reweight_of_pooled_estep_equals_per_sample_estep(pkg, K, D, S):
    cl, X, rng = _params(pkg, K, D, 10 * K + D)
    off = np.concatenate([[0], np.sort(rng.choice(np.arange(1, len(X)), S - 1, replace=False)), [len(X)]])
    pi = rng.dirichlet(np.ones(K), size=S)
    pooled = cl.pi[:K].astype(np.float64)
    r, lp = ms.estep(X, cl, K, np.log(pooled))
    r2, lnS = ms.reweight64(r, pi / pooled[None, :], off)
    rd, lpd = ms.estep_multi(X, cl, K, off, pi)
    np.testing.assert_allclose(r2, rd, rtol=0, atol=1e-12)
    np.testing.assert_allclose(lp + lnS, lpd, rtol=1e-12, atol=1e-12)


def test_equal_rows_are_the_pooled_estep(pkg):
    K, D, S = 6, 3, 4
    cl, X, _ = _params(pkg, K, D, 3)
    off = np.linspace(0, len(X), S + 1).astype(np.int64)
    pooled = cl.pi[:K].astype(np.float64)
    r, lp = ms.estep(X, cl, K, np.log(pooled))
    rd, lpd = ms.estep_multi(X, cl, K, off, np.tile(pooled, (S, 1)))
    np.testing.assert_allclose(rd, r, rtol=0, atol=1e-12)
    np.testing.assert_allclose(lpd, lp, rtol=1e-13)


def test_one_sample_is_the_pooled_em(pkg):
    """S = 1: pi_{1,k} = S0_k / n, the pooled pi is (float) N_k / sum N: the same EM up to float rounding of pi."""
    K, D = 4, 3
    rng = np.random.default_rng(5)
    centres = rng.uniform(-6, 6, size=(K, D))
    X = np.concatenate([c + rng.standard_normal((500 + 300 * i, D)) for i, c in enumerate(centres)])
    a, b = pkg.Clusters(K, D), pkg.Clusters(K, D)
    for cl in (a, b):
        cl.means[:K] = (centres + 0.5).astype(np.float32)
        cl.R[:K] = np.eye(D, dtype=np.float32)
        cl.Rinv[:K] = np.eye(D, dtype=np.float32)
        cl.constant[:K] = np.float32(-0.5 * D * np.log(2 * np.pi))
        cl.pi[:K] = np.float32(1.0 / K)
        cl.N[:K] = np.float32(len(X) / K)
        cl.avgvar[:K] = 0.01
    pi, ns, lls, resp = ms.em(pkg, X, a, K, [0, len(X)], None, 8)
    shift = np.zeros(D)
    r, lp = ms.estep(X, b, K, np.log(b.pi[:K].astype(np.float64)))
    pooled = [float(lp.sum())]
    for _ in range(8):
        pkg.host_finalize(ms.stats_from_resp(X, r, shift), shift, b, K)
        r, lp = ms.estep(X, b, K, np.log(b.pi[:K].astype(np.float64)))
        pooled.append(float(lp.sum()))
    np.testing.assert_allclose(lls, pooled, rtol=1e-7)
    np.testing.assert_allclose(resp, r, rtol=0, atol=1e-6)
    np.testing.assert_allclose(pi[0], b.pi[:K], rtol=1e-6)
    np.testing.assert_allclose(a.means[:K], b.means[:K], rtol=1e-6, atol=1e-6)
    assert ns[0] == len(X)
    assert np.all(np.diff(lls) >= -1e-9 * np.abs(lls[1:]))


def test_reweight32_hand_cases():
    f = np.float32
    # a tie: t = 0.5, 0.5, 0.5 -> S = 1.5 and three equal thirds
    m = np.array([[0.5], [0.25], [0.25]], np.float32)
    out, S, corr = ms.reweight32(m, np.array([[1, 2, 2]], np.float32), [0, 1])
    assert S[0] == f(1.5)
    assert np.all(out[:, 0] == f(0.5) / f(1.5))
    assert corr == np.log(1.5)
    # S is summed in increasing k: 1 + 3e-8 + 3e-8 stays 1 (the reverse order would round up to 1 + 2^-23)
    m = np.array([[1.0], [3e-8], [3e-8]], np.float32)
    out, S, _ = ms.reweight32(m, np.ones((1, 3), np.float32), [0, 1])
    assert S[0] == f(1.0) and f(f(3e-8) + f(3e-8)) + f(1.0) > f(1.0)
    assert out[0, 0] == f(1.0) and out[1, 0] == f(3e-8)
    # a 1-event sample between two others, rho at its bounds (N / n_s large, the 1e-10 floor over a pooled pi of 1)
    m = np.array([[0.9, 0.1, 0.6, 0.2], [0.1, 0.9, 0.4, 0.8]], np.float32)
    rho = np.array([[1.0, 1.0], [4096.0, f(1e-10)], [f(1e-10), 2.0]], np.float32)
    out, S, corr = ms.reweight32(m, rho, [0, 1, 2, 4])
    t1 = np.array([f(0.1) * f(4096.0), f(0.9) * f(1e-10)], np.float32)
    assert S[1] == t1[0] + t1[1]
    assert out[0, 1] == t1[0] / S[1] and out[1, 1] == t1[1] / S[1]
    t3 = np.array([f(0.2) * f(1e-10), f(0.8) * f(2.0)], np.float32)
    assert S[3] == t3[0] + t3[1] and out[0, 3] == t3[0] / S[3]
    assert S[0] == f(f(0.9) + f(0.1))
    np.testing.assert_allclose(corr, np.log(S.astype(np.float64)).sum(), rtol=0, atol=0)
    # weights scale the correction and the masses
    w = np.array([2.0, 0.0, 1.0, 3.0], np.float32)
    _, _, cw = ms.reweight32(m, rho, [0, 1, 2, 4], w)
    assert cw == float((w.astype(np.float64) * np.log(S.astype(np.float64))).sum())
    M, ns = ms.masses(out, [0, 1, 2, 4], 2, w)
    np.testing.assert_array_equal(ns, [2.0, 0.0, 4.0])
    o = out.astype(np.float64)
    np.testing.assert_allclose(M[2], o[:, 2] + 3.0 * o[:, 3], rtol=1e-15)


def test_rho_and_pi_update():
    pooled = np.array([0.5, 0.5, 0.0], np.float32)
    rho = ms.rho_of(np.array([[0.25, 0.75, 0.0]]), pooled)
    np.testing.assert_array_equal(rho, np.array([[0.5, 1.5, 0.0]], np.float32))
    pi = ms.update_pi(np.array([[3.0, 0.0, 1.0]]), np.array([4.0]))
    np.testing.assert_array_equal(pi, [[0.75, 1e-10, 0.25]])
