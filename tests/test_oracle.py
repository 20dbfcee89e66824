"""CPU tests of the oracle itself (oracle/gmm_oracle.c): invariants, agreement of
the FP32 (reference arithmetic) and FP64 builds, an independent cross-check
against scikit-learn, and the golden fixtures produced by the unmodified
reference on an H100 (tests/golden/, when present)."""
import os

import numpy as np
import pytest

from conftest import random_spd_params

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def small_problem(pkg, N=3000, D=4, K=5, seed=3):
    ev = pkg.synth.make_blobs(N, D, K, seed=seed)
    return ev


def test_invert_matches_numpy(oracle64):
    rng = np.random.default_rng(0)
    for n in (1, 2, 3, 8, 24, 32):
        A = rng.standard_normal((n, n))
        M = (A @ A.T / n + 0.5 * np.eye(n)).astype(np.float32)
        inv, ld = oracle64.invert(M, use_log10=False)
        np.testing.assert_allclose(inv, np.linalg.inv(M.astype(np.float64)), rtol=2e-3, atol=2e-4)
        assert abs(ld - np.linalg.slogdet(M.astype(np.float64))[1]) < 1e-3 * max(1, n)
        _, ld10 = oracle64.invert(M, use_log10=True)      # quirk Q3: invert_cpu returns log10
        if n > 1:
            assert abs(ld10 - ld / np.log(10)) < 1e-3


def test_seed_semantics(pkg, oracle64):
    ev = small_problem(pkg, N=1001, D=3, K=4)
    K = 4
    cl = pkg.Clusters(K, 3, ev.shape[0])
    oracle64.seed(ev, K, cl)
    seed = np.float32(ev.shape[0] - 1.0) / np.float32(K - 1.0)
    for k in range(K):
        np.testing.assert_array_equal(cl.means[k], ev[int(np.float32(k) * seed)])
        np.testing.assert_array_equal(cl.R[k], np.eye(3, dtype=np.float32))
        np.testing.assert_array_equal(cl.Rinv[k], np.eye(3, dtype=np.float32))
    assert np.all(cl.N == ev.shape[0] // K)                 # integer division, gaussian.cu:118
    np.testing.assert_allclose(cl.pi, 1.0 / K, rtol=1e-6)
    var = (ev.astype(np.float64) ** 2).mean(0) - ev.astype(np.float64).mean(0) ** 2
    np.testing.assert_allclose(cl.avgvar, var.mean() / 1e3, rtol=1e-5)
    np.testing.assert_allclose(cl.constant, -3 * 0.5 * np.log(2 * np.pi), rtol=1e-6)


def test_estep_invariants_and_f32_f64(pkg, oracle64, oracle32):
    ev = small_problem(pkg)
    N, D = ev.shape
    K = 5
    rng = np.random.default_rng(1)
    out = {}
    for name, orc in (("f64", oracle64), ("f32", oracle32)):
        cl = random_spd_params(pkg, K, D, rng=np.random.default_rng(1))
        cl.memberships = np.zeros((K, N), np.float32)
        orc.constants(cl, K)
        ll = orc.estep(orc.transpose(ev), cl, K)
        np.testing.assert_allclose(cl.memberships.sum(0), 1.0, atol=5e-6)
        assert np.all(cl.memberships >= 0)
        out[name] = (ll, cl.memberships.copy())
    assert abs(out["f32"][0] - out["f64"][0]) < 1e-5 * abs(out["f64"][0])
    np.testing.assert_allclose(out["f32"][1], out["f64"][1], rtol=2e-4, atol=1e-6)


def test_mstep_invariants(pkg, oracle64):
    ev = small_problem(pkg)
    N, D = ev.shape
    K = 5
    cl = random_spd_params(pkg, K, D, np.random.default_rng(2))
    cl.memberships = np.zeros((K, N), np.float32)
    oracle64.constants(cl, K)
    soa = oracle64.transpose(ev)
    oracle64.estep(soa, cl, K)
    oracle64.mstep(soa, cl, K)
    assert abs(cl.N.sum() - N) < 1e-3 * N
    for k in range(K):
        np.testing.assert_allclose(cl.R[k], cl.R[k].T, atol=0)      # mirrored exactly
        assert np.all(np.linalg.eigvalsh(cl.R[k].astype(np.float64)) > 0)


def test_cross_check_sklearn(pkg, oracle64):
    """Independent restatement: one E-step + one M-step from fixed parameters must
    match sklearn.mixture.GaussianMixture (same maximum-likelihood updates)."""
    sk = pytest.importorskip("sklearn.mixture")
    ev = small_problem(pkg, N=4000, D=4, K=5, seed=11)
    N, D = ev.shape
    K = 5
    cl = random_spd_params(pkg, K, D, np.random.default_rng(5))
    cl.memberships = np.zeros((K, N), np.float32)
    cl.avgvar[...] = 0.0
    cl.N[...] = cl.N / cl.N.sum() * N
    oracle64.constants(cl, K)
    weights0 = cl.pi.astype(np.float64).copy()
    means0 = cl.means.astype(np.float64).copy()
    prec0 = cl.Rinv.astype(np.float64).copy()
    prec0 = 0.5 * (prec0 + prec0.transpose(0, 2, 1))
    soa = oracle64.transpose(ev)
    ll = oracle64.estep(soa, cl, K)
    gm = sk.GaussianMixture(n_components=K, covariance_type="full", tol=0.0, reg_covar=0.0, max_iter=1,
                            weights_init=weights0 / weights0.sum(), means_init=means0, precisions_init=prec0)
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        gm.fit(ev.astype(np.float64))
    # responsibilities of the initial parameters
    gm0 = sk.GaussianMixture(n_components=K, covariance_type="full")
    gm0.weights_ = weights0 / weights0.sum()
    gm0.means_ = means0
    gm0.precisions_cholesky_ = np.stack([np.linalg.cholesky(p) for p in prec0])
    gm0.covariances_ = np.linalg.inv(prec0)
    resp = gm0.predict_proba(ev.astype(np.float64))
    np.testing.assert_allclose(cl.memberships.T, resp, rtol=2e-4, atol=1e-6)
    assert abs(ll - gm0.score(ev.astype(np.float64)) * N) < 1e-5 * abs(ll)
    oracle64.mstep(soa, cl, K)
    np.testing.assert_allclose(cl.means, gm.means_, rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(cl.R, gm.covariances_, rtol=1e-3, atol=2e-4)
    np.testing.assert_allclose(cl.N / N, gm.weights_, rtol=1e-4)


def test_em_loglik_monotone(pkg, oracle64):
    ev = small_problem(pkg, N=5000, D=4, K=6, seed=5)
    K = 6
    soa = oracle64.transpose(ev)
    cl = pkg.Clusters(K, 4, ev.shape[0])
    oracle64.seed(ev, K, cl)
    prev = oracle64.estep(soa, cl, K)
    for _ in range(15):
        oracle64.mstep(soa, cl, K)
        oracle64.constants(cl, K)
        ll = oracle64.estep(soa, cl, K)
        assert ll >= prev - 1e-4 * abs(prev)      # regulariser makes it only approximately monotone
        prev = ll


def test_fit_reduces_order(pkg, oracle64):
    ev = pkg.synth.make_blobs(2000, 3, 3, seed=9)
    K0 = 6
    cl = pkg.Clusters(K0, 3, ev.shape[0])
    saved = pkg.Clusters(K0, 3, ev.shape[0])
    ideal, mr = oracle64.fit(ev, K0, 0, 10, 10, cl, saved)
    assert 1 <= ideal <= K0
    ideal3, _ = oracle64.fit(ev, K0, 3, 10, 10, cl, saved)
    assert ideal3 == 3
    np.testing.assert_allclose(saved.memberships[:3].sum(0), 1.0, atol=1e-5)


def _parse_summary(path):
    clusters = []
    cur = None
    mode = None
    with open(path) as f:
        for line in f:
            s = line.strip()
            if s.startswith("Cluster #"):
                cur = dict(R=[])
                clusters.append(cur)
                mode = None
            elif s.startswith("Probability:"):
                cur["pi"] = float(s.split(":")[1])
            elif s.startswith("N:"):
                cur["N"] = float(s.split(":")[1])
            elif s.startswith("Means:"):
                cur["means"] = [float(v) for v in s.split(":")[1].split()]
            elif s.startswith("R Matrix"):
                mode = "R"
            elif mode == "R" and s:
                cur["R"].append([float(v) for v in s.split()])
    return clusters


@pytest.mark.skipif(not os.path.exists(os.path.join(GOLDEN, "ref_c1.summary")),
                    reason="golden fixtures from the reference binary not generated yet (parity unpinned)")
def test_oracle_matches_reference_golden(pkg, oracle64, oracle32):
    """tests/golden/ref_c1.* were written by the UNMODIFIED reference program
    (oracle/_ref/gaussianMPI_ref, built by oracle/Makefile `ref`) on an H100:
    K=8 on the config-1 data set (N=10k, D=4), GMM_REF_ITERS iterations, target 8."""
    meta = dict(l.strip().split("=") for l in open(os.path.join(GOLDEN, "ref_c1.meta")))
    iters, K = int(meta["iters"]), int(meta["K"])
    ev = pkg.synth.read_bin(os.path.join(GOLDEN, "c1.bin")) if os.path.exists(os.path.join(GOLDEN, "c1.bin")) \
        else pkg.synth.make_blobs(int(meta["N"]), int(meta["D"]), K, seed=int(meta["seed"]))
    D = ev.shape[1]
    golden = _parse_summary(os.path.join(GOLDEN, "ref_c1.summary"))
    assert len(golden) == K
    for orc in (oracle64, oracle32):
        cl = pkg.Clusters(K, D, ev.shape[0])
        orc.seed(ev, K, cl)
        orc.em(orc.transpose(ev), cl, K, iters, iters)
        for k in range(K):
            g = golden[k]
            assert abs(cl.pi[k] - g["pi"]) < 2e-5
            assert abs(cl.N[k] - g["N"]) < 1e-3 * max(1.0, g["N"]) + 2e-2
            np.testing.assert_allclose(cl.means[k], g["means"], atol=2e-3)
            np.testing.assert_allclose(cl.R[k], np.array(g["R"]), atol=2e-3)
        res = os.path.join(GOLDEN, "ref_c1.results.head")
        if os.path.exists(res):
            rows = [l.rstrip("\n").split("\t") for l in open(res)]
            memb = np.array([[float(v) for v in r[1].split(",")] for r in rows])
            np.testing.assert_allclose(cl.memberships[:, :len(rows)].T, memb, atol=2e-4)


def test_estep_permutation_equivariance_and_mstep_linearity(pkg, oracle64):
    """Size-independent properties the GPU parity tests rely on at full size: relabelling the
    clusters permutes the responsibilities and leaves the log-likelihood unchanged; the
    M-step statistics are linear in the responsibilities (N_k and N_k * mean_k add up)."""
    ev = small_problem(pkg, N=2500, D=5, K=4, seed=11)
    N, D = ev.shape
    K = 4
    soa = oracle64.transpose(ev)
    cl = random_spd_params(pkg, K, D, rng=np.random.default_rng(5))
    cl.memberships = np.zeros((K, N), np.float32)
    oracle64.constants(cl, K)
    ll = oracle64.estep(soa, cl, K)
    perm = np.array([2, 0, 3, 1])
    cp = cl.copy()
    for name in ("N", "pi", "constant", "avgvar"):
        getattr(cp, name)[:] = getattr(cl, name)[perm]
    cp.means[:] = cl.means[perm]; cp.R[:] = cl.R[perm]; cp.Rinv[:] = cl.Rinv[perm]
    cp.memberships = np.zeros((K, N), np.float32)
    llp = oracle64.estep(soa, cp, K)
    assert abs(ll - llp) <= 1e-6 * abs(ll)
    np.testing.assert_allclose(cp.memberships, cl.memberships[perm], rtol=1e-5, atol=1e-7)
    np.testing.assert_allclose(cl.memberships.sum(0), 1.0, atol=1e-5)

    # linearity: split the responsibilities of every cluster into two parts a + b
    rng = np.random.default_rng(6)
    w = rng.uniform(0.2, 0.8, size=(K, N)).astype(np.float32)
    full, pa, pb = cl.copy(), cl.copy(), cl.copy()
    full.memberships = cl.memberships.copy()
    pa.memberships = (cl.memberships * w).astype(np.float32)
    pb.memberships = (cl.memberships - pa.memberships).astype(np.float32)
    for c in (full, pa, pb):
        oracle64.mstep(soa, c, K)
    np.testing.assert_allclose(pa.N + pb.N, full.N, rtol=2e-6)
    np.testing.assert_allclose(pa.N[:, None] * pa.means + pb.N[:, None] * pb.means, full.N[:, None] * full.means,
                               rtol=1e-4, atol=1e-3)
