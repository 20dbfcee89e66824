"""Variational Bayesian EM (gmm_vb_em, Engine.vb_em) on the GPU (run with -m gpu on an H100), against the float64
restatement tests/_vb_ref.py (itself checked against sklearn's BayesianGaussianMixture in tests/test_vb_host.py)."""
import threading

import numpy as np
import pytest

import _vb_ref as vb
from conftest import RUN_MEMB, RUN_RTOL_N, assert_params_close, gpu_count

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def loaded(pkg):
    pkg.load_library()
    return pkg


def _ref_params(pkg, p, K, D):
    cl = pkg.Clusters(K, D)
    for f in ("N", "pi", "constant", "means", "R", "Rinv"):
        getattr(cl, f)[...] = p[f]
    return cl


def _start(eng, K, kmeans=True):
    """The start set and its responsibilities g0 [n][K] (gmm_estep + gmm_get_clusters)."""
    if kmeans:
        eng.seed_kmeans(K, max_iter=5, seed=3)
    else:
        eng.seed(K)
    eng.estep(K)
    return eng.get_clusters(K, with_memberships=True).memberships[:K].T.astype(np.float64)


def _prior_of(post, K, D, ptype):
    return vb.prior(K, D, ptype, m0=post["mean_prior"], psi0=post["covariance_prior"])


ONE_STEP = [(D, K) for D in (8, 16, 24, 5, 32) for K in (1, 7, 64, 65, 130)]


@pytest.mark.parametrize("ptype", [vb.DP, vb.DIRICHLET])
@pytest.mark.parametrize("D,K", ONE_STEP)
def test_one_step(loaded, D, K, ptype):
    """max_iters = 0: posterior 0 from the engine's g0 equals the restatement's at the per-operator bar; the default prior is
    the events' mean and np.cov."""
    pkg = loaded
    N = 6000
    ev = pkg.synth.make_blobs(N, D, max(2, min(K, 12)), seed=40 + D + K)
    with pkg.Engine(ev, K) as eng:
        g0 = _start(eng, K)
        cl, post, lb, lbs, it, conv = eng.vb_em(K, 0, 0, prior_type=ptype)
        assert it == 0 and not conv and lb == -np.inf
        m0, psi0 = vb.default_moments(ev)
        np.testing.assert_allclose(post["mean_prior"], m0, rtol=1e-5, atol=1e-5 * np.abs(m0).max())
        np.testing.assert_allclose(post["covariance_prior"], psi0, rtol=1e-5, atol=1e-5 * np.abs(psi0).max())
        p = vb.m_step(vb.stats_from_resp(ev, g0, np.zeros(D)), np.zeros(D), K, D, _prior_of(post, K, D, ptype))
        assert_params_close(cl, _ref_params(pkg, p, K, D), K)
        np.testing.assert_allclose(post["weights"], p["weights"], rtol=1e-4, atol=1e-7)
        np.testing.assert_allclose(post["dof"], p["nu"], rtol=1e-4)
        # the memberships left are those of posterior 0 (the last E-step)
        got = eng.get_clusters(K, with_memberships=True).memberships[:K].T
        lr, _ = vb.e_step(ev, p)
        np.testing.assert_allclose(got, np.exp(lr), **RUN_MEMB)


def test_one_step_kmax_128_at_k_64(loaded):
    pkg = loaded
    N, D, K = 6000, 24, 64
    ev = pkg.synth.make_blobs(N, D, 12, seed=77)
    res = []
    for kmax in (64, 128):
        with pkg.Engine(ev, kmax) as eng:
            _start(eng, K)
            cl, post, *_ = eng.vb_em(K, 0, 0)
            res.append((cl, post))
    assert_params_close(res[1][0], res[0][0], K)


@pytest.mark.parametrize("D,path", [(16, 0), (24, 0), (5, 0), (16, 1)])
def test_fixed_iterations(loaded, D, path):
    """min = max = 30 against the restatement run from the same g0, at the run-level bars."""
    pkg = loaded
    N, K = 8000, 12
    ev = pkg.synth.make_blobs(N, D, 6, seed=90 + D)
    with pkg.Engine(ev, K) as eng:
        eng.set_option("path", path)
        g0 = _start(eng, K)
        cl, post, lb, lbs, it, conv = eng.vb_em(K, 30, 30, lower_bounds=True)
        assert it == 30 and not conv and len(lbs) == 30
        got = eng.get_clusters(K, with_memberships=True).memberships[:K].T
    p, lb_ref, lbs_ref, it_ref, _, resp = vb.fit(ev.astype(np.float64), g0, _prior_of(post, K, D, vb.DP), 30, 30, 0.0)
    ref = _ref_params(pkg, p, K, D)
    # pi = weights_ is a function of every N (the DP's stick-breaking products), and E[ln pi] moves every logit by about dN / N:
    # both carry N's run-level bar, and the memberships the corresponding share of it (measured up to 1.9e-3 after 30 iterations)
    np.testing.assert_allclose(cl.pi[:K], ref.pi[:K], rtol=RUN_RTOL_N, atol=1e-7)
    ref.pi[:K] = cl.pi[:K]
    assert_params_close(cl, ref, K, rtol_N=RUN_RTOL_N)
    np.testing.assert_allclose(got, resp, rtol=3e-3, atol=RUN_MEMB["atol"])
    np.testing.assert_allclose(lbs, lbs_ref, rtol=1e-5)


@pytest.mark.parametrize("weighted", [False, True])
def test_bound(loaded, weighted):
    """The entropy pass equals float64 -sum w g ln g of the returned memberships; the bounds rise within noise; the stop
    decision is the tol rule applied to the returned bounds."""
    pkg = loaded
    N, D, K = 20000, 16, 20
    ev = pkg.synth.make_blobs(N, D, 6, seed=5)
    w = np.random.default_rng(1).integers(1, 4, N).astype(np.float32) if weighted else None
    with pkg.Engine(ev, K) as eng:
        eng.set_option("mstep_path", 1)                  # FP64 statistics: the bound's parameter part is reproduced to ~1e-12
        if weighted:
            eng.set_weights(w)
        _start(eng, K, kmeans=False)
        eng.vb_em(K, 0, 0)
        g1 = eng.get_clusters(K, with_memberships=True).memberships[:K].T.astype(np.float64)   # E-step under posterior 0
        _start(eng, K, kmeans=False)
        cl1, post1, lb1, *_ = eng.vb_em(K, 1, 1)          # LB_1 = entropy of that E-step + parameter part of posterior 1
        ent = vb.entropy_sum(g1, w)
        pr = _prior_of(post1, K, D, vb.DP)
        _, bound_par = pkg.host_vb_finalize(vb.stats_from_resp(ev, g1, np.zeros(D), w), np.zeros(D), pkg.Clusters(K, D), K,
                                            pr["m0"], pr["psi0"])
        assert abs(ent) > 1e3
        assert abs((lb1 - bound_par) + ent) <= 1e-6 * abs(ent) + 1e-9 * abs(bound_par), (lb1, bound_par, ent)
        _start(eng, K, kmeans=False)
        tol = 1e-2
        cl, post, lb, lbs, it, conv = eng.vb_em(K, 3, 200, tol=tol, lower_bounds=True)
    noise = 1e-6 * np.abs(lbs).max()
    assert (np.diff(lbs) >= -noise).all(), np.diff(lbs).min()
    d = np.abs(np.diff(np.concatenate([[-np.inf], lbs])))
    stop = [i + 1 for i in range(len(lbs)) if i + 1 >= 3 and d[i] < tol]
    if conv:
        assert stop and stop[0] == it
    else:
        assert not stop and it == 200
    assert lb == lbs[-1]


def test_pruning_matches_sklearn(loaded):
    """8 well-separated blobs drawn with gmm_sample, fitted at K = 40 after gmm_seed_kmeans: 8 components with weights_ >
    0.01, the set sklearn's BayesianGaussianMixture picks from the same g0."""
    pkg = loaded
    D, Kt, N, K = 8, 8, 30000, 40
    rng = np.random.default_rng(11)
    src = pkg.Clusters(Kt, D)
    src.means[...] = rng.uniform(-30, 30, (Kt, D)).astype(np.float32)
    src.R[...] = np.eye(D, dtype=np.float32)
    src.pi[...] = 1.0 / Kt
    src.N[...] = N / Kt
    with pkg.Engine(np.zeros((16, D), np.float32), Kt) as gen:
        gen.set_clusters(Kt, src)
        ev, _ = gen.sample(Kt, N, seed=5)
    with pkg.Engine(ev, K) as eng:
        g0 = _start(eng, K)
        cl, post, lb, lbs, it, conv = eng.vb_em(K, 0, 500, tol=1e-3)
    keep = set(np.flatnonzero(post["weights"] > 0.01))
    assert len(keep) == Kt, (len(keep), post["weights"])
    mixture = pytest.importorskip("sklearn.mixture")
    X = ev.astype(np.float64)
    bgm = mixture.BayesianGaussianMixture(n_components=K, covariance_type="full", max_iter=500)
    bgm._check_parameters(X)
    bgm._initialize(X, g0)
    prev = -np.inf
    for _ in range(500):
        lpn, lr = bgm._e_step(X)
        bgm._m_step(X, lr)
        cur = bgm._compute_lower_bound(lr, lpn)
        if abs(cur - prev) < 1e-3:
            break
        prev = cur
    bgm._set_parameters(bgm._get_parameters())
    assert set(np.flatnonzero(bgm.weights_ > 0.01)) == keep


def test_after_fit_score_and_estep(loaded):
    """On new events gmm_score's labels and log-densities are the restatement's predict / score_samples; gmm_estep's
    memberships are its predict_proba."""
    pkg = loaded
    N, D, K = 8000, 16, 10
    ev = pkg.synth.make_blobs(N, D, 5, seed=21)
    new = pkg.synth.make_blobs(3000, D, 5, seed=21 + 1)
    with pkg.Engine(ev, K) as eng:
        g0 = _start(eng, K)
        cl, post, *_ = eng.vb_em(K, 0, 0)
        p = vb.m_step(vb.stats_from_resp(ev, g0, np.zeros(D)), np.zeros(D), K, D, _prior_of(post, K, D, vb.DP))
        lab, mr, lp, _ = eng.score(K, new)
        eng.estep(K)
        got = eng.get_clusters(K, with_memberships=True).memberships[:K].T
    lr_new, norm_new = vb.e_step(new.astype(np.float64), p)
    np.testing.assert_allclose(lp, norm_new, rtol=1e-4, atol=1e-3)
    top2 = np.sort(lr_new, 1)[:, -2:]
    clear = top2[:, 1] - top2[:, 0] > 1e-3
    assert (lab[clear] == lr_new.argmax(1)[clear]).all()
    lr, _ = vb.e_step(ev.astype(np.float64), p)
    np.testing.assert_allclose(got, np.exp(lr), **RUN_MEMB)


def test_integer_weights_equal_replicated_rows(loaded):
    """Integer weights 1..5 give the fit of replicated rows, default prior included."""
    pkg = loaded
    N, D, K = 5000, 8, 8
    ev = pkg.synth.make_blobs(N, D, 4, seed=33)
    w = np.random.default_rng(2).integers(1, 6, N)
    rep = np.repeat(ev, w, axis=0)
    out = []
    with pkg.Engine(ev, K) as eng:
        start = eng.seed(K)
        eng.set_weights(w.astype(np.float32))
        out.append(eng.vb_em(K, 10, 10, lower_bounds=True))
    with pkg.Engine(rep, K) as eng:
        eng.set_clusters(K, start)
        out.append(eng.vb_em(K, 10, 10, lower_bounds=True))
    (ca, pa, la, lsa, *_), (cb, pb, lb, lsb, *_) = out
    np.testing.assert_allclose(pa["mean_prior"], pb["mean_prior"], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(pa["covariance_prior"], pb["covariance_prior"], rtol=1e-5, atol=1e-5 * np.abs(pb["covariance_prior"]).max())
    assert_params_close(ca, cb, K, rtol_N=RUN_RTOL_N)
    np.testing.assert_allclose(lsa, lsb, rtol=1e-5)


def test_errors_and_state(loaded):
    pkg = loaded
    N, D, K = 4000, 8, 6
    ev = pkg.synth.make_blobs(N, D, 3, seed=8)
    with pkg.Engine(ev, K) as eng:
        eng.seed(K)
        for kw in (dict(min_iters=-1), dict(min_iters=3, max_iters=2), dict(tol=-1.0), dict(tol=np.nan), dict(dof=3.0),
                   dict(weight_concentration=np.inf), dict(mean_precision=np.nan), dict(prior_type=5),
                   dict(covariance=-np.eye(D)), dict(covariance=np.triu(np.ones((D, D))) + np.eye(D))):
            with pytest.raises(pkg.GmmError) as e:
                eng.vb_em(K, **kw)
            assert e.value.code == 1, kw
        with pytest.raises(pkg.GmmError) as e:
            eng.vb_em(K + 1 if K + 1 <= eng.Kmax else K - 1)
        assert e.value.code == 6
        with pytest.raises(pkg.GmmError) as e:
            eng.vb_em(0)
        assert e.value.code == 1
        L = pkg.load_library()
        assert L.gmm_vb_em(eng.h, K, None, 0, 1, 0.0, None, None, None, None, None, None) == 1
        eng.estep(K)
        eng.mstep(K)
        with pytest.raises(pkg.GmmError) as e:
            eng.vb_em(K)
        assert e.value.code == 6
        eng.constants(K)
        # after a fit the set counts as given from outside: a device-side EM batch whose first iteration is replayed on the
        # host keeps its Rinv and constant, as an all-host batch from gmm_set_clusters of the same set does
        cl, *_ = eng.vb_em(K, 5, 5)
        assert eng.profile()["iterations"] >= 5
        np.testing.assert_array_equal(eng.get_clusters(K).constant[:K], cl.constant[:K])
        replays = eng.fit_profile()["host_replays"]
        eng.set_option("finalize_fault_iter", 0)
        eng.em_iterations(K, 2)
        eng.set_option("finalize_fault_iter", -1)
        assert eng.fit_profile()["host_replays"] == replays + 1
        got = eng.get_clusters(K)
    with pkg.Engine(ev, K) as e2:
        e2.set_option("finalize", 0)
        e2.set_clusters(K, cl)
        e2.estep(K)
        e2.em_iterations(K, 2)
        ref = e2.get_clusters(K)
    for f in ("N", "pi", "constant", "means", "R", "Rinv"):
        np.testing.assert_array_equal(getattr(got, f)[:K], getattr(ref, f)[:K], err_msg=f)


def test_two_gpus_equal_one(loaded):
    if gpu_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    pkg = loaded
    N, D, K = 40_001, 16, 10
    ev = pkg.synth.make_blobs(N, D, 5, seed=55)
    with pkg.Engine(ev, K) as eng:
        start = eng.seed(K)
        one = eng.vb_em(K, 10, 10, lower_bounds=True)
    uid = pkg.nccl_unique_id()
    res = [None, None]

    def worker(g):
        try:
            b, n = pkg.shard_range(N, 2, g)
            with pkg.Engine(np.ascontiguousarray(ev[b:b + n]), K, device=g, n_global=N, offset=b) as e:
                e.comm_init(2, g, uid)
                e.set_clusters(K, start)
                res[g] = e.vb_em(K, 10, 10, lower_bounds=True)
        except Exception as ex:  # noqa: BLE001
            res[g] = ex

    ts = [threading.Thread(target=worker, args=(g,)) for g in range(2)]
    for t in ts:
        t.start()
    for t in ts:
        t.join(timeout=600)
    for r in res:
        assert not isinstance(r, Exception), r
        assert_params_close(r[0], one[0], K, rtol_N=RUN_RTOL_N)
        np.testing.assert_allclose(r[3], one[3], rtol=1e-6)
    np.testing.assert_array_equal(res[0][3], res[1][3])
