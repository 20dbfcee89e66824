"""EM over several samples with shared components (gmm_em_multisample, Engine.em_multisample) on the GPU (run with -m gpu
on an H100), against the restatement tests/_multisample_ref.py (itself checked in tests/test_multisample_host.py).  Every
case fixes the E-step path (a forced path never degrades silently) and checks which M-step kernel ran."""
import threading

import numpy as np
import pytest

import _multisample_ref as ms
from conftest import RUN_MEMB, RUN_RTOL_N, assert_params_close, gpu_count

pytestmark = pytest.mark.gpu

ARG, STATE = 1, 6                          # GMM_ERR_ARG, GMM_ERR_STATE
MSTEP_TOL_N = 1.5e-5                       # the tensor M-step's per-cluster bar on N (tests/test_mstep_error_model.py)


@pytest.fixture(scope="module")
def loaded(pkg):
    pkg.load_library()
    return pkg


def _tensor_estep(D):
    return D in (8, 16, 24)


def _engine(pkg, ev, K, D):
    eng = pkg.Engine(ev, K)
    eng.set_option("estep_path", pkg.PATH_TENSOR if _tensor_estep(D) else pkg.PATH_SIMT)
    return eng


def _memb(eng, K):
    return eng.get_clusters(K, with_memberships=True).memberships[:K].copy()


def _offsets(n, S, rng):
    """S samples of n events: boundaries at odd offsets, a 1-event sample, and a sample inside one 32-event window."""
    if S == 1:
        return np.array([0, n], np.int64)
    if S == 3:
        return np.array([0, 1001, 1002, n], np.int64)
    cuts = set(int(v) | 1 for v in rng.choice(np.arange(40, n - 40), S - 4, replace=False))
    cuts |= {5, 6, 17}                                       # [5, 6) one event; [6, 17) inside the window [0, 32)
    cuts = sorted(c for c in cuts if 0 < c < n)[:S - 1]
    while len(cuts) < S - 1:
        cuts = sorted(set(cuts) | {int(rng.integers(40, n - 40))})
    return np.array([0] + cuts + [n], np.int64)


def _assert_bits(a, b, msg=""):
    np.testing.assert_array_equal(np.asarray(a, np.float32).view(np.int32), np.asarray(b, np.float32).view(np.int32), err_msg=msg)


ONE_STEP = [(D, K) for D in (8, 16, 24, 5, 32) for K in (1, 7, 64, 65, 130, 512)]
SAMPLES = [(1, False), (3, True), (257, False), (257, True)]


def _one_reweight(pkg, D, K, n, S, weighted, seed):
    """max_iters = 0: the memberships are the float32 reweight of gmm_estep's, bit for bit; the correction enters the
    log-likelihood; one more call's masses are float64 sums of the stored r', and their sum over the samples is the next
    M-step's S0 within that M-step's bar."""
    rng = np.random.default_rng(seed)
    ev = pkg.synth.make_blobs(n, D, max(2, min(K, 12)), seed=D + K)
    off = _offsets(n, S, rng)
    pi0 = rng.dirichlet(np.ones(K), size=S)
    w = rng.integers(0, 4, n).astype(np.float32) if weighted else None
    if weighted:
        w[off[:-1]] = 1.0                                    # every sample keeps a positive total weight
    with _engine(pkg, ev, K, D) as eng:
        eng.seed(K)
        if weighted:
            eng.set_weights(w)
        ll0 = eng.estep(K)
        r = _memb(eng, K)
        pooled = eng.get_clusters(K).pi[:K].copy()
        pi, ns, ll, it, lls = eng.em_multisample(K, off, pi0, 0, 0, logliks=True)
        assert it == 0 and lls.shape == (1,) and lls[0] == ll
        np.testing.assert_allclose(pi, pi0 / pi0.sum(1, keepdims=True), rtol=1e-14)
        want, _, corr = ms.reweight32(r, ms.rho_of(pi, pooled), off, w)
        del r
        _assert_bits(_memb(eng, K), want)
        _, ns_ref = ms.masses(want, off, K, w)
        np.testing.assert_allclose(ns, ns_ref, rtol=1e-12)
        assert abs(ll - (ll0 + corr)) <= 1e-5 * max(abs(ll0), abs(ll0 + corr), 1.0), (ll, ll0, corr)
        # one iteration from the same start: pi^1 = max(M / n_s, 1e-10) from the masses of the same r'
        eng.profile(reset=True)
        pi1, *_ = eng.em_multisample(K, off, pi0, 1, 1)
        M_ref, _ = ms.masses(want, off, K, w)
        np.testing.assert_allclose(pi1, ms.update_pi(M_ref, ns_ref), rtol=1e-12, atol=0)
        N = eng.get_clusters(K).N[:K].astype(np.float64)
        Msum = M_ref.sum(0)
        assert float((np.abs(N - Msum) / np.maximum(Msum, 1.0)).max()) <= MSTEP_TOL_N
        p = eng.profile()
        assert p["mstep_tensor_launches"] + p["mstep_simt_launches"] == 1, p


@pytest.mark.parametrize("S,weighted", SAMPLES)
@pytest.mark.parametrize("D,K", ONE_STEP)
def test_one_reweight_bit_for_bit(loaded, D, K, S, weighted):
    _one_reweight(loaded, D, K, 4099, S, weighted, 1000 * D + K + S)


def _window_events(K):
    """kernels_multisample.cuh's window: the largest power of two in [32, 256] whose K x E float tile fits 64 KB."""
    E = 256
    while E > 32 and K * E * 4 > 64 * 1024:
        E >>= 1
    return E


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("D,K,n", [(8, 7, 1_000_001), (5, 7, 1_000_001), (8, 512, 300_001), (32, 512, 300_001)])
def test_one_reweight_persistent_ctas(loaded, D, K, n, weighted):
    """The same checks where every CTA walks several units and several samples: the units outnumber twice the most CTAs
    the SMs can hold (8 per SM at 256 threads), so the grid's CTAs reload rho, flush records and restart their sums."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert n // _window_events(K) >= 2 * 8 * sms
    _one_reweight(loaded, D, K, n, 257, weighted, 7 * D + K)


@pytest.mark.parametrize("K", [7, 65])
def test_rows_beyond_k_keep_their_contents(loaded, K):
    """Rows K .. of the memberships (read by the tensor M-step's 32-cluster boxes) are not written by the pass."""
    pkg = loaded
    D, n, rows = 8, 5003, 96
    ev = pkg.synth.make_blobs(n, D, 6, seed=31)
    off = np.array([0, 17, 18, 2501, n], np.int64)
    pi0 = np.random.default_rng(K).dirichlet(np.ones(K), size=4)
    with pkg.Engine(ev, rows) as eng:
        eng.set_option("estep_path", pkg.PATH_TENSOR)
        eng.seed(K)
        eng.estep(K)
        before = eng.get_clusters(rows, with_memberships=True).memberships[K:].copy()
        eng.em_multisample(K, off, pi0, 0, 0)
        after = eng.get_clusters(rows, with_memberships=True).memberships[K:]
    _assert_bits(after, before)


def _fit_fixture(pkg, D, K, n, seed):
    ev = pkg.synth.make_blobs(n, D, K, seed=seed)
    off = np.array([0, n // 5, n // 5 + 7, (2 * n) // 3 + 1, n], np.int64)
    return ev, off


@pytest.mark.parametrize("D,K,tensor_mstep", [(8, 6, True), (24, 9, True), (5, 6, False), (32, 5, False)])
@pytest.mark.parametrize("iters", [1, 30])
def test_iterations_against_restatement(loaded, D, K, tensor_mstep, iters):
    pkg = loaded
    n = 12000
    ev, off = _fit_fixture(pkg, D, K, n, 60 + D + K)
    rng = np.random.default_rng(D * K)
    pi0 = rng.dirichlet(np.full(K, 3.0), size=len(off) - 1)
    with _engine(pkg, ev, K, D) as eng:
        eng.set_option("mstep_path", pkg.PATH_TENSOR if tensor_mstep else pkg.PATH_SIMT)
        eng.seed(K)
        cl_ref = eng.get_clusters(K)
        pi, ns, ll, it, lls = eng.em_multisample(K, off, pi0, iters, iters, logliks=True)
        got = eng.get_clusters(K, with_memberships=True)
        p = eng.profile()
        assert (p["mstep_tensor_launches"] > 0) == tensor_mstep and (p["mstep_simt_launches"] > 0) != tensor_mstep, p
    pi_r, ns_r, lls_r, resp_r = ms.em(pkg, ev, cl_ref, K, off, pi0, iters)
    assert it == iters
    np.testing.assert_array_equal(ns, ns_r)
    if iters == 1:
        assert_params_close(got, cl_ref, K, rtol=1e-4)
        np.testing.assert_allclose(pi, pi_r, rtol=1e-4, atol=1e-9)
    else:
        assert_params_close(got, cl_ref, K, rtol=1e-4, rtol_N=RUN_RTOL_N)
        np.testing.assert_allclose(pi, pi_r, rtol=RUN_RTOL_N, atol=1e-9)
    np.testing.assert_allclose(got.memberships[:K], resp_r.T, **RUN_MEMB)
    np.testing.assert_allclose(lls, lls_r, rtol=1e-5)


@pytest.mark.parametrize("D,K", [(16, 8), (5, 7)])
def test_one_sample_is_the_pooled_fit(loaded, D, K):
    pkg = loaded
    n = 20000
    ev = pkg.synth.make_blobs(n, D, K, seed=D + 3 * K)
    with _engine(pkg, ev, K, D) as eng:
        start = eng.seed(K)
        eng.estep(K)
        r = _memb(eng, K)
        for S in (1, 3):                                      # pi_init = NULL: the start is gmm_estep, bit for bit
            eng.set_clusters(K, start)
            off = np.array([0, n], np.int64) if S == 1 else np.array([0, 11, 5000, n], np.int64)
            pi, ns, ll, it, _ = eng.em_multisample(K, off, None, 0, 0)
            _assert_bits(_memb(eng, K), r)
            np.testing.assert_array_equal(pi, np.tile(start.pi[:K].astype(np.float64), (S, 1)))
        eng.set_clusters(K, start)
        pi, ns, ll, it, _ = eng.em_multisample(K, [0, n], None, 20, 20)
        ms_cl = eng.get_clusters(K, with_memberships=True)
        eng.set_clusters(K, start)
        ll_em, it_em = eng.em(K, 20, 20)
        em_cl = eng.get_clusters(K, with_memberships=True)
    assert it == it_em == 20
    assert_params_close(ms_cl, em_cl, K, rtol=1e-4, rtol_N=RUN_RTOL_N)
    np.testing.assert_allclose(ms_cl.memberships[:K], em_cl.memberships[:K], **RUN_MEMB)
    np.testing.assert_allclose(pi[0], em_cl.pi[:K], rtol=RUN_RTOL_N, atol=1e-9)
    assert abs(ll - ll_em) <= 1e-5 * abs(ll_em)


def _truth(pkg, K, D):
    cl = pkg.Clusters(K, D)
    for k in range(K):
        cl.means[k] = 0.0
        cl.means[k, k % D] = 10.0 * (1 + k // D)
    cl.R[:K] = np.eye(D, dtype=np.float32)
    cl.Rinv[:K] = np.eye(D, dtype=np.float32)
    cl.constant[:K] = np.float32(-0.5 * D * np.log(2 * np.pi))
    cl.N[:K] = 1.0
    cl.pi[:K] = 1.0 / K
    cl.avgvar[:K] = 0.0
    return cl


def test_recovery_of_per_sample_weights(loaded):
    pkg = loaded
    D, K, n = 8, 4, 1_000_000
    truth = np.array([[0.2, 0.3, 0.25, 0.25], [0.005, 0.495, 0.3, 0.2], [0.0, 0.2, 0.2, 0.6]])
    cl = _truth(pkg, K, D)
    parts = []
    with pkg.Engine(np.zeros((1, D), np.float32), K) as g:
        for s in range(3):
            cl.pi[:K] = truth[s].astype(np.float32)
            g.set_clusters(K, cl)
            x, _ = g.sample(K, n, seed=11 + s, labels=False)
            parts.append(x)
    ev = np.concatenate(parts)
    off = np.array([0, n, 2 * n, 3 * n], np.int64)
    cl.pi[:K] = 1.0 / K
    cl.N[:K] = 3 * n / K
    with _engine(pkg, ev, K, D) as eng:
        eng.set_clusters(K, cl)
        pi, ns, ll, it, lls = eng.em_multisample(K, off, None, 0, 100, logliks=True)
        assert eng.profile()["mstep_tensor_launches"] > 0
        eng.set_clusters(K, cl)
        ll_pool, _ = eng.em(K, 0, 100)
    se = np.sqrt(np.maximum(truth * (1 - truth), 1.0 / n) / n)
    assert np.all(np.abs(pi - truth) <= 4 * se), (pi, truth)
    np.testing.assert_array_equal(ns, [n, n, n])
    assert ll >= ll_pool - 1e-6 * abs(ll_pool), (ll, ll_pool)
    assert np.all(np.diff(lls.astype(np.float64)) >= -2e-6 * np.abs(lls[1:])), lls


def test_integer_weights_equal_replicated_rows(loaded):
    pkg = loaded
    D, K, n = 8, 5, 6000
    rng = np.random.default_rng(4)
    ev = pkg.synth.make_blobs(n, D, K, seed=21)
    off = np.array([0, 1500, 1501, 4000, n], np.int64)
    w = rng.integers(1, 4, n)
    rep = np.repeat(ev, w, axis=0)
    cw = np.concatenate([[0], np.cumsum(w)])
    off_rep = cw[off]
    pi0 = rng.dirichlet(np.ones(K), size=4)
    res = []
    for x, ww, o in ((ev, w.astype(np.float32), off), (rep, None, off_rep)):
        with _engine(pkg, x, K, D) as eng:
            eng.set_option("mstep_path", pkg.PATH_SIMT)
            eng.set_clusters(K, _seeded(pkg, ev, K))
            if ww is not None:
                eng.set_weights(ww)
            out = eng.em_multisample(K, o, pi0, 6, 6, logliks=True)
            res.append((out, eng.get_clusters(K)))
    (a, ca), (b, cb) = res
    np.testing.assert_allclose(a[0], b[0], rtol=1e-5, atol=1e-10)
    np.testing.assert_array_equal(a[1], b[1])
    np.testing.assert_allclose(a[4], b[4], rtol=1e-5)
    assert_params_close(ca, cb, K, rtol=1e-4, rtol_N=RUN_RTOL_N)


def _seeded(pkg, ev, K):
    with pkg.Engine(ev, K) as e:
        return e.seed(K)


def test_scoring_recipe_matches_stored_posteriors(loaded):
    pkg = loaded
    D, K, n = 16, 6, 30000
    ev = pkg.synth.make_blobs(n, D, K, seed=8)
    off = np.array([0, 9000, 9001, 20000, n], np.int64)
    with _engine(pkg, ev, K, D) as eng:
        eng.seed(K)
        pi, ns, ll, it, _ = eng.em_multisample(K, off, None, 5, 5)
        memb = _memb(eng, K)
        tot = 0.0
        for s in range(len(off) - 1):
            cl = eng.get_clusters(K)
            cl.pi[:K] = pi[s].astype(np.float32)
            eng.set_clusters(K, cl)
            lab, mr, lp, lls = eng.score(K, ev[off[s]:off[s + 1]])
            m = memb[:, off[s]:off[s + 1]]
            np.testing.assert_allclose(mr, m.max(0), rtol=1e-4, atol=1e-5)
            top2 = np.sort(m, 0)[-2:]
            sure = top2[1] - top2[0] > 1e-3
            np.testing.assert_array_equal(lab[sure], m.argmax(0)[sure])
            tot += lls
    assert abs(tot - ll) <= 1e-5 * abs(ll), (tot, ll)


def test_repeatable_state_and_combine(loaded):
    pkg = loaded
    D, K, n = 24, 10, 20000
    ev = pkg.synth.make_blobs(n, D, K, seed=9)
    off = np.array([0, 333, 7777, n], np.int64)
    pi0 = np.random.default_rng(2).dirichlet(np.ones(K), size=3)
    runs = []
    with _engine(pkg, ev, K, D) as eng:
        start = eng.seed(K)
        it0 = eng.profile(reset=True)["iterations"]
        assert it0 >= 0
        for _ in range(2):
            eng.set_clusters(K, start)
            out = eng.em_multisample(K, off, pi0, 4, 4)
            runs.append((out, eng.get_clusters(K, with_memberships=True)))
        p = eng.profile()
        assert p["iterations"] == 8 and p["mstep_tensor_launches"] == 8 and p["mstep_simt_launches"] == 0, p
        (a, ca), (b, cb) = runs
        np.testing.assert_array_equal(a[0], b[0])
        np.testing.assert_array_equal(a[1], b[1])
        _assert_bits(ca.memberships[:K], cb.memberships[:K])
        _assert_bits(ca.means[:K], cb.means[:K])
        _assert_bits(ca.R[:K], cb.R[:K])
        # the state afterwards: the pooled set, the per-sample posteriors, gmm_combine on them
        comb = eng.combine(K)
        assert comb["merges"].shape == (K - 1, 2) and np.all(np.isfinite(comb["gain"]))
        lab, _ = eng.combine_labels(K, np.arange(K))
        np.testing.assert_array_equal(lab, ca.memberships[:K].argmax(0))
        eng.score(K, ev[:100])
        eng.sample(K, 10)
        mp = eng.multisample_profile(reset=True)
        assert mp["kernel_ms"] > 0 and mp["host_ms"] > 0 and mp["wall_ms"] >= mp["kernel_ms"], mp
        assert eng.multisample_profile() == dict(kernel_ms=0.0, host_ms=0.0, wall_ms=0.0)
        # a later gmm_estep replaces them with the pooled ones
        eng.estep(K)
        assert not np.array_equal(_memb(eng, K), ca.memberships[:K])


def test_errors(loaded):
    pkg = loaded
    D, K, n = 8, 4, 3000
    ev = pkg.synth.make_blobs(n, D, K, seed=5)
    off = np.array([0, 1000, n], np.int64)
    with _engine(pkg, ev, K, D) as eng:
        with pytest.raises(pkg.GmmError) as e:
            eng.em_multisample(K, off)                         # before any parameter set
        assert e.value.code == STATE
        start = eng.seed(K)
        lib = eng.lib

        def code(*a):
            with pytest.raises(pkg.GmmError) as ex:
                eng.em_multisample(*a)
            return ex.value.code
        assert code(0, off) == ARG
        assert code(K + 1, off) == ARG
        assert code(K - 1, off) == STATE
        assert code(K, [0, n + 1]) == ARG
        assert code(K, [1, n]) == ARG
        assert code(K, [0, 5, 5, n]) == ARG
        assert code(K, np.linspace(0, n, 4098).astype(np.int64)) == ARG     # S = 4097
        assert code(K, off, np.array([[1, 1, -1, 1], [1, 1, 1, 1]])) == ARG
        assert code(K, off, np.array([[1, 1, np.nan, 1], [1, 1, 1, 1]])) == ARG
        assert code(K, off, np.array([[1, 1, np.inf, 1], [1, 1, 1, 1]])) == ARG
        assert code(K, off, np.array([[0, 0, 0, 0], [1, 1, 1, 1]])) == ARG
        assert code(K, off, None, -1, 3) == ARG
        assert code(K, off, None, 4, 3) == ARG
        zero = pkg.Clusters(K, D)
        for f in ("N", "pi", "constant", "means", "R", "Rinv", "avgvar"):
            getattr(zero, f)[...] = getattr(start, f)
        zero.pi[2] = 0.0
        eng.set_clusters(K, zero)
        assert code(K, off, np.array([[1, 1, 1, 1], [1, 1, 0, 1]])) == ARG
        eng.em_multisample(K, off, np.array([[1, 1, 0, 1], [1, 1, 0, 1]]), 0, 0)   # 0 where pi_k = 0 is fine
        eng.set_clusters(K, start)
        eng.estep(K)
        eng.mstep(K)
        assert code(K, off) == STATE                 # between gmm_mstep and gmm_constants
        eng.constants(K)
        w = np.ones(n, np.float32)
        w[1000:] = 0.0
        eng.set_weights(w)
        assert code(K, off) == ARG                   # a sample of total weight 0
        eng.set_weights(None)
        prof = np.zeros(3)
        assert lib.gmm_get_multisample_profile(None, prof.ctypes.data_as(lib.gmm_get_multisample_profile.argtypes[1]), 0) == ARG
        pi, ns, ll, it, _ = eng.em_multisample(K, off, None, 2, 2)
        assert it == 2 and np.isfinite(ll)


def test_two_gpus_equal_one(loaded):
    if gpu_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    pkg = loaded
    D, K, N = 16, 8, 40_001
    ev = pkg.synth.make_blobs(N, D, K, seed=12)
    b0, n0 = pkg.shard_range(N, 2, 0)
    off = np.array([0, 5000, n0 - 1001, n0 + 3001, N], np.int64)     # sample 2 straddles the shard boundary
    pi0 = np.random.default_rng(3).dirichlet(np.ones(K), size=4)
    start = _seeded(pkg, ev, K)
    with _engine(pkg, ev, K, D) as eng:
        eng.set_clusters(K, start)
        one = eng.em_multisample(K, off, pi0, 5, 5)
        cl1 = eng.get_clusters(K)
    uid = pkg.nccl_unique_id()
    res = [None, None]

    def worker(g):
        try:
            b, n = pkg.shard_range(N, 2, g)
            with pkg.Engine(np.ascontiguousarray(ev[b:b + n]), K, device=g, n_global=N, offset=b) as e:
                e.set_option("estep_path", pkg.PATH_TENSOR)
                e.comm_init(2, g, uid)
                e.set_clusters(K, start)
                res[g] = (e.em_multisample(K, off, pi0, 5, 5), e.get_clusters(K))
        except Exception as ex:  # noqa: BLE001
            res[g] = ex

    ts = [threading.Thread(target=worker, args=(g,)) for g in range(2)]
    for t in ts:
        t.start()
    for t in ts:
        t.join(timeout=600)
    for r in res:
        assert not isinstance(r, Exception), r
        np.testing.assert_allclose(r[0][0], one[0], rtol=1e-5, atol=1e-10)
        np.testing.assert_array_equal(r[0][1], one[1])
        assert abs(r[0][2] - one[2]) <= 1e-5 * abs(one[2])
        assert_params_close(r[1], cl1, K, rtol=1e-4, rtol_N=RUN_RTOL_N)
    np.testing.assert_array_equal(res[0][0][0], res[1][0][0])
