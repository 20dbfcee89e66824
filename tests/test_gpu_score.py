"""gmm_score: assigning and scoring new events with a fitted mixture (run with -m gpu on an H100).

On the training shard the outputs must be the E-step's own (max_resp bit for bit, at every K on both paths); on
new events, held out, between the clusters and up to ~50 standard deviations outside them, they are held against a
float64 log-sum-exp over the same parameter set.  The cases also cover the chunked streaming, the range fallback to the
SIMT kernel, the state errors and the claim that scoring leaves the EM state untouched."""
import ctypes as C

import numpy as np
import pytest
from scipy.special import logsumexp

from conftest import fitted_params

pytestmark = pytest.mark.gpu

TENSOR_D = (8, 16, 24)
SIMT_D = (5, 24, 32)
ERR_ARG, ERR_STATE = 1, 6


# ---- fixtures ---------------------------------------------------------------------------------------------------------
def blobs(pkg, n, D, seed=11, K_true=6):
    return pkg.synth.make_blobs(n, D, K_true, seed=seed)


def mixture(pkg, ev, K, seed=3):
    """A consistent parameter set (Rinv, constant, pi from R) with means on data points."""
    rng = np.random.default_rng(seed)
    D = ev.shape[1]
    cl = pkg.Clusters(K, D)
    cl.means[...] = ev[rng.choice(ev.shape[0], K, replace=False)]
    for k in range(K):
        A = rng.standard_normal((D, D))
        R = (A @ A.T / D + 0.5 * np.eye(D)) * rng.uniform(0.5, 3.0)
        cl.R[k] = R.astype(np.float32)
        R64 = cl.R[k].astype(np.float64)
        cl.Rinv[k] = np.linalg.inv(R64).astype(np.float32)
        cl.constant[k] = np.float32(-0.5 * D * np.log(2 * np.pi) - 0.5 * np.linalg.slogdet(R64)[1])
    w = rng.dirichlet(np.full(K, 5.0))
    cl.N[...] = (w * ev.shape[0]).astype(np.float32)
    cl.pi[...] = (w / w.sum()).astype(np.float32)
    cl.avgvar[...] = 0.01
    return cl


def engine(pkg, ev, K, path, Kmax=None):
    eng = pkg.Engine(ev, Kmax or K)
    eng.set_option("estep_path", path)
    return eng


def path_of(pkg, name):
    return pkg.PATH_TENSOR if name == "tensor" else pkg.PATH_SIMT


def ref_logits(cl, K, x):
    """float64 logits ln pi_k + constant_k - 0.5 (x - mu_k)^T Rinv_k (x - mu_k) of the parameter set."""
    x = np.asarray(x, np.float64)
    out = np.empty((x.shape[0], K))
    for k in range(K):
        d = x - cl.means[k].astype(np.float64)
        q = np.einsum("ni,ni->n", d @ cl.Rinv[k].astype(np.float64), d)
        out[:, k] = np.log(np.float64(cl.pi[k])) + np.float64(cl.constant[k]) - 0.5 * q
    return out


def top_two_gap(a, axis):
    s = np.sort(a, axis=axis)
    return np.take(s, -1, axis=axis) - np.take(s, -2, axis=axis)


def check_f64(cl, K, x, lab, mr, lp, what):
    """The float64 bar; returns the worst deviations (|dlogp| / (1 + |logp|), |dmax_resp| / (1e-6 + 1e-4 max_resp) units)."""
    L = ref_logits(cl, K, x)
    ref_lp = logsumexp(L, axis=1)
    ref_lab = L.argmax(1)
    ref_mr = np.exp(L.max(1) - ref_lp)
    dlp = np.abs(lp.astype(np.float64) - ref_lp) / (1.0 + np.abs(ref_lp))
    assert dlp.max() <= 1e-4, (what, float(dlp.max()))
    # a float32 logit of magnitude |l| carries ~1e-7 |l| of rounding: the label bar grows with it (1e-3 near the clusters)
    lmax = np.abs(L.max(1))
    sure = top_two_gap(L, 1) > 1e-3 + 1e-6 * lmax if K > 1 else np.ones(len(x), bool)
    np.testing.assert_array_equal(lab[sure], ref_lab[sure], err_msg=what)
    rtol = 1e-4 + 1e-6 * lmax
    dmr = np.abs(mr.astype(np.float64) - ref_mr) / (1e-6 + rtol * ref_mr)
    assert dmr.max() <= 1.0, (what, float(dmr.max()))
    rel_mr = np.abs(mr.astype(np.float64) - ref_mr) / ref_mr
    print(f"\nSCORE-DEV {what}: max |dlogp|/(1+|logp|) = {dlp.max():.2e}, max rel dmax_resp = {rel_mr.max():.2e}")
    return float(dlp.max()), float(rel_mr.max())


def check_shard(eng, K, ev, ll, bit_exact_mr=True):
    memb = eng.get_clusters(K, with_memberships=True).memberships[:K]
    lab, mr, lp, sll = eng.score(K, ev)
    top = memb.max(0)
    if bit_exact_mr:
        np.testing.assert_array_equal(mr, top)
    else:
        np.testing.assert_allclose(mr, top, rtol=1e-6, atol=0)
    differ = top_two_gap(memb, 0) > 0 if K > 1 else np.ones(ev.shape[0], bool)
    np.testing.assert_array_equal(lab[differ], memb.argmax(0)[differ])
    assert abs(float(np.sum(lp, dtype=np.float64)) - ll) <= 1e-6 * abs(ll), (np.sum(lp, dtype=np.float64), ll)
    assert abs(sll - ll) <= 1e-6 * abs(ll), (sll, ll)
    return lab, mr, lp


# ---- 1. training shard, bit-exact ----------------------------------------------------------------------------------------
SHARD_CASES = [("tensor", D, K) for D in TENSOR_D for K in (1, 7, 64)] + [("simt", D, K) for D in SIMT_D for K in (1, 7, 130)]


@pytest.mark.parametrize("path,D,K", SHARD_CASES)
def test_training_shard_matches_estep(pkg, path, D, K):
    ev = blobs(pkg, 20_011, D)
    with engine(pkg, ev, K, path_of(pkg, path)) as eng:
        eng.set_clusters(K, mixture(pkg, ev, K))
        ll = eng.estep(K)
        eng.score_profile(reset=True)
        check_shard(eng, K, ev, ll)
        prof = eng.score_profile()
        assert (prof["tensor_chunks"] > 0) == (path == "tensor") and (prof["simt_chunks"] > 0) == (path == "simt"), prof


def test_training_shard_after_device_iterations(pkg):
    D, K = 24, 64
    ev = blobs(pkg, 50_000, D)
    with engine(pkg, ev, K, pkg.PATH_AUTO) as eng:
        eng.set_option("finalize", 1)
        eng.set_clusters(K, mixture(pkg, ev, K))
        eng.estep(K)
        ll = eng.em_iterations(K, 5)
        assert eng.fit_profile()["device_finalize_launches"] >= 5
        check_shard(eng, K, ev, ll)


# ---- 2. tensor K > 64 on the training shard ------------------------------------------------------------------------------
@pytest.mark.parametrize("D,K", [(24, 65), (16, 130), (8, 512)])
def test_tensor_passes(pkg, D, K):
    ev = blobs(pkg, 20_011, D)
    cl = mixture(pkg, ev, K)
    with engine(pkg, ev, K, pkg.PATH_TENSOR) as eng:
        eng.set_clusters(K, cl)
        ll = eng.estep(K)
        lab, mr, lp = check_shard(eng, K, ev, ll)
        ref_lp = logsumexp(ref_logits(eng.get_clusters(K), K, ev), axis=1)
        assert np.max(np.abs(lp - ref_lp) / (1 + np.abs(ref_lp))) <= 1e-4


# ---- 3. new events against float64 ----------------------------------------------------------------------------------------
NEW_CASES = [("tensor", D, 7) for D in TENSOR_D] + [("tensor", 24, 130)] + [("simt", D, 7) for D in SIMT_D] + [("simt", 24, 130)]


def new_batches(ev_all, n_train, rng):
    held = ev_all[n_train:]
    a, b = held[rng.integers(0, len(held), 3000)], held[rng.integers(0, len(held), 3000)]
    between = (a + rng.uniform(0, 1, (3000, 1)) * (b - a)).astype(np.float32)
    mu, sd = ev_all[:n_train].mean(0), ev_all[:n_train].std(0)
    dirs = rng.standard_normal((3000, ev_all.shape[1]))
    dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    far = (mu + dirs * sd * rng.uniform(3, 50, (3000, 1))).astype(np.float32)
    return {"held-out": held, "between": between, "far": far}


@pytest.mark.parametrize("path,D,K", NEW_CASES)
def test_new_events_against_f64(pkg, oracle64, path, D, K):
    n_train = 20_000
    ev_all = blobs(pkg, n_train + 10_000, D, seed=21)
    ev = np.ascontiguousarray(ev_all[:n_train])
    cl = fitted_params(pkg, oracle64, ev, K)
    rng = np.random.default_rng(5)
    with engine(pkg, ev, K, path_of(pkg, path)) as eng:
        eng.set_clusters(K, cl)
        held = eng.get_clusters(K)
        for name, x in new_batches(ev_all, n_train, rng).items():
            lab, mr, lp, ll = eng.score(K, x)
            check_f64(held, K, x, lab, mr, lp, f"{path} D={D} K={K} {name}")
            assert abs(ll - float(np.sum(lp, dtype=np.float64))) <= 1e-9 * abs(ll) + 1e-6


# ---- 4. chunking --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("path,D,K", [("tensor", 24, 7), ("tensor", 16, 130), ("simt", 5, 7)])
def test_chunking_is_invisible(pkg, path, D, K):
    ev = blobs(pkg, 10_000, D)
    x = blobs(pkg, 4097, D, seed=99)
    with engine(pkg, ev, K, path_of(pkg, path)) as eng:
        eng.set_clusters(K, mixture(pkg, ev, K))
        for n in (1, 63, 64, 65, 999, 1000, 1001, 4097):
            eng.set_option("score_chunk", 1 << 20)
            whole = eng.score(K, x[:n])
            eng.set_option("score_chunk", 1000)
            eng.score_profile(reset=True)
            parts = eng.score(K, x[:n])
            prof = eng.score_profile()
            assert prof["tensor_chunks"] + prof["simt_chunks"] == (n + 999) // 1000, (n, prof)
            for a, b in zip(whole[:3], parts[:3]):
                np.testing.assert_array_equal(a, b, err_msg=f"n={n}")
            assert abs(whole[3] - parts[3]) <= 1e-9 * abs(whole[3])
        lab, mr, lp, ll = eng.score(K, x[:0])
        assert lab.size == mr.size == lp.size == 0 and ll == 0.0
        full = eng.score(K, x)
        for mask in range(8):
            want = [bool(mask & 1), bool(mask & 2), bool(mask & 4)]
            got = eng.score(K, x, labels=want[0], max_resp=want[1], logp=want[2])
            for i in range(3):
                if want[i]:
                    np.testing.assert_array_equal(got[i], full[i])
                else:
                    assert got[i] is None
            assert abs(got[3] - full[3]) <= 1e-9 * abs(full[3])


# ---- 5. range fallback ---------------------------------------------------------------------------------------------------
def test_range_fallback(pkg):
    D, K = 24, 7
    ev = blobs(pkg, 10_000, D)
    cl = mixture(pkg, ev, K)
    x = blobs(pkg, 3000, D, seed=8)
    sd = ev.std(0)
    x[1500] = ev.mean(0) + 1e5 * sd
    x[1700] = np.nan
    with engine(pkg, ev, K, pkg.PATH_AUTO) as eng:
        eng.set_clusters(K, cl)
        eng.set_option("score_chunk", 1000)
        eng.score_profile(reset=True)
        lab, mr, lp, ll = eng.score(K, x)
        prof = eng.score_profile()
        assert prof["tensor_chunks"] == 2 and prof["simt_chunks"] == 1, prof
        assert lab[1700] == -1 and np.isnan(lp[1700]) and np.isnan(mr[1700])
        ok = np.ones(len(x), bool)
        ok[1700] = False
        check_f64(eng.get_clusters(K), K, x[ok], lab[ok], mr[ok], lp[ok], "range fallback (AUTO)")
        # the re-scored chunk equals a SIMT scoring of the same rows
        eng.set_option("estep_path", pkg.PATH_SIMT)
        eng.set_clusters(K, cl)
        simt = eng.score(K, x[1000:2000])
        np.testing.assert_array_equal(simt[0], lab[1000:2000])
        np.testing.assert_array_equal(simt[2], lp[1000:2000])
        eng.set_option("estep_path", pkg.PATH_TENSOR)
        eng.set_clusters(K, cl)
        with pytest.raises(pkg.GmmError) as e:
            eng.score(K, x)
        assert e.value.code == ERR_STATE


# ---- 6. no interference ---------------------------------------------------------------------------------------------------
# (dimensions the tensor M-step covers: its statistics carry no atomics, so two runs are bit-identical)
@pytest.mark.parametrize("path,D,K", [("tensor", 24, 7), ("tensor", 24, 130), ("simt", 8, 7)])
def test_scoring_leaves_em_state_alone(pkg, path, D, K):
    ev = blobs(pkg, 30_000, D)
    cl = mixture(pkg, ev, K)
    x = blobs(pkg, 5000, D, seed=31)
    res = []
    for do_score in (False, True):
        with engine(pkg, ev, K, path_of(pkg, path)) as eng:
            eng.set_clusters(K, cl)
            eng.estep(K)
            if do_score:
                eng.set_option("score_chunk", 1024)
                eng.score(K, x)
            ll = eng.em_iterations(K, 3)
            got = eng.get_clusters(K, with_memberships=True)
            prof = eng.profile()
            res.append((ll, got, {k: prof[k] for k in ("iterations", "mstep_tensor_launches", "mstep_simt_launches")}))
    (ll0, a, p0), (ll1, b, p1) = res
    assert ll0 == ll1 and p0 == p1, (ll0, ll1, p0, p1)
    for f in pkg.Clusters.FIELDS + ("memberships",):
        np.testing.assert_array_equal(getattr(a, f)[:K], getattr(b, f)[:K], err_msg=f)


# ---- 7. state errors -----------------------------------------------------------------------------------------------------
def test_state_errors(pkg):
    D, K = 24, 7
    ev = blobs(pkg, 5000, D)
    lib = pkg.load_library()
    x = blobs(pkg, 100, D, seed=4)
    ll = C.c_double()

    def raw(eng, K, ptr, n):
        return lib.gmm_score(eng.h, K, ptr, n, None, None, None, C.byref(ll))

    with engine(pkg, ev, K + 3, pkg.PATH_AUTO) as eng:
        eng.set_clusters(K, mixture(pkg, ev, K))
        assert raw(eng, K, x.ctypes.data, len(x)) == 0
        assert raw(eng, K + 1, x.ctypes.data, len(x)) == ERR_STATE
        assert raw(eng, 0, x.ctypes.data, len(x)) == ERR_ARG
        assert raw(eng, K + 4, x.ctypes.data, len(x)) == ERR_ARG
        assert raw(eng, K, x.ctypes.data, -1) == ERR_ARG
        assert raw(eng, K, None, len(x)) == ERR_ARG
        assert raw(eng, K, None, 0) == 0 and ll.value == 0.0
        eng.estep(K)
        eng.mstep(K)
        assert raw(eng, K, x.ctypes.data, len(x)) == ERR_STATE
        eng.estep(K)                                   # the E-step keeps its behaviour between M-step and constants
        assert raw(eng, K, x.ctypes.data, len(x)) == ERR_STATE
        eng.constants(K)
        assert raw(eng, K, x.ctypes.data, len(x)) == 0
    with pytest.raises(pkg.GmmError):
        with engine(pkg, ev, K, pkg.PATH_AUTO) as eng:
            eng.set_option("score_chunk", 0)


# ---- 8. fit workflow ------------------------------------------------------------------------------------------------------
def test_fit_then_score(pkg):
    D = 24
    ev = blobs(pkg, 30_000, D, K_true=4)
    with pkg.Engine(ev, 16) as eng:
        ideal, _, saved = eng.fit(16, 4, 10, 10, with_memberships=True)
        assert ideal == 4
        memb = saved.memberships[:ideal]
        eng.set_clusters(ideal, saved)
        lab, mr, lp, ll = eng.score(ideal, ev)
    # set_clusters rebuilds the operand from the stored float Rinv: only near-ties may go either way
    sure = top_two_gap(memb, 0) > 1e-4
    assert sure.mean() > 0.99
    np.testing.assert_array_equal(lab[sure], memb.argmax(0)[sure])


# ---- 9. many chunks ------------------------------------------------------------------------------------------------------
def test_two_million_events(pkg, oracle64):
    D, K, n_train = 24, 64, 20_000
    ev = blobs(pkg, n_train, D, seed=41)
    x = blobs(pkg, 2_000_000, D, seed=42)
    cl = fitted_params(pkg, oracle64, ev, K, iters=1)
    with engine(pkg, ev, K, pkg.PATH_AUTO) as eng:
        eng.set_clusters(K, cl)
        eng.score_profile(reset=True)
        lab, mr, lp, ll = eng.score(K, x)
        assert eng.score_profile()["tensor_chunks"] == 2
        held = eng.get_clusters(K)
    idx = np.random.default_rng(0).choice(len(x), 50_000, replace=False)
    check_f64(held, K, x[idx], lab[idx], mr[idx], lp[idx], "2M events D=24 K=64")
    assert abs(ll - float(np.sum(lp, dtype=np.float64))) <= 1e-9 * abs(ll)
