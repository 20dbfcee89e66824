"""gmm_score_stats: soft memberships and M-step statistics of new events under a fitted mixture (run with -m gpu on an H100).

On the training shard in one chunk the memberships must be gmm_estep's bit for bit, and the statistics finalised on the host
must give gmm_mstep + gmm_constants' parameters bit for bit where the wgmma M-step forms them.  In chunks and on new events
(held out, between the clusters, up to ~50 standard deviations out) the statistics are held against the exact M-step on the
memberships the call returned (MSTEP_TOL of tests/test_mstep_error_model.py), and the memberships against a float64
posterior.  The cases also cover the per-chunk range fallbacks, the errors, the claim that nothing of the EM state changes,
and EM run over streamed batches.  Every case asserts which E- and M-step kernels ran."""
import numpy as np
import pytest
from scipy.special import logsumexp

from conftest import RUN_MEMB, RUN_RTOL_N, assert_params_close, fitted_params
from test_gpu_score import blobs, mixture, new_batches, ref_logits, top_two_gap
from test_mstep_error_model import MSTEP_TOL, exact_mstep_stats, mstep_errors, standardise

pytestmark = pytest.mark.gpu

ERR_ARG, ERR_STATE = 1, 6
TENSOR_M_D = (4, 8, 12, 16, 20, 24)
PARAMS = ("N", "pi", "constant", "means", "R", "Rinv")


def engine(pkg, ev, Kmax, estep, mstep=None):
    eng = pkg.Engine(ev, Kmax)
    eng.set_option("estep_path", estep)
    eng.set_option("mstep_path", pkg.PATH_AUTO if mstep is None else mstep)
    return eng


def chunks(p):
    return p["estep_tensor_chunks"], p["estep_simt_chunks"], p["mstep_tensor_chunks"], p["mstep_simt_chunks"]


def finalise(pkg, st, sh, K, D, avgvar):
    cl = pkg.Clusters(K, D)
    cl.avgvar[:K] = avgvar[:K]
    pkg.host_finalize(st, sh, cl, K)
    return cl


def check_stats(st, x, mb, sh, K, exact_fp64, what):
    """Statistics against the exact M-step on the memberships the call returned: MSTEP_TOL for the wgmma M-step, 1e-10
    relative to the cluster's raw second moment for the FP64 one."""
    ref = exact_mstep_stats(x, mb, sh)
    e = mstep_errors(st, ref, sh, K)
    print(f"\n[score-stats] {what}: N {e['N']:.2e}  mean {e['mean']:.2e}  R {e['R']:.2e}  worst/bar {e['worst']:.3f}")
    if exact_fp64:
        assert max(e["N"], e["mean"], e["R"]) <= 1e-10, (what, e)
    else:
        assert e["worst"] <= 1.0, (what, e)


# ---- 1. training shard, one chunk: bit-identical to the resident steps ------------------------------------------------------
SHARD = ([("tensor", "tensor", D, K) for D in (8, 16, 24) for K in (1, 7, 64, 130)]
         + [("simt", "tensor", D, 7) for D in (4, 12, 20)]
         + [("simt", "simt", D, K) for D in (5, 32) for K in (7, 130)])


@pytest.mark.parametrize("epath,mpath,D,K", SHARD)
def test_training_shard_matches_resident_steps(pkg, epath, mpath, D, K):
    P = {"tensor": pkg.PATH_TENSOR, "simt": pkg.PATH_SIMT}
    ev = blobs(pkg, 20_011, D)
    with engine(pkg, ev, K, P[epath], P[mpath]) as eng:
        eng.set_clusters(K, mixture(pkg, ev, K))
        ll = eng.estep(K)
        eng.score_stats_profile(reset=True)
        st, sh, mb = eng.score_stats(K, ev, memberships=True)
        prof = eng.score_stats_profile()
        assert chunks(prof) == ((1, 0) if epath == "tensor" else (0, 1)) + ((1, 0) if mpath == "tensor" else (0, 1)), prof
        before = eng.get_clusters(K, with_memberships=True)
        np.testing.assert_array_equal(mb, before.memberships[:K])
        assert abs(st[-1] - ll) <= 1e-6 * abs(ll), (st[-1], ll)
        if D in TENSOR_M_D:
            np.testing.assert_array_equal(sh, standardise(ev)[0])
        else:
            np.testing.assert_allclose(sh, ev.astype(np.float64).mean(0), rtol=1e-12, atol=1e-12)
        eng.mstep(K)
        eng.constants(K)
        res = eng.get_clusters(K)
    got = finalise(pkg, st, sh, K, D, before.avgvar)
    if mpath == "tensor":
        for f in PARAMS:
            np.testing.assert_array_equal(getattr(got, f)[:K], getattr(res, f)[:K], err_msg=f)
    else:
        # the FP64 SIMT M-step adds per-block partial sums with atomics: their order, and so the last bits, vary from run to run
        check_stats(st, ev, mb, sh, K, True, f"shard SIMT D={D} K={K}")
        assert_params_close(got, res, K, rtol=1e-5)


@pytest.mark.parametrize("estep", ["tensor", "simt"])
def test_training_shard_kmax_above_k(pkg, estep):
    """A Kmax = 100 context run at K = 40: the same bit-identity."""
    D, K = 24, 40
    ev = blobs(pkg, 20_011, D)
    with engine(pkg, ev, 100, pkg.PATH_TENSOR if estep == "tensor" else pkg.PATH_SIMT, pkg.PATH_TENSOR) as eng:
        eng.set_clusters(100, mixture(pkg, ev, 100))
        eng.estep(100)
        eng.set_clusters(K, mixture(pkg, ev, K))
        ll = eng.estep(K)
        eng.score_stats_profile(reset=True)
        st, sh, mb = eng.score_stats(K, ev, memberships=True)
        assert chunks(eng.score_stats_profile()) == ((1, 0) if estep == "tensor" else (0, 1)) + (1, 0)
        before = eng.get_clusters(K, with_memberships=True)
        np.testing.assert_array_equal(mb, before.memberships[:K])
        assert abs(st[-1] - ll) <= 1e-6 * abs(ll)
        eng.mstep(K)
        eng.constants(K)
        res = eng.get_clusters(K)
    got = finalise(pkg, st, sh, K, D, before.avgvar)
    for f in PARAMS:
        np.testing.assert_array_equal(getattr(got, f)[:K], getattr(res, f)[:K], err_msg=f)


# ---- 2. chunked ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("epath,D,K", [("tensor", 24, 7), ("tensor", 16, 130), ("simt", 12, 7), ("simt", 5, 7)])
@pytest.mark.parametrize("chunk", [1, 33, 4097, 667])
def test_chunked(pkg, epath, D, K, chunk):
    n = 300 if chunk == 1 else 20_011             # 667: 30 full chunks and a last one of 1 event
    ev = blobs(pkg, n, D)
    with engine(pkg, ev, K, pkg.PATH_TENSOR if epath == "tensor" else pkg.PATH_SIMT) as eng:
        eng.set_clusters(K, mixture(pkg, ev, K))
        eng.estep(K)
        memb = eng.get_clusters(K, with_memberships=True).memberships[:K]
        eng.set_option("score_chunk", chunk)
        eng.score_stats_profile(reset=True)
        st, sh, mb = eng.score_stats(K, ev, memberships=True)
        e_t, e_s, m_t, m_s = chunks(eng.score_stats_profile())
    nch = -(-n // chunk)
    assert (e_t, e_s) == ((nch, 0) if epath == "tensor" else (0, nch))
    tensor_m = D in TENSOR_M_D
    assert (m_t, m_s) == ((nch, 0) if tensor_m else (0, nch))
    np.testing.assert_array_equal(mb, memb)
    check_stats(st, ev, mb, sh, K, not tensor_m, f"chunk={chunk} {epath} D={D} K={K}")


# ---- 3. new events ------------------------------------------------------------------------------------------------------
NEW = [("tensor", D, 7) for D in (8, 16, 24)] + [("tensor", 24, 130), ("simt", 5, 7), ("simt", 24, 7)]


@pytest.mark.parametrize("epath,D,K", NEW)
def test_new_events(pkg, oracle64, epath, D, K):
    n_train = 20_000
    ev_all = blobs(pkg, n_train + 10_000, D, seed=21)
    ev = np.ascontiguousarray(ev_all[:n_train])
    cl = fitted_params(pkg, oracle64, ev, K)
    rng = np.random.default_rng(5)
    with engine(pkg, ev, K, pkg.PATH_TENSOR if epath == "tensor" else pkg.PATH_SIMT) as eng:
        eng.set_clusters(K, cl)
        held = eng.get_clusters(K)
        eng.set_option("score_chunk", 1000)
        for name, x in new_batches(ev_all, n_train, rng).items():
            what = f"{epath} D={D} K={K} {name}"
            eng.score_stats_profile(reset=True)
            st, sh, mb = eng.score_stats(K, x, memberships=True)
            e_t, e_s, m_t, m_s = chunks(eng.score_stats_profile())
            nch = -(-len(x) // 1000)
            assert e_t + e_s == nch and m_t + m_s == nch and (e_s == 0 if epath == "tensor" else e_t == 0), (what, e_t, e_s, m_t, m_s)
            # memberships against the float64 posterior, at gmm_score's bars
            L = ref_logits(held, K, x)
            lse = logsumexp(L, axis=1)
            post = np.exp(L - lse[:, None]).T
            # (a float32 logit of magnitude |l| carries ~1e-7 |l| of rounding: the bar grows with the larger of l_k and l_max)
            rtol = 1e-4 + 1e-6 * np.maximum(np.abs(L), np.abs(L.max(1))[:, None]).T
            dm = np.abs(mb.astype(np.float64) - post) / (1e-6 + rtol * post)
            assert dm.max() <= 1.0, (what, float(dm.max()))
            assert abs(st[-1] - lse.sum()) <= 1e-4 * np.sum(1 + np.abs(lse)), (what, st[-1], lse.sum())
            # the statistics against the exact M-step on the memberships the call returned (isolates the M-step)
            check_stats(st, x, mb, sh, K, m_t == 0, what)
            # consistency with gmm_score
            lab, mr, lp, ll = eng.score(K, x)
            if K <= 64:
                np.testing.assert_array_equal(mb.max(0), mr, err_msg=what)
            differ = top_two_gap(mb, 0) > 0
            np.testing.assert_array_equal(mb.argmax(0)[differ], lab[differ], err_msg=what)


# ---- 4. range ----------------------------------------------------------------------------------------------------------
def test_range_fallbacks(pkg):
    D, K = 24, 7
    ev = blobs(pkg, 10_000, D)
    cl = mixture(pkg, ev, K)
    sf, scale, _, zb = standardise(ev)
    assert zb <= 64
    # training rows: every chunk inside zb but for the one event moved past it (far inside 2^14)
    x = ev[np.random.default_rng(8).permutation(len(ev))[:3000]].copy()
    x[1500, 0] = np.float32(sf[0] + 1.5 * zb * scale[0])
    with engine(pkg, ev, K, pkg.PATH_AUTO) as eng:
        eng.set_clusters(K, cl)
        eng.set_option("score_chunk", 1000)
        eng.score_stats_profile(reset=True)
        st, sh, mb = eng.score_stats(K, x, memberships=True)
        assert chunks(eng.score_stats_profile()) == (3, 0, 2, 1)
        check_stats(st, x, mb, sh, K, False, "one chunk past zb")
        # the chunk past zb alone: FP64 statistics
        eng.score_stats_profile(reset=True)
        st1, _, mb1 = eng.score_stats(K, x[1000:2000], memberships=True)
        assert chunks(eng.score_stats_profile()) == (1, 0, 0, 1)
        check_stats(st1, x[1000:2000], mb1, sh, K, True, "chunk past zb")
        eng.set_option("mstep_path", pkg.PATH_TENSOR)
        with pytest.raises(pkg.GmmError) as e:
            eng.score_stats(K, x)
        assert e.value.code == ERR_STATE
        _, _, mb_only = eng.score_stats(K, x, stats=False, memberships=True)  # no M-step: nothing to refuse
        np.testing.assert_array_equal(mb_only, mb)
        eng.set_option("mstep_path", pkg.PATH_AUTO)
        far = x.copy()
        far[2500] = (sf + 1e5 * scale).astype(np.float32)          # beyond 2^14: the SIMT E-step (and the FP64 M-step)
        eng.score_stats_profile(reset=True)
        st2, _, mb2 = eng.score_stats(K, far, memberships=True)
        assert chunks(eng.score_stats_profile()) == (2, 1, 1, 2)
        check_stats(st2, far, mb2, sh, K, False, "one chunk beyond 2^14")
        eng.set_option("estep_path", pkg.PATH_TENSOR)
        with pytest.raises(pkg.GmmError) as e:
            eng.score_stats(K, far)
        assert e.value.code == ERR_STATE
        bad = x.copy()
        bad[1700, 3] = np.nan
        with pytest.raises(pkg.GmmError) as e:
            eng.score_stats(K, bad)
        assert e.value.code == ERR_ARG


# ---- 5. no interference -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [7, 130])
def test_em_state_untouched(pkg, K):
    D = 24
    ev = blobs(pkg, 30_000, D)
    cl = mixture(pkg, ev, K)
    x = blobs(pkg, 5000, D, seed=31)
    res = []
    for interleave in (False, True):
        with engine(pkg, ev, K, pkg.PATH_AUTO) as eng:
            eng.set_clusters(K, cl)
            eng.estep(K)
            eng.set_option("score_chunk", 1024)
            lls = []
            for _ in range(3):
                if interleave:
                    eng.score_stats(K, x, memberships=True)
                    eng.score_stats(K, ev[:3000], stats=True)
                lls.append(eng.em_iterations(K, 2))
            got = eng.get_clusters(K, with_memberships=True)
            prof = eng.profile()
            res.append((lls, got, {k: prof[k] for k in ("iterations", "mstep_tensor_launches", "mstep_simt_launches")},
                        eng.score_profile()))
    (ll0, a, p0, s0), (ll1, b, p1, s1) = res
    assert ll0 == ll1 and p0 == p1 and s0 == s1, (ll0, ll1, p0, p1, s0, s1)
    for f in pkg.Clusters.FIELDS + ("memberships",):
        np.testing.assert_array_equal(getattr(a, f)[:K], getattr(b, f)[:K], err_msg=f)


# ---- 6. errors ----------------------------------------------------------------------------------------------------------
def test_errors(pkg):
    D, K = 24, 7
    ev = blobs(pkg, 5000, D)
    lib = pkg.load_library()
    x = blobs(pkg, 100, D, seed=4)
    F = 1 + D + D * (D + 1) // 2
    st = np.full(K * F + 1, 7.0)
    sh = np.zeros(D)
    mb = np.zeros((K, len(x)), np.float32)

    def raw(eng, K, ptr, n, s=st.ctypes.data, m=None):
        return lib.gmm_score_stats(eng.h, K, ptr, n, s, sh.ctypes.data, m)

    with engine(pkg, ev, K + 3, pkg.PATH_AUTO) as eng:
        eng.set_clusters(K, mixture(pkg, ev, K))
        assert raw(eng, K, x.ctypes.data, len(x)) == 0
        assert raw(eng, K, x.ctypes.data, len(x), s=None, m=mb.ctypes.data) == 0
        assert raw(eng, K + 1, x.ctypes.data, len(x)) == ERR_STATE
        assert raw(eng, 0, x.ctypes.data, len(x)) == ERR_ARG
        assert raw(eng, K + 4, x.ctypes.data, len(x)) == ERR_ARG
        assert raw(eng, K, x.ctypes.data, -1) == ERR_ARG
        assert raw(eng, K, None, len(x)) == ERR_ARG
        assert raw(eng, K, x.ctypes.data, len(x), s=None, m=None) == ERR_ARG
        sh[:] = 0
        assert raw(eng, K, None, 0) == 0
        assert np.all(st == 0.0)
        np.testing.assert_array_equal(sh, standardise(ev)[0])
        eng.estep(K)
        eng.mstep(K)
        assert raw(eng, K, x.ctypes.data, len(x)) == ERR_STATE
        eng.constants(K)
        assert raw(eng, K, x.ctypes.data, len(x)) == 0
        y = x.copy()
        y[50, 2] = np.inf
        assert raw(eng, K, y.ctypes.data, len(y)) == ERR_ARG
    # a SIMT-only context after gmm_set_clusters has no centre yet: a single-rank context fixes it here
    ev5 = blobs(pkg, 5000, 5)
    with engine(pkg, ev5, K, pkg.PATH_SIMT) as eng:
        eng.set_clusters(K, mixture(pkg, ev5, K))
        st0, sh0, _ = eng.score_stats(K, ev5[:0])
        assert np.all(st0 == 0.0)
        np.testing.assert_allclose(sh0, ev5.astype(np.float64).mean(0), rtol=1e-12, atol=1e-12)


# ---- 7. EM over streamed batches ------------------------------------------------------------------------------------------
def test_streamed_em_matches_resident(pkg):
    D, K, T, n, batch = 24, 16, 10, 200_000, 32_768
    ev = blobs(pkg, n, D, seed=77, K_true=8)
    with pkg.Engine(ev, K) as res_eng:
        seed = res_eng.seed(K)
        res_eng.estep(K)
        res_eng.em_iterations(K, T)
        ref = res_eng.get_clusters(K, with_memberships=True)
    # the streaming context holds only the first batch: the data of every iteration is streamed from the host
    with pkg.Engine(np.ascontiguousarray(ev[:batch]), K) as eng:
        eng.set_clusters(K, seed)
        cl = eng.get_clusters(K)
        eng.score_stats_profile(reset=True)
        for _ in range(T):
            total, shift = None, None
            for b0 in range(0, n, batch):
                st, sh, _ = eng.score_stats(K, ev[b0:b0 + batch])
                total = st if total is None else total + st
                assert shift is None or np.array_equal(shift, sh)
                shift = sh
            pkg.host_finalize(total, shift, cl, K)
            eng.set_clusters(K, cl)
        prof = eng.score_stats_profile()
        assert prof["estep_tensor_chunks"] + prof["estep_simt_chunks"] == T * (-(-n // batch)), prof
        _, _, memb = eng.score_stats(K, ev, stats=False, memberships=True)
        got = eng.get_clusters(K)
    assert_params_close(got, ref, K, rtol_N=RUN_RTOL_N)
    np.testing.assert_allclose(memb, ref.memberships[:K], **RUN_MEMB)


def test_raw_abi_rows_land_cluster_major(pkg):
    """memberships + k * n + e0: a chunk boundary inside a row of the caller's [K][n] array."""
    D, K = 16, 5
    ev = blobs(pkg, 5000, D)
    with engine(pkg, ev, K, pkg.PATH_AUTO) as eng:
        eng.set_clusters(K, mixture(pkg, ev, K))
        eng.set_option("score_chunk", 777)
        mb = np.full((K, 2500), -1.0, np.float32)
        sh = np.zeros(D)
        assert pkg.load_library().gmm_score_stats(eng.h, K, ev.ctypes.data, 2500, None, sh.ctypes.data, mb.ctypes.data) == 0
        eng.set_option("score_chunk", 1 << 20)
        _, _, whole = eng.score_stats(K, ev[:2500], stats=False, memberships=True)
    np.testing.assert_array_equal(mb, whole)
