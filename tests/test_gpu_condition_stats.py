"""gmm_condition_stats: the expected full-D M-step statistics of events measured on a subset of the dimensions, so that EM can
fit a mixture across the tubes of a split panel (run with -m gpu on an H100).

With every dimension observed the call is gmm_score_stats bit for bit.  Otherwise the memberships are the marginal posteriors
of gmm_condition (its max_resp bit for bit), and the statistics are held against the float64 restatement of gmm.h
(tests/_condition_stats_ref.py) applied to the memberships the call returned, which isolates the M-step and the expansion from
the E-step's rounding: MSTEP_TOL (tests/test_mstep_error_model.py) where the wgmma M-step formed them, 1e-10 relative where
the FP64 one did.  Every case asserts which M-step kernel ran.  The workflow case runs EM over three tubes that share a
backbone, each iteration against a float64 EM with missing data, and checks the fit against the mixture that drew the tubes."""
import numpy as np
import pytest

import _condition_stats_ref as ref
from conftest import RUN_MEMB, RUN_RTOL_N, assert_params_close
from test_gpu_condition import events, model
from test_mstep_error_model import mstep_errors, standardise

pytestmark = pytest.mark.gpu

ERR_ARG, ERR_STATE = 1, 6


def context(pkg, cl, K, n=12_000, seed=1, Kmax=None, estep=None, mstep=None):
    """A context whose shard is drawn around the model, so that its centre and range cover rows drawn the same way."""
    ev = events(cl, K, n, seed, far=0.0)
    eng = pkg.Engine(ev, Kmax or K)
    if estep is not None:
        eng.set_option("estep_path", estep)
    if mstep is not None:
        eng.set_option("mstep_path", mstep)
    eng.set_clusters(K, cl)
    return eng, ev


def m_chunks(p):
    return p["mstep_tensor_chunks"], p["mstep_simt_chunks"]


def check_stats(st, cl, K, obs, xo, mb, sh, fp64, what):
    """Statistics against the restatement's expansion of the returned memberships."""
    want = ref.expected_stats(cl, K, obs, xo, mb, sh)
    e = mstep_errors(st, want, sh, K)
    print(f"\n[cond-stats] {what}: N {e['N']:.2e}  mean {e['mean']:.2e}  R {e['R']:.2e}  worst/bar {e['worst']:.3f}")
    if fp64:
        assert max(e["N"], e["mean"], e["R"]) <= 1e-10, (what, e)
    else:
        assert e["worst"] <= 1.0, (what, e)


def obs_sets(D):
    """One dimension, all but one, a non-contiguous set, and a backbone of the first half plus the last dimension."""
    s = {(D // 2,), tuple(d for d in range(D) if d != D // 3), tuple(range(0, D, 2)), tuple(range(D // 2)) + (D - 1,)}
    return sorted(t for t in s if 0 < len(t) < D)


def top_two_gap(m):
    s = np.sort(m, axis=0)
    return s[-1] - s[-2]


# ---- 1. every dimension observed = gmm_score_stats -----------------------------------------------------------------------
@pytest.mark.parametrize("epath,D,K", [("tensor", 24, 7), ("tensor", 16, 130), ("simt", 24, 7), ("simt", 5, 7), ("simt", 32, 3)])
def test_full_set_is_score_stats(pkg, epath, D, K):
    cl = model(pkg, K, D, seed=D * 10 + K)
    eng, ev = context(pkg, cl, K, n=20_011, estep=pkg.PATH_TENSOR if epath == "tensor" else pkg.PATH_SIMT)
    with eng:
        eng.set_option("score_chunk", 4096)
        st, sh, mb = eng.score_stats(K, ev, memberships=True)
        ps = eng.score_stats_profile()
        eng.condition_stats_profile(reset=True)
        st2, sh2, mb2 = eng.condition_stats(K, np.arange(D), ev, memberships=True)
        assert eng.score_stats_profile() == ps
        prof = eng.condition_stats_profile()
    nch = -(-len(ev) // 4096)
    assert sum(m_chunks(prof)) == nch, prof
    np.testing.assert_array_equal(mb2, mb)
    np.testing.assert_array_equal(sh2, sh)
    assert abs(st2[-1] - st[-1]) <= 1e-12 * abs(st[-1])              # (the block sums are added by atomics)
    if prof["mstep_simt_chunks"] == 0:
        np.testing.assert_array_equal(st2[:-1], st[:-1])
    else:                                                             # the FP64 M-step's atomics: order, so last bits, vary
        F = 1 + D + D * (D + 1) // 2
        scale = np.abs(st[:-1]).reshape(K, F).max(1).repeat(F)
        assert np.all(np.abs(st2[:-1] - st[:-1]) <= 1e-12 * scale)


# ---- 2. the marginal posteriors are gmm_condition's ---------------------------------------------------------------------
@pytest.mark.parametrize("D,K", [(8, 3), (24, 64), (32, 65), (4, 512)])
def test_marginal_posteriors(pkg, D, K):
    cl = model(pkg, K, D, seed=D + K)
    eng, ev = context(pkg, cl, K, n=20_000, estep=pkg.PATH_SIMT)
    obs = tuple(range(0, D, 2)) if D > 4 else (1, 2)
    xo = np.ascontiguousarray(ev[:, obs])
    with eng:
        lab, mr, _, _, _, ll = eng.condition(K, obs, xo, mean=False)
        st, _, mb = eng.condition_stats(K, obs, xo, memberships=True)
        np.testing.assert_array_equal(mb.max(0), mr)
        np.testing.assert_array_equal(mb[lab, np.arange(len(xo))], mr)
        differ = top_two_gap(mb) > 0 if K > 1 else np.ones(len(xo), bool)
        np.testing.assert_array_equal(mb.argmax(0)[differ], lab[differ])
        assert abs(st[-1] - ll) <= 1e-9 * abs(ll), (st[-1], ll)
        for chunk in (1, 33, 4097):
            eng.set_option("score_chunk", chunk)
            n = 300 if chunk == 1 else len(xo)
            _, _, m = eng.condition_stats(K, obs, xo[:n], stats=False, memberships=True)
            np.testing.assert_array_equal(m, mb[:, :n], err_msg=f"chunk {chunk}")
        eng.set_option("score_chunk", 1 << 20)
        _, _, a = eng.condition_stats(K, obs, xo[:7_777], stats=False, memberships=True)
        _, _, b = eng.condition_stats(K, obs, xo[7_777:], stats=False, memberships=True)
        np.testing.assert_array_equal(np.concatenate([a, b], axis=1), mb)


# ---- 3. the statistics against the float64 restatement --------------------------------------------------------------------
RESTATE = [(D, K) for D in (3, 8, 16, 24, 32) for K in (1, 3, 64, 65)] + [(4, 512)]


@pytest.mark.parametrize("D,K", RESTATE)
def test_matches_restatement(pkg, D, K):
    cl = model(pkg, K, D, seed=D * 1000 + K)
    # (Kmax >= 2: at D = 3 a one-cluster context's statistics buffer cannot hold the column moments that fix its centre,
    # a limit gmm_score_stats shares)
    eng, ev = context(pkg, cl, K, n=8_000, seed=D + K, Kmax=max(K, 2))
    with eng:
        for obs in obs_sets(D):
            xo = np.ascontiguousarray(ev[:, obs])
            eng.condition_stats_profile(reset=True)
            st, sh, mb = eng.condition_stats(K, obs, xo, memberships=True)
            m_t, m_s = m_chunks(eng.condition_stats_profile())
            assert m_t + m_s == 1
            check_stats(st, cl, K, obs, xo, mb, sh, m_t == 0, f"D={D} K={K} obs={obs}")
            post, lp = ref.marginal_posterior(cl, K, obs, xo)
            np.testing.assert_allclose(mb, post, **RUN_MEMB)
            assert abs(st[-1] - lp.sum()) <= 1e-4 * np.sum(1 + np.abs(lp)), (st[-1], lp.sum())


@pytest.mark.parametrize("D,K", [(24, 64), (8, 65), (32, 3)])
@pytest.mark.parametrize("chunk", [1, 33, 4097])
def test_restatement_in_chunks(pkg, D, K, chunk):
    cl = model(pkg, K, D, seed=7 * D + K)
    eng, ev = context(pkg, cl, K, n=9_000, seed=3)
    n = 300 if chunk == 1 else len(ev)
    obs = tuple(range(D // 2)) + (D - 1,)
    xo = np.ascontiguousarray(ev[:n, obs])
    with eng:
        eng.set_option("score_chunk", chunk)
        eng.condition_stats_profile(reset=True)
        st, sh, mb = eng.condition_stats(K, obs, xo, memberships=True)
        m_t, m_s = m_chunks(eng.condition_stats_profile())
    assert m_t + m_s == -(-n // chunk) and (m_t == 0 or m_s == 0), (m_t, m_s)
    check_stats(st, cl, K, obs, xo, mb, sh, m_t == 0, f"chunk={chunk} D={D} K={K}")


# ---- 4. kernel selection ----------------------------------------------------------------------------------------------------
def test_kernel_selection(pkg):
    D, K = 24, 7
    cl = model(pkg, K, D, seed=4)
    eng, ev = context(pkg, cl, K, n=10_000)
    obs = tuple(range(0, D, 2))
    x = ev[:3000].copy()
    sf, scale, _, zb = standardise(ev)
    with eng:
        eng.set_option("score_chunk", 1000)
        eng.condition_stats_profile(reset=True)
        st, sh, mb = eng.condition_stats(K, obs, x[:, obs], memberships=True)
        assert m_chunks(eng.condition_stats_profile()) == (3, 0)
        check_stats(st, cl, K, obs, x[:, obs], mb, sh, False, "D=24 wgmma")
        far = x.copy()
        far[1500, obs[1]] = np.float32(sf[obs[1]] + 1.5 * zb * scale[obs[1]])   # one observed coordinate past zb
        eng.condition_stats_profile(reset=True)
        st, sh, mb = eng.condition_stats(K, obs, far[:, obs], memberships=True)
        assert m_chunks(eng.condition_stats_profile()) == (2, 1)
        check_stats(st, cl, K, obs, far[:, obs], mb, sh, False, "one chunk past zb")
        eng.condition_stats_profile(reset=True)
        st1, _, mb1 = eng.condition_stats(K, obs, far[1000:2000, obs], memberships=True)
        assert m_chunks(eng.condition_stats_profile()) == (0, 1)
        check_stats(st1, cl, K, obs, far[1000:2000, obs], mb1, sh, True, "the chunk past zb alone")
        eng.set_option("mstep_path", pkg.PATH_TENSOR)
        with pytest.raises(pkg.GmmError) as e:
            eng.condition_stats(K, obs, far[:, obs])
        assert e.value.code == ERR_STATE
        _, _, only = eng.condition_stats(K, obs, far[:, obs], stats=False, memberships=True)   # no M-step: nothing to refuse
        np.testing.assert_array_equal(only, mb)
    cl32 = model(pkg, 3, 32, seed=5)
    eng, ev = context(pkg, cl32, 3, n=5_000)
    with eng:
        eng.set_option("score_chunk", 1000)
        eng.condition_stats_profile(reset=True)
        obs = tuple(range(16))
        st, sh, mb = eng.condition_stats(3, obs, ev[:, obs], memberships=True)
        assert m_chunks(eng.condition_stats_profile()) == (0, 5)
        check_stats(st, cl32, 3, obs, ev[:, obs], mb, sh, True, "D=32 FP64")


# ---- 5. EM over a split panel -------------------------------------------------------------------------------------------------
PANEL_D, PANEL_K, TUBE_N = 12, 4, 300_000
BACKBONE = tuple(range(6))
TUBES = [BACKBONE + (6 + 2 * t, 7 + 2 * t) for t in range(3)]


def truth(pkg):
    D, K = PANEL_D, PANEL_K
    rng = np.random.default_rng(2011)
    cl = pkg.Clusters(K, D)
    cl.means[...] = (rng.standard_normal((K, D)) * 6.0).astype(np.float32)
    for k in range(K):
        A = rng.standard_normal((D, D))
        cl.R[k] = (A @ A.T / D + 0.5 * np.eye(D)).astype(np.float32)
    cl.pi[...] = np.array([0.1, 0.2, 0.3, 0.4], np.float32)
    cl.N[...] = cl.pi * 1e6
    return consistent(cl, K)


def consistent(cl, K):
    for k in range(K):
        R64 = cl.R[k].astype(np.float64)
        cl.Rinv[k] = np.linalg.inv(R64).astype(np.float32)
        cl.constant[k] = np.float32(-0.5 * cl.D * np.log(2 * np.pi) - 0.5 * np.linalg.slogdet(R64)[1])
    return cl


def panel(pkg):
    """The truth, three tubes drawn from it by gmm_sample (their observed columns), a held-out complete tube and a complete
    shard for the fitting context's centre."""
    tr = truth(pkg)
    with pkg.Engine(pkg.synth.make_blobs(4096, PANEL_D, 4, seed=1), PANEL_K) as eng:
        eng.set_clusters(PANEL_K, tr)
        x, _ = eng.sample(PANEL_K, 3 * TUBE_N + 70_000, seed=99)
    tubes = [np.ascontiguousarray(x[t * TUBE_N:(t + 1) * TUBE_N]) for t in range(3)]
    return tr, tubes, x[3 * TUBE_N:3 * TUBE_N + 50_000], np.ascontiguousarray(x[3 * TUBE_N + 50_000:])


def start(pkg, tr):
    rng = np.random.default_rng(5)
    cl = tr.copy()
    cl.means[...] += (rng.standard_normal(cl.means.shape) * 0.7).astype(np.float32)
    cl.R[...] *= np.float32(1.5)
    cl.pi[...] = np.float32(1.0 / PANEL_K)
    cl.N[...] = np.float32(1e6 / PANEL_K)
    cl.avgvar[...] = 0.0
    return consistent(cl, PANEL_K)


def ref_step(pkg, cur, parts, sh):
    """One float64 EM iteration with missing data from the parameters `cur`: parts = [(obs, rows)]."""
    K = PANEL_K
    total = 0.0
    for obs, xo in parts:
        post, lp = ref.marginal_posterior(cur, K, obs, xo)
        total = total + ref.expected_stats(cur, K, obs, xo, post, sh, ll=lp.sum())
    nxt = cur.copy()
    pkg.host_finalize(total, sh, nxt, K)
    return nxt, total


def test_split_panel_em(pkg):
    D, K, T = PANEL_D, PANEL_K, 40
    tr, tubes, hold, shard = panel(pkg)
    parts = [(obs, np.ascontiguousarray(x[:, obs])) for obs, x in zip(TUBES, tubes)]
    with pkg.Engine(shard, K) as eng:
        cur = start(pkg, tr)
        eng.set_clusters(K, cur)
        lls, worst = [], 0.0
        for it in range(T):
            total, shift = 0.0, None
            for obs, xo in parts:
                st, sh, _ = eng.condition_stats(K, obs, xo)
                assert shift is None or np.array_equal(shift, sh)
                shift = sh
                total = total + st
            lls.append(total[-1])
            nxt = cur.copy()
            pkg.host_finalize(total, shift, nxt, K)
            want, rtotal = ref_step(pkg, cur, parts, shift)
            assert abs(total[-1] - rtotal[-1]) <= 1e-5 * abs(rtotal[-1]), (it, total[-1], rtotal[-1])
            assert_params_close(nxt, want, K, rtol_N=RUN_RTOL_N)
            worst = max(worst, float(np.abs(nxt.means[:K] - want.means[:K]).max() / max(1.0, np.abs(want.means[:K]).max())))
            eng.set_clusters(K, nxt)
            cur = nxt
        print(f"\n[split-panel] worst relative mean deviation from the float64 EM in one iteration: {worst:.2e}")
        print(f"[split-panel] observed-data log-likelihood: {lls[0]:.6e} -> {lls[-1]:.6e}")
        # (b) EM does not decrease the observed-data log-likelihood
        for a, b in zip(lls, lls[1:]):
            assert b >= a - 1e-6 * abs(a), (a, b)
        # (c) pi and the means against the truth
        n_all = 3 * TUBE_N
        order = [int(np.argmin(np.abs(cur.means[:K] - tr.means[k]).sum(1))) for k in range(K)]
        assert sorted(order) == list(range(K)), order
        for k, j in enumerate(order):
            p = float(tr.pi[k])
            assert abs(float(cur.pi[j]) - p) <= 4 * np.sqrt(p * (1 - p) / n_all), (k, cur.pi[j], p)
            n_d = np.array([n_all if d in BACKBONE else TUBE_N for d in range(D)]) * p
            se = np.sqrt(np.diag(tr.R[k]).astype(np.float64) / n_d)
            dev = np.abs(cur.means[j].astype(np.float64) - tr.means[k]) / se
            assert dev.max() <= 6, (k, dev)
            # (d) variances and covariances of the pairs measured together
            for a in range(D):
                for b in range(a + 1):
                    together = [t for t, obs in enumerate(TUBES) if a in obs and b in obs]
                    if not together:
                        continue
                    n_ab = len(together) * TUBE_N * p
                    Rt = tr.R[k].astype(np.float64)
                    se_ab = np.sqrt((Rt[a, a] * Rt[b, b] + Rt[a, b] ** 2) / n_ab)
                    assert abs(float(cur.R[j][a, b]) - Rt[a, b]) <= 6 * se_ab, (k, a, b, cur.R[j][a, b], Rt[a, b])
        # (e) gmm_condition with the fit, on a held-out tube's backbone, is calibrated on its markers
        mis = [d for d in range(D) if d not in BACKBONE]
        _, _, _, mean, var, _ = eng.condition(K, BACKBONE, np.ascontiguousarray(hold[:, BACKBONE]), labels=False, max_resp=False,
                                              logp=False, var=True)
    z2 = ((hold[:, mis].astype(np.float64) - mean) ** 2 / var).mean(0)
    print(f"[split-panel] held-out mean z^2 per marker: {np.round(z2, 4).tolist()}")
    assert np.all(np.abs(z2 - 1.0) <= 0.05), z2


def test_split_panel_with_a_complete_tube(pkg):
    """Tube 0 complete through gmm_score_stats, the others through gmm_condition_stats: the sum is the same EM iteration."""
    K, T = PANEL_K, 10
    tr, tubes, _, shard = panel(pkg)
    parts = [(tuple(range(PANEL_D)), tubes[0])] + [(obs, np.ascontiguousarray(x[:, obs])) for obs, x in zip(TUBES[1:], tubes[1:])]
    with pkg.Engine(shard, K) as eng:
        cur = start(pkg, tr)
        eng.set_clusters(K, cur)
        for it in range(T):
            st, shift, _ = eng.score_stats(K, tubes[0])
            total = st
            for obs, xo in parts[1:]:
                st, sh, _ = eng.condition_stats(K, obs, xo)
                assert np.array_equal(sh, shift)
                total = total + st
            nxt = cur.copy()
            pkg.host_finalize(total, shift, nxt, K)
            want, _ = ref_step(pkg, cur, parts, shift)
            assert_params_close(nxt, want, K, rtol_N=RUN_RTOL_N)
            eng.set_clusters(K, nxt)
            cur = nxt


# ---- 6. nothing else changes --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [7, 130])
def test_no_interference(pkg, K):
    D = 24
    cl = model(pkg, K, D, seed=K)
    ev = events(cl, K, 30_000, seed=2, far=0.0)
    x = events(cl, K, 5_000, seed=3, far=0.0)
    obs = (0, 3, 4, 9, 17, 23)
    res = []
    for interleave in (False, True):
        with pkg.Engine(ev, K) as eng:
            eng.set_clusters(K, cl)
            eng.estep(K)
            eng.set_option("score_chunk", 1024)
            lls = []
            for _ in range(3):
                if interleave:
                    profs = (eng.profile(), eng.score_profile(), eng.score_stats_profile(), eng.sample_profile(), eng.condition_profile())
                    eng.condition_stats(K, obs, x[:, obs], memberships=True)
                    eng.condition_stats(K, np.arange(D), ev[:3000])
                    assert (eng.profile(), eng.score_profile(), eng.score_stats_profile(), eng.sample_profile(),
                            eng.condition_profile()) == profs
                lls.append(eng.em_iterations(K, 2))
            got = eng.get_clusters(K, with_memberships=True)
            lab, mr, lp, _ = eng.score(K, x)
            res.append((lls, got, lab, mr, lp))
    (l0, a, *s0), (l1, b, *s1) = res
    assert l0 == l1, (l0, l1)
    for f in pkg.Clusters.FIELDS + ("memberships",):
        np.testing.assert_array_equal(getattr(a, f)[:K], getattr(b, f)[:K], err_msg=f)
    for u, v in zip(s0, s1):
        np.testing.assert_array_equal(u, v)


# ---- 7. errors --------------------------------------------------------------------------------------------------------------
def test_errors(pkg):
    D, K, Kmax = 4, 4, 8
    good = model(pkg, K, D, seed=3)
    eng, ev = context(pkg, good, K, n=4096, Kmax=Kmax)
    lib = pkg.load_library()
    F = 1 + D + D * (D + 1) // 2
    x = np.ascontiguousarray(ev[:16, [0, 2]])
    st = np.full(K * F + 1, 7.0)
    sh = np.zeros(D)
    mb = np.zeros((K, 16), np.float32)
    ptr = lambda a: a.ctypes.data if a is not None else None  # noqa: E731

    def raw(K, obs, n_obs, rows, n, s=st, m=None):
        return lib.gmm_condition_stats(eng.h, K, ptr(obs), n_obs, ptr(rows), n, ptr(s), sh.ctypes.data, ptr(m))

    obs = np.array([0, 2], np.int32)
    with eng:
        assert raw(K, obs, 2, x, 16) == 0
        assert raw(K, obs, 2, x, 16, s=None, m=mb) == 0
        assert raw(0, obs, 2, x, 16) == ERR_ARG
        assert raw(Kmax + 1, obs, 2, x, 16) == ERR_ARG
        assert raw(K, obs, 2, x, -1) == ERR_ARG
        assert raw(K, obs, 2, None, 16) == ERR_ARG                                   # no rows
        assert raw(K, None, 2, x, 16) == ERR_ARG                                     # no obs_dims
        assert raw(K, obs, 0, x, 16) == ERR_ARG
        assert raw(K, np.arange(5, dtype=np.int32), 5, np.ones((16, 5), np.float32), 16) == ERR_ARG   # n_obs > D
        for bad in ([2, 0], [1, 1], [0, 4], [-1, 2]):
            assert raw(K, np.array(bad, np.int32), 2, x, 16) == ERR_ARG, bad
        assert raw(K, obs, 2, x, 16, s=None, m=None) == ERR_ARG                      # neither output
        y = x.copy()
        y[9, 1] = np.inf
        assert raw(K, obs, 2, y, 16) == ERR_ARG                                      # not finite
        y[9, 1] = np.nan
        assert raw(K, obs, 2, y, 16, s=None, m=mb) == ERR_ARG
        sh[:] = 0
        assert raw(K, obs, 2, None, 0) == 0                                          # n = 0: zero statistics and the centre
        assert np.all(st == 0.0) and np.array_equal(sh, standardise(ev)[0])
        assert raw(K + 1, obs, 2, x, 16) == ERR_STATE                                # not the current K
        eng.estep(K)
        eng.mstep(K)
        assert raw(K, obs, 2, x, 16) == ERR_STATE                                    # between gmm_mstep and gmm_constants
        eng.constants(K)
        assert raw(K, obs, 2, x, 16) == 0
        bad = good.copy()
        bad.Rinv[2] = np.diag([1.0, -1.0, 1.0, 1.0]).astype(np.float32)             # P_MM indefinite for M = {1, 3}
        eng.set_clusters(K, bad)
        with pytest.raises(pkg.GmmError) as e:
            eng.condition_stats(K, obs, x)
        assert e.value.code == ERR_STATE and "cluster 2" in str(e.value) and "gmm_condition_stats" in str(e.value), str(e.value)
        eng.condition_stats(K, [1, 2], x)                                            # M = {0, 3}: positive definite
        eng.set_clusters(K, good)
        eng.condition_stats(K, obs, x)
        prof = eng.condition_stats_profile(reset=True)
        assert prof["kernel_ms"] > 0 and prof["wall_ms"] >= prof["kernel_ms"]
        assert eng.condition_stats_profile() == dict(kernel_ms=0.0, wall_ms=0.0, mstep_tensor_chunks=0, mstep_simt_chunks=0)
