"""gmm_modes / gmm_mode_labels (Engine.modes, Engine.mode_labels) on the GPU (run with -m gpu on an H100), against the
float64 restatement tests/_modes_ref.py and analytic cases."""
import ctypes as C
import threading

import numpy as np
import pytest

import _modes_ref as mr
from conftest import gpu_count
from test_modes_host import triangle_sigma

pytestmark = pytest.mark.gpu
ARG, STATE = 1, 6
MERGE = 1e-2
ROUND = 16                # iterations per launch of mode_iter_kernel (kModeRound)


@pytest.fixture(scope="module")
def loaded(pkg):
    pkg.load_library()
    return pkg


def _mixture(pkg, D, K, seed, spread=6.0, aniso=0.3):
    """K components with random SPD covariances around centres `spread` apart on average, raw offsets of 1e3."""
    rng = np.random.default_rng(seed)
    cl = pkg.Clusters(K, D)
    means = rng.normal(size=(K, D)) * spread + 1e3
    Ls = rng.normal(size=(K, D, D)) * aniso / np.sqrt(D) + np.eye(D)
    R = Ls @ np.swapaxes(Ls, 1, 2)
    Rinv = np.linalg.inv(R)
    pi = rng.dirichlet(np.full(K, 3.0))
    cl.means[:K] = means
    cl.R[:K] = R
    cl.Rinv[:K] = Rinv.astype(np.float32)
    cl.pi[:K] = pi
    cl.N[:K] = pi * 1000
    cl.constant[:K] = -0.5 * D * np.log(2 * np.pi) - 0.5 * np.linalg.slogdet(R)[1]
    cl.avgvar[:K] = 0.0
    return cl


def _ref(cl, K):
    return mr.params(cl.means[:K], cl.Rinv[:K], cl.R[:K], cl.constant[:K], cl.pi[:K])


def _engine(pkg, D, Kmax, n=256, seed=0, events=None):
    ev = events if events is not None else np.random.default_rng(seed).normal(size=(n, D)).astype(np.float32) + 1e3
    return pkg.Engine(np.ascontiguousarray(ev, np.float32), Kmax, device=0)


@pytest.mark.parametrize("D", [8, 16, 24, 5, 32])
@pytest.mark.parametrize("K", [1, 2, 7, 64, 65, 130, 512])
def test_modes_against_the_restatement(loaded, D, K):
    cl = _mixture(loaded, D, K, seed=D * 1000 + K)
    p = _ref(cl, K)
    ends, _, st = mr.climb(p, p["mu"])
    rmodes, rcm = mr.dedup(p, ends, st, MERGE)
    if len(rmodes) > 1:
        dm = np.array([[mr.rho(p, a, b) for b in rmodes] for a in rmodes]) + np.eye(len(rmodes)) * 1e9
        if dm.min() < 10 * MERGE:
            pytest.skip("reference modes closer than 10 merge_tol")
    with _engine(loaded, D, K) as eng:
        eng.set_clusters(K, cl)
        got = eng.modes(K, max_iter=500)
        again = eng.modes(K, max_iter=500)
    assert len(got["modes"]) == len(rmodes)
    np.testing.assert_array_equal(got["comp_mode"][p["live"]], rcm)
    assert np.max(mr.rho(p, got["modes"] - p["c"], rmodes)) <= MERGE / 4
    np.testing.assert_array_equal(got["is_max"], mr.is_max(p, rmodes))
    for k in ("modes", "comp_mode", "iters"):
        np.testing.assert_array_equal(got[k], again[k])


@pytest.mark.parametrize("D, K", [(8, 7), (16, 64), (24, 130), (5, 12)])
def test_labels_against_the_restatement(loaded, D, K):
    cl = _mixture(loaded, D, K, seed=7 + D + K, spread=2.5)
    p = _ref(cl, K)
    with _engine(loaded, D, K) as eng:
        eng.set_clusters(K, cl)
        ev, _ = eng.sample(K, 3000, seed=11)
        md = eng.modes(K)
        got = eng.mode_labels(K, md["modes"], ev, endpoints=True, logp=True, iters=True)
    modes = md["modes"] - p["c"]
    x0 = ev.astype(np.float64) - p["c"]
    ends, _, st = mr.climb(p, x0)
    ref = mr.labels(p, ends, st, modes, MERGE)
    sig = 1.0 / p["inv_sigma"]
    decided = np.ones(len(ev), bool)
    rng = np.random.default_rng(5)
    for _ in range(4):
        e2, _, s2 = mr.climb(p, x0 + rng.normal(size=x0.shape) * 1e-4 * sig)
        decided &= mr.labels(p, e2, s2, modes, MERGE) == ref
    assert np.mean(~decided) <= 1e-3
    np.testing.assert_array_equal(got["labels"][decided], ref[decided])
    lp0 = mr.logp(p, x0)
    assert np.all(got["logp"] >= lp0 - 1e-4 * np.maximum(1, np.abs(lp0)))
    assert got["unconverged"] == 0


def test_invariance_bit_for_bit(loaded):
    D, K = 24, 64
    cl = _mixture(loaded, D, K, seed=3, spread=2.5)
    with _engine(loaded, D, K, n=4) as e0:
        e0.set_clusters(K, cl)
        ev, _ = e0.sample(K, 20000, seed=2)
    with _engine(loaded, D, K, events=ev) as eng:
        eng.set_clusters(K, cl)
        md = eng.modes(K)["modes"]
        a = eng.mode_labels(K, md, ev, endpoints=True, logp=True, iters=True)
        b = eng.mode_labels(K, md, None, endpoints=True, logp=True, iters=True)
        c = eng.mode_labels(K, md, ev, endpoints=True, logp=True, iters=True)
        eng.set_option("score_chunk", 3001)
        d = eng.mode_labels(K, md, ev, endpoints=True, logp=True, iters=True)
        h1 = eng.mode_labels(K, md, ev[:7777], endpoints=True, logp=True, iters=True)
        h2 = eng.mode_labels(K, md, ev[7777:], endpoints=True, logp=True, iters=True)
    for k in ("labels", "endpoints", "logp", "iters"):
        for o in (b, c, d):
            np.testing.assert_array_equal(a[k], o[k], err_msg=k)
        np.testing.assert_array_equal(a[k], np.concatenate([h1[k], h2[k]]), err_msg=k)


@pytest.mark.parametrize("sep, want", [(1.9, 1), (2.1, 2)])
def test_two_components_at_two_sigma(loaded, sep, want):
    D, K = 2, 2
    cl = _mixture(loaded, D, K, 0)
    cl.means[:2] = [[1e3, 1e3], [1e3 + sep, 1e3]]
    cl.R[:2] = np.eye(2); cl.Rinv[:2] = np.eye(2)
    cl.pi[:2] = 0.5
    cl.constant[:2] = -np.log(2 * np.pi)
    with _engine(loaded, D, K) as eng:
        eng.set_clusters(K, cl)
        md = eng.modes(K, max_iter=2000)
        lab = eng.mode_labels(K, md["modes"], max_iter=2000, iters=True)
    assert len(md["modes"]) == want and np.all(md["is_max"])
    assert lab["unmatched"] == 0 and lab["unconverged"] == 0
    if want == 1:
        # the single mode at 1.9 sigma is flat: events climb for many rounds, and their counts run on across round ends
        it = lab["iters"]
        assert it.max() > 4 * ROUND
        assert np.count_nonzero((it > ROUND) & (it % ROUND != 0)) > np.count_nonzero((it > ROUND) & (it % ROUND == 0))


def _far_narrow_pair(pkg, D=8, L=600.0, s=1e-2, corr=0.999):
    """Three unit components near the origin and, about 600 sigma away in every coordinate, two equal narrow components
    with correlation 0.999 within each pair of dimensions, 0.5 s apart along their long axis: one mode at their midpoint.
    Its position needs g from each dx_k: A x and b are both about 1e9 here, and their difference is what moves x."""
    K = 5
    cl = pkg.Clusters(K, D)
    blk = np.array([[1.0, corr], [corr, 1.0]])
    Cn = np.kron(np.eye(D // 2), blk) * s * s
    u = np.ones(D) / np.sqrt(D)
    means = np.array([np.zeros(D), np.full(D, 3.0), np.full(D, -3.0), np.full(D, L), np.full(D, L) + 0.5 * s * u])
    Rs = [np.eye(D)] * 3 + [Cn, Cn]
    cl.means[:K] = means
    for k in range(K):
        cl.R[k] = Rs[k]
        cl.Rinv[k] = np.linalg.inv(Rs[k]).astype(np.float32)
        cl.constant[k] = -0.5 * D * np.log(2 * np.pi) - 0.5 * np.linalg.slogdet(Rs[k])[1]
    cl.pi[:K] = [0.3, 0.3, 0.3, 0.05, 0.05]
    cl.N[:K] = cl.pi[:K] * 1000
    cl.avgvar[:K] = 0.0
    return cl


def test_modes_far_from_the_centre_keep_their_position(loaded):
    """The step form keeps a mode 570 sigma from the centre to about one float ulp there (6e-5 sigma); forming g as A x - b
    would lose it to the cancellation of two terms of about 1e9."""
    D, K = 8, 5
    cl = _far_narrow_pair(loaded, D)
    p = _ref(cl, K)
    p["mu"] = p["mu"].astype(np.float32).astype(np.float64)      # the device's float records
    ends, _, st = mr.climb(p, p["mu"])
    rmodes, rcm = mr.dedup(p, ends, st, MERGE)
    assert rcm[3] == rcm[4] and np.min(np.abs(rmodes[rcm[3]])) > 500
    with _engine(loaded, D, K) as eng:
        eng.set_clusters(K, cl)
        got = eng.modes(K)
    np.testing.assert_array_equal(got["comp_mode"], rcm)
    assert mr.rho(p, got["modes"][rcm[3]] - p["c"], rmodes[rcm[3]]) <= 1e-4


def test_triangle_centroid_basin(loaded):
    s = triangle_sigma()
    D, K = 2, 3
    cl = _mixture(loaded, D, K, 0)
    verts = np.array([[np.cos(t), np.sin(t)] for t in (np.pi / 2, np.pi / 2 + 2 * np.pi / 3, np.pi / 2 + 4 * np.pi / 3)])
    cl.means[:3] = verts
    cl.R[:3] = np.eye(2) * s * s; cl.Rinv[:3] = np.eye(2) / (s * s)
    cl.pi[:3] = 1 / 3
    cl.constant[:3] = -np.log(2 * np.pi * s * s)
    p = _ref(cl, K)
    ev = (np.random.default_rng(1).normal(size=(200, 2)) * 0.02).astype(np.float32)
    with _engine(loaded, D, K) as eng:
        eng.set_clusters(K, cl)
        md = eng.modes(K)
        got = eng.mode_labels(K, md["modes"], ev, endpoints=True, max_iter=5000)
    assert len(md["modes"]) == 3
    cen = -p["c"]
    assert np.all(got["labels"] == -2)
    assert np.max(mr.rho(p, got["endpoints"].astype(np.float64) - p["c"], cen[None])) < 2e-3


def test_one_component_and_zero_weights(loaded):
    D, K = 16, 9
    cl = _mixture(loaded, D, K, 4, spread=8.0)
    with _engine(loaded, D, K, n=3000, seed=1) as eng:
        eng.set_clusters(1, cl)
        one = eng.modes(1)
        assert len(one["modes"]) == 1 and one["iters"][0] == 1          # a start at the mean stops at once
        assert np.all(eng.mode_labels(1, one["modes"])["labels"] == 0)
        # pi = 0 components: never a start, no change to any other output
        live = [0, 2, 3, 5, 8]
        c2 = _mixture(loaded, D, len(live), 4, spread=8.0)
        for i, k in enumerate(live):
            for f in ("means", "R", "Rinv", "pi", "constant", "N"):
                getattr(c2, f)[i] = getattr(cl, f)[k]
        for f in ("pi", "N"):
            getattr(cl, f)[[1, 4, 6, 7]] = 0
        eng.set_clusters(len(live), c2)
        a = eng.modes(len(live))
        la = eng.mode_labels(len(live), a["modes"], endpoints=True, logp=True, iters=True)
        eng.set_clusters(K, cl)
        b = eng.modes(K)
        lb = eng.mode_labels(K, b["modes"], endpoints=True, logp=True, iters=True)
    np.testing.assert_array_equal(a["modes"], b["modes"])
    np.testing.assert_array_equal(b["comp_mode"][[1, 4, 6, 7]], -1)
    np.testing.assert_array_equal(b["comp_mode"][live], a["comp_mode"])
    for k in ("labels", "endpoints", "logp", "iters"):
        np.testing.assert_array_equal(la[k], lb[k])


def test_scale_well_separated(loaded):
    D, K, n = 24, 64, 1_000_000
    cl = _mixture(loaded, D, K, 9, spread=12.0, aniso=0.2)
    with _engine(loaded, D, K, n=4) as e0:
        e0.set_clusters(K, cl)
        ev, _ = e0.sample(K, n, seed=3)
    with _engine(loaded, D, K, events=ev) as eng:
        eng.set_clusters(K, cl)
        md = eng.modes(K)
        got = eng.mode_labels(K, md["modes"], max_iter=500)
        sl, _, _, _ = eng.score(K, ev, max_resp=False, logp=False)
        prof = eng.modes_profile()
    assert got["unconverged"] == 0
    assert np.mean(got["labels"] == md["comp_mode"][sl]) >= 0.999
    assert prof["event_iterations"] > n


def test_state_and_errors(loaded, pkg):
    D, K = 8, 5
    cl = _mixture(loaded, D, K, 1)
    with _engine(loaded, D, 8, n=2000, seed=3) as eng:
        eng.set_clusters(K, cl)
        eng.estep(K)
        before = eng.get_clusters(K, with_memberships=True)
        prof = eng.profile()
        sprof = eng.score_profile()
        md = eng.modes(K)
        eng.mode_labels(K, md["modes"])
        after = eng.get_clusters(K, with_memberships=True)
        np.testing.assert_array_equal(before.memberships, after.memberships)
        assert eng.profile() == prof and eng.score_profile() == sprof

        def code(f):
            with pytest.raises(pkg.GmmError) as e:
                f()
            return e.value.code
        assert code(lambda: eng.modes(0)) == ARG
        assert code(lambda: eng.modes(9)) == ARG
        assert code(lambda: eng.modes(4)) == STATE
        assert code(lambda: eng.modes(K, max_iter=0)) == ARG
        assert code(lambda: eng.modes(K, tol=float("nan"))) == ARG
        assert code(lambda: eng.modes(K, merge_tol=float("inf"))) == ARG
        assert code(lambda: eng.modes(K, tol=1e-3, merge_tol=5e-3)) == ARG
        assert code(lambda: eng.mode_labels(K, np.zeros((0, D)))) == ARG
        assert code(lambda: eng.mode_labels(K, md["modes"], max_iter=0)) == ARG
        bad = eng.get_clusters(K)
        bad.Rinv[2] = -np.eye(D)
        eng.set_clusters(K, bad)
        with pytest.raises(pkg.GmmError) as e:
            eng.modes(K)
        assert e.value.code == STATE and "component 2" in str(e.value)
        # n < 0, and the shard (events NULL) with n != n_local, through the C entry point
        lib, md64 = eng.lib, np.ascontiguousarray(md["modes"], np.float64)
        lab = np.zeros(eng.n + 1, np.int32)
        um, uc = C.c_longlong(), C.c_longlong()

        def raw(ev, n):
            return lib.gmm_mode_labels(eng.h, K, ev, n, md64.ctypes.data, len(md64), 100, -1.0, -1.0, lab.ctypes.data, None, None,
                                       None, C.byref(um), C.byref(uc))
        one_ev = np.zeros((1, D), np.float32)
        assert raw(one_ev.ctypes.data, -1) == ARG
        assert raw(None, eng.n + 1) == ARG
        assert raw(None, eng.n - 1) == ARG
        eng.set_clusters(K, cl)
        eng.estep(K)
        eng.mstep(K)
        assert code(lambda: eng.modes(K)) == STATE
        assert code(lambda: eng.mode_labels(K, md["modes"])) == STATE
        assert code(lambda: eng.mode_labels(K, md["modes"], one_ev)) == STATE


def _profiles(eng):
    return {f: getattr(eng, f)() for f in ("profile", "score_profile", "score_stats_profile", "sample_profile", "condition_profile",
                                           "condition_stats_profile", "vb_profile", "combine_profile", "multisample_profile",
                                           "fit_profile")}


def test_em_state_unchanged(loaded):
    """Memberships, every other profile, and the statistics and log-likelihood of the next EM iterations are those of a
    twin context that never called gmm_modes / gmm_mode_labels."""
    D, K = 16, 7
    cl = _mixture(loaded, D, K, 2, spread=2.5)
    ev = np.random.default_rng(8).normal(size=(5000, D)).astype(np.float32) * 4 + 1e3
    out = []
    for call in (False, True):
        with _engine(loaded, D, K, events=ev) as eng:
            eng.set_clusters(K, cl)
            eng.estep(K)
            m0 = eng.get_clusters(K, with_memberships=True).memberships.copy()
            pr = _profiles(eng)
            if call:
                md = eng.modes(K)
                eng.mode_labels(K, md["modes"])
                eng.mode_labels(K, md["modes"], ev[:100])
                assert _profiles(eng) == pr
                np.testing.assert_array_equal(eng.get_clusters(K, with_memberships=True).memberships, m0)
            ll = eng.em_iterations(K, 2)
            cc = eng.get_clusters(K, with_memberships=True)
            out.append((ll, cc.means.copy(), cc.R.copy(), cc.pi.copy(), cc.memberships.copy()))
    assert out[0][0] == out[1][0]
    for a, b in zip(out[0][1:], out[1][1:]):
        np.testing.assert_array_equal(a, b)


def test_two_gpus_equal_one(loaded):
    if gpu_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    pkg = loaded
    D, K = 24, 64
    cl = _mixture(pkg, D, K, 13, spread=2.5)
    with _engine(pkg, D, K, n=4) as e0:
        e0.set_clusters(K, cl)
        ev, _ = e0.sample(K, 30001, seed=4)
    N = len(ev)
    with _engine(pkg, D, K, events=ev) as eng:
        eng.set_clusters(K, cl)
        one = eng.modes(K)
        one_lab = eng.mode_labels(K, one["modes"], None, endpoints=True, logp=True, iters=True)
    uid = pkg.nccl_unique_id()
    res = [None, None]

    def worker(g):
        try:
            b, n = pkg.shard_range(N, 2, g)
            with pkg.Engine(np.ascontiguousarray(ev[b:b + n]), K, device=g, n_global=N, offset=b) as e:
                e.comm_init(2, g, uid)
                e.set_clusters(K, cl)
                md = e.modes(K)
                res[g] = (md, e.mode_labels(K, md["modes"], None, endpoints=True, logp=True, iters=True))
        except Exception as ex:  # noqa: BLE001
            res[g] = ex

    ts = [threading.Thread(target=worker, args=(g,)) for g in range(2)]
    for t in ts:
        t.start()
    for t in ts:
        t.join(timeout=600)
    for r in res:
        assert not isinstance(r, Exception), r
        for f in ("modes", "logp", "is_max", "comp_mode", "iters"):
            np.testing.assert_array_equal(r[0][f], one[f], err_msg=f)
    for f in ("labels", "endpoints", "logp", "iters"):
        np.testing.assert_array_equal(np.concatenate([res[0][1][f], res[1][1][f]]), one_lab[f], err_msg=f)
