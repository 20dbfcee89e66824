"""gmm_combine / gmm_combine_labels (Engine.combine, Engine.combine_labels) on the GPU (run with -m gpu on an H100), against
the restatement tests/_combine_ref.py evaluated on the engine's own memberships."""
import threading

import numpy as np
import pytest

import _combine_ref as cr
from conftest import gpu_count

pytestmark = pytest.mark.gpu

GAIN_RTOL = 2e-6          # a gain: the float phi's per-term bound plus the double sums
COL_RTOL = 1e-6           # entropy_out[K-1] and the masses
ARG, STATE = 1, 6


@pytest.fixture(scope="module")
def loaded(pkg):
    pkg.load_library()
    return pkg


def _fixture(pkg, D, K, n, seed):
    """ceil(K/2) unit-variance blobs of unequal sizes on a chain 6 sigma apart, each carried by two components displaced
    +-0.5 sigma (the last by one when K is odd); events and the parameter set for gmm_set_clusters."""
    rng = np.random.default_rng(seed)
    nb = (K + 1) // 2
    frac = rng.dirichlet(np.full(nb, 4.0)) if nb > 1 else np.ones(1)
    counts = np.maximum((frac * n).astype(int), 20)
    counts[-1] = max(20, n - counts[:-1].sum())
    centres = np.zeros((nb, D))
    centres[:, 0] = 6.0 * np.arange(nb)
    centres[:, 2:] = rng.normal(0, 0.3, (nb, D - 2))
    ev = np.concatenate([rng.standard_normal((c, D)) + centres[j] for j, c in enumerate(counts)]).astype(np.float32)
    ev = np.ascontiguousarray(ev[rng.permutation(len(ev))])
    cl = pkg.Clusters(K, D)
    k = 0
    for j in range(nb):
        shifts = (-0.5, 0.5) if 2 * j + 1 < K else (0.0,)
        for s in shifts:
            cl.means[k] = centres[j]
            cl.means[k, 1] += s
            cl.pi[k] = frac[j] / len(shifts)
            k += 1
    cl.pi /= cl.pi.sum()
    cl.N[:] = cl.pi * len(ev)
    cl.R[:] = np.eye(D, dtype=np.float32)
    cl.Rinv[:] = np.eye(D, dtype=np.float32)
    cl.constant[:] = -0.5 * D * np.log(2 * np.pi)
    cl.avgvar[:] = 0.01
    return ev, cl


def _memberships(eng, K):
    return np.ascontiguousarray(eng.get_clusters(K, with_memberships=True).memberships[:K])


def _gaps_ok(ref, bar=GAIN_RTOL):
    g = ref["gap"]
    return bool(np.all((g >= 10 * bar) | np.isnan(g)))


def _check_against(got, ref, K, n, nsteps=None):
    s = K - 1 if nsteps is None else nsteps
    np.testing.assert_array_equal(got["merges"][:s], ref["merges"][:s])
    zero = ref["gain"][:s] == 0
    assert np.all(got["gain"][:s][zero] == 0)
    np.testing.assert_allclose(got["gain"][:s], ref["gain"][:s], rtol=GAIN_RTOL, atol=0)
    np.testing.assert_allclose(got["mass"][:s], ref["mass"][:s], rtol=COL_RTOL, atol=0)
    np.testing.assert_allclose(got["entropy"][K - 1], ref["entropy"][K - 1], rtol=COL_RTOL, atol=1e-12 * n)
    if nsteps is None:
        # sum_k tau_k = 1 within K float roundings per event, so the one-cluster entropy is about 0
        bar = 2.4e-7 * K * n + GAIN_RTOL * float(np.sum(ref["gain"])) + COL_RTOL * abs(ref["entropy"][K - 1])
        assert abs(got["entropy"][0]) <= bar, (got["entropy"][0], bar)
        np.testing.assert_allclose(np.diff(got["entropy"]), got["gain"][::-1], rtol=1e-12, atol=1e-9 * abs(got["entropy"]).max())


GRID = [(D, K) for D in (8, 16, 24, 5, 32) for K in (1, 2, 7, 64, 65, 130)]


@pytest.mark.parametrize("D,K", GRID)
def test_shape_grid(loaded, D, K):
    """Merges, gains, entropy and masses against the restatement on blobs carried by pairs of components; labels at every
    level bit for bit; the identity grouping against gmm_score's labels at K <= 64."""
    pkg = loaded
    n = 12_000
    for attempt in range(4):
        ev, cl = _fixture(pkg, D, K, n, 1000 * attempt + 10 * D + K)
        with pkg.Engine(ev, K) as eng:
            eng.set_clusters(K, cl)
            eng.estep(K)
            tau = _memberships(eng, K)
            ref = cr.combine(tau)
            if not _gaps_ok(ref):
                continue
            got = eng.combine(K)
            _check_against(got, ref, K, len(ev))
            for L in range(1, K + 1):
                grp = pkg.host_combine_groups(got["merges"], K, L)
                lab, mx = eng.combine_labels(K, grp)
                rl, rm = cr.labels(tau, grp, L)
                np.testing.assert_array_equal(lab, rl, err_msg=f"L={L}")
                np.testing.assert_array_equal(mx.view(np.int32), rm.view(np.int32), err_msg=f"L={L}")
            if K <= 64:
                lab, _ = eng.combine_labels(K, np.arange(K))
                slab, _, _, _ = eng.score(K, ev, max_resp=False, logp=False)
                np.testing.assert_array_equal(lab, slab)
        return
    pytest.fail("no fixture seed gave every step a top-two gap of 10x the gain bar")


@pytest.mark.parametrize("D,K", [(16, 9), (24, 20), (5, 70)])
def test_integer_weights_equal_replicated_rows(loaded, D, K):
    """Integer weights (zeros included) against the rows replicated that many times.  Both engines run the SIMT E-step,
    whose memberships depend on the event and the parameters alone, so every phi term is the same float and only the
    order of the double sums differs."""
    pkg = loaded
    ev, cl = _fixture(pkg, D, K, 6000, 77 + K)
    w = np.random.default_rng(K).integers(0, 4, size=len(ev)).astype(np.float32)
    rep = np.ascontiguousarray(np.repeat(ev, w.astype(int), axis=0))
    with pkg.Engine(ev, K) as eng:
        eng.set_option("path", pkg.PATH_SIMT)
        eng.set_weights(w)
        eng.set_clusters(K, cl)
        eng.estep(K)
        tau = _memberships(eng, K)
        got = eng.combine(K)
    with pkg.Engine(rep, K) as eng:
        eng.set_option("path", pkg.PATH_SIMT)
        eng.set_clusters(K, cl)
        eng.estep(K)
        one = eng.combine(K)
    ref = cr.combine(tau, w)
    steps = K - 1 if _gaps_ok(ref) else int(np.argmax(ref["gap"] < 10 * GAIN_RTOL))
    _check_against(got, ref, K, len(rep), None if steps == K - 1 else steps)
    np.testing.assert_array_equal(got["merges"][:steps], one["merges"][:steps])
    np.testing.assert_allclose(got["gain"][:steps], one["gain"][:steps], rtol=1e-9)
    np.testing.assert_allclose(got["mass"][:steps], one["mass"][:steps], rtol=1e-9)
    np.testing.assert_allclose(got["entropy"][K - 1], one["entropy"][K - 1], rtol=1e-9)


def test_state_unchanged_and_repeatable(loaded):
    pkg = loaded
    D, K = 16, 40
    ev, cl = _fixture(pkg, D, K, 30_000, 5)
    with pkg.Engine(ev, K) as eng:
        eng.set_clusters(K, cl)
        eng.estep(K)
        eng.em(K, 3, 3)
        before = eng.get_clusters(K, with_memberships=True)
        prof = eng.profile()
        a = eng.combine(K)
        grp = pkg.host_combine_groups(a["merges"], K, 5)
        la = eng.combine_labels(K, grp)
        b = eng.combine(K)
        lb = eng.combine_labels(K, grp)
        for f in ("merges", "gain", "entropy", "mass"):
            np.testing.assert_array_equal(a[f], b[f], err_msg=f)
        np.testing.assert_array_equal(la[0], lb[0])
        np.testing.assert_array_equal(la[1].view(np.int32), lb[1].view(np.int32))
        after = eng.get_clusters(K, with_memberships=True)
        for f in pkg.Clusters.FIELDS:
            np.testing.assert_array_equal(getattr(after, f)[:K], getattr(before, f)[:K], err_msg=f)
        np.testing.assert_array_equal(after.memberships[:K], before.memberships[:K])
        assert eng.profile() == prof
        p = eng.combine_profile(reset=True)
        assert p["kernel_ms"] > 0 and p["wall_ms"] >= p["kernel_ms"] * 0.5 and p["labels_wall_ms"] > 0
        assert eng.combine_profile() == dict(kernel_ms=0.0, wall_ms=0.0, labels_wall_ms=0.0)


def test_errors(loaded):
    pkg = loaded
    D, K = 8, 6
    ev, cl = _fixture(pkg, D, K, 4000, 9)
    L = pkg.load_library()
    m = np.zeros((K - 1, 2), np.int32)
    grp = np.zeros(K, np.int32)
    lab = np.zeros(len(ev), np.int32)
    with pkg.Engine(ev, 2 * K) as eng:
        call = lambda k: L.gmm_combine(eng.h, k, m.ctypes.data, None, None, None)  # noqa: E731
        labels = lambda k, g, G: L.gmm_combine_labels(eng.h, k, g.ctypes.data if g is not None else None, G, lab.ctypes.data, None)  # noqa: E731
        eng.set_clusters(K, cl)
        assert call(K) == STATE                                  # no E-step yet
        assert labels(K, grp, 1) == STATE
        eng.estep(K)
        assert call(K) == 0
        assert call(0) == ARG and call(2 * K + 1) == ARG
        assert L.gmm_combine(eng.h, K, None, None, None, None) == ARG
        assert call(K - 1) == STATE                              # K != cur_K
        assert labels(K, grp, 0) == ARG and labels(K, grp, K + 1) == ARG and labels(K, None, 1) == ARG
        assert labels(K, np.full(K, 2, np.int32), 2) == ARG and labels(K, np.full(K, -1, np.int32), 1) == ARG
        assert labels(K, grp, 1) == 0
        eng.mstep(K)                                             # between gmm_mstep and gmm_constants
        assert call(K) == STATE
        eng.constants(K)
        eng.estep(K)
        assert call(K) == 0
        eng.set_weights(np.ones(len(ev), np.float32))            # weights mark the memberships stale
        assert call(K) == STATE
        eng.estep(K)
        assert call(K) == 0
        eng.set_clusters(K, cl)
        assert call(K) == STATE
        # K = 1 needs no merges_out and writes entropy_out[0]
        one = pkg.Clusters(1, D)
        one.means[0] = ev.mean(axis=0)
        one.R[0] = one.Rinv[0] = np.eye(D, dtype=np.float32)
        one.pi[0], one.N[0], one.constant[0], one.avgvar[0] = 1.0, len(ev), -0.5 * D * np.log(2 * np.pi), 0.01
        eng.set_clusters(1, one)
        eng.estep(1)
        ent = np.array([np.nan])
        assert L.gmm_combine(eng.h, 1, None, None, ent.ctypes.data, None) == 0
        assert abs(ent[0]) <= 1e-6 * len(ev)
    # after gmm_fit, ideal_K needs gmm_set_clusters + gmm_estep first
    with pkg.Engine(ev, 8) as eng:
        eng.seed(8)
        ideal, _, saved = eng.fit(8, 2, 3, 3)
        if ideal != 2:
            assert L.gmm_combine(eng.h, ideal, m.ctypes.data, None, None, None) == STATE
        eng.set_clusters(ideal, saved)
        eng.estep(ideal)
        assert eng.combine(ideal)["merges"].shape == (ideal - 1, 2)
    # memberships that are not finite (an event with a NaN coordinate on the SIMT E-step)
    bad = ev.copy()
    bad[17, 3] = np.nan
    with pkg.Engine(bad, K) as eng:
        eng.set_option("path", pkg.PATH_SIMT)
        eng.set_clusters(K, cl)
        eng.estep(K)
        if np.isnan(_memberships(eng, K)).any():
            with pytest.raises(pkg.GmmError) as ex:
                eng.combine(K)
            assert ex.value.code == STATE and "component 0" in str(ex.value)


def test_c2_after_em(loaded):
    """c2's size (1M events, D = 16, K = 32) after 20 EM iterations, against the restatement chunked in numpy, step by
    step while the reference's top-two gap clears the bar."""
    pkg = loaded
    N, D, K = 1_000_000, 16, 32
    ev = pkg.synth.make_blobs(N, D, 16, seed=21)
    with pkg.Engine(ev, K) as eng:
        eng.seed(K)
        eng.em(K, 20, 20)
        tau = _memberships(eng, K)
        got = eng.combine(K)
        grp = pkg.host_combine_groups(got["merges"], K, 16)
        lab, mx = eng.combine_labels(K, grp)
    ref = cr.combine(tau)
    ok = ref["gap"] >= 10 * GAIN_RTOL
    steps = K - 1 if ok.all() else int(np.argmin(ok))
    assert steps >= K // 2, ref["gap"]
    _check_against(got, ref, K, N, None if steps == K - 1 else steps)
    rl, rm = cr.labels(tau, grp, 16)
    np.testing.assert_array_equal(lab, rl)
    np.testing.assert_array_equal(mx.view(np.int32), rm.view(np.int32))


def test_two_gpus_equal_one(loaded):
    if gpu_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    pkg = loaded
    D, K = 16, 24
    ev, cl = _fixture(pkg, D, K, 40_001, 3)
    N = len(ev)
    with pkg.Engine(ev, K) as eng:
        eng.set_clusters(K, cl)
        eng.estep(K)
        one = eng.combine(K)
    uid = pkg.nccl_unique_id()
    res = [None, None]

    def worker(g):
        try:
            b, n = pkg.shard_range(N, 2, g)
            with pkg.Engine(np.ascontiguousarray(ev[b:b + n]), K, device=g, n_global=N, offset=b) as e:
                e.comm_init(2, g, uid)
                e.set_clusters(K, cl)
                e.estep(K)
                res[g] = e.combine(K)
        except Exception as ex:  # noqa: BLE001
            res[g] = ex

    ts = [threading.Thread(target=worker, args=(g,)) for g in range(2)]
    for t in ts:
        t.start()
    for t in ts:
        t.join(timeout=600)
    for r in res:
        assert not isinstance(r, Exception), r
        np.testing.assert_array_equal(r["merges"], one["merges"])
        np.testing.assert_allclose(r["gain"], one["gain"], rtol=2 * GAIN_RTOL)
    for f in ("merges", "gain", "entropy", "mass"):
        np.testing.assert_array_equal(res[0][f], res[1][f], err_msg=f)
