"""gmm_seed_kmeans: k-means++ and Lloyd initialisation of a mixture on the GPU (run with -m gpu on an H100).

The k-means++ part is reproduced bit for bit by the numpy reference below (splitmix64 draws, sequential float64 distances,
block sums of 1024 events added in index order, np.cumsum + searchsorted(side="right"), greedy choice).  The one-hot
M-step is held against the exact float64 M-step of tests/test_mstep_error_model.py; Lloyd against a float64 numpy Lloyd
(sklearn's algorithm="lloyd" with tol=0) and against sklearn itself when it is installed.  Every case asserts which
M-step kernel ran through gmm_get_profile's launch counters, which count the call's M-steps (one per Lloyd assignment
whose labels changed, plus the first)."""
import threading

import numpy as np
import pytest

from conftest import assert_params_close, gpu_count
from test_mstep_error_model import MSTEP_TOL, exact_mstep_stats, param_errors, standardise

pytestmark = pytest.mark.gpu

ERR_ARG, ERR_STATE = 1, 6
TENSOR_M_D = (4, 8, 12, 16, 20, 24)
BLOCK = 1024                 # kSeedBlockEvents
M64 = (1 << 64) - 1
AMBIG = 4e-6                 # two nearest centres closer than this (relative) could swap under FP32 rounding


# ---- numpy reference of the k-means++ semantics (include/gmm.h) -----------------------------------------------------------
def splitmix(seed):
    s = seed & M64
    while True:
        s = (s + 0x9E3779B97F4A7C15) & M64
        z = s
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
        z ^= z >> 31
        yield float(z >> 11) * 2.0 ** -53


def dist(x64, c):
    """sum_d (x_d - c_d)^2 in dimension order, each operation rounded once (what __dsub_rn / __dmul_rn / __dadd_rn do)."""
    s = np.zeros(len(x64))
    for d in range(x64.shape[1]):
        t = x64[:, d] - np.float64(c[d])
        s = s + t * t
    return s


def kmeanspp_ref(x, K, seed):
    """Indices of the chosen centres, and whether any greedy choice was a near-tie between distinct candidates (the
    device adds the potentials in another order than np.sum)."""
    n = len(x)
    x64 = x.astype(np.float64)
    rng = splitmix(seed)
    L = 2 + int(np.floor(np.log(K)))
    idx = [min(int(next(rng) * n), n - 1)]
    ambiguous = False
    if K == 1:
        return idx, ambiguous
    d2 = dist(x64, x[idx[0]])
    nb = -(-n // BLOCK)
    for _ in range(1, K):
        pad = np.zeros(nb * BLOCK)
        pad[:n] = d2
        P = np.cumsum(np.cumsum(pad.reshape(nb, BLOCK), axis=1)[:, -1])
        T = P[-1]
        if not T > 0:
            idx += [idx[0]] * (K - len(idx))
            break
        cands = []
        for _ in range(L):
            t = next(rng) * T
            b = int(np.searchsorted(P, t, side="right"))
            if b == nb:
                cands.append(int(np.nonzero(d2 > 0)[0][-1]))
                continue
            blk = d2[b * BLOCK:(b + 1) * BLOCK]
            run = np.cumsum(np.concatenate([[P[b - 1] if b else 0.0], blk]))[1:]
            i = int(np.searchsorted(run, t, side="right"))
            cands.append(b * BLOCK + (i if i < len(blk) else int(np.nonzero(blk > 0)[0][-1])))
        dc = [dist(x64, x[c]) for c in cands]
        pots = np.array([np.minimum(d2, v).sum() for v in dc])
        best = int(np.argmin(pots))
        others = [p for c, p in zip(cands, pots) if not np.array_equal(x[c], x[cands[best]])]   # equal rows: equal bits
        if others and min(others) - pots[best] <= 1e-9 * pots[best]:
            ambiguous = True
        idx.append(cands[best])
        d2 = np.minimum(d2, dc[best])
    return idx, ambiguous


def nearest(x, centres):
    """float64 labels, distances to the nearest centre, and the number of events whose two nearest centres are within FP32
    rounding of each other (either label is then legal for the device)."""
    x64, c64 = x.astype(np.float64), centres.astype(np.float64)
    d = ((x64[:, None, :] - c64[None, :, :]) ** 2).sum(-1)
    lab = np.argmin(d, 1)
    if centres.shape[0] > 1:
        two = np.partition(d, 1, axis=1)[:, :2]
        amb = int(((two[:, 1] - two[:, 0]) <= AMBIG * np.maximum(two[:, 1], 1e-30)).sum())
    else:
        amb = 0
    return lab, d[np.arange(len(x)), lab], amb


def labelings(x, centres, most=4):
    """Every legal labelling: the float64 labels, with each event whose two nearest centres lie within FP32 rounding of
    each other given either of them (at most `most` such events)."""
    x64, c64 = x.astype(np.float64), centres.astype(np.float64)
    d = ((x64[:, None, :] - c64[None, :, :]) ** 2).sum(-1)
    order = np.argsort(d, 1, kind="stable")[:, :2]
    first, second = d[np.arange(len(x)), order[:, 0]], d[np.arange(len(x)), order[:, 1]]
    amb = np.nonzero((second - first) <= AMBIG * np.maximum(second, 1e-30))[0]
    assert len(amb) <= most, f"{len(amb)} events within FP32 rounding of two centres: pick other data"
    for bits in range(1 << len(amb)):
        lab = order[:, 0].copy()
        for j, i in enumerate(amb):
            if bits >> j & 1:
                lab[i] = order[i, 1]
        yield lab


def onehot(lab, K):
    g = np.zeros((K, len(lab)), np.float32)
    g[lab, np.arange(len(lab))] = 1.0
    return g


def centroids(x, lab, old):
    c = old.astype(np.float64).copy()
    for k in range(len(old)):
        m = lab == k
        if m.any():
            c[k] = x[m].astype(np.float64).mean(0)
    return c


def data(pkg, n, D, seed):
    return pkg.synth.make_blobs(n, D, 12, seed=seed)


def engine(pkg, ev, Kmax, mstep=None):
    eng = pkg.Engine(ev, Kmax)
    if mstep is not None:
        eng.set_option("mstep_path", mstep)
    return eng


def mstep_launches(eng):
    p = eng.profile()
    return int(p["mstep_tensor_launches"]), int(p["mstep_simt_launches"])


def check_onehot_mstep(pkg, x, cl, centres, K, tensor, what):
    """N, means, R returned against the exact float64 M-step on the numpy labels of the returned centres, finalised by the
    same host code with the same avgvar.  Bar: MSTEP_TOL on the wgmma M-step; 2 float32 ulps (the parameters' own rounding)
    on the FP64 SIMT M-step."""
    lab, _, amb = nearest(x, centres)
    assert amb == 0, f"{what}: {amb} events have two nearest centres within FP32 rounding: pick other data"
    sh = standardise(x)[0]
    st = exact_mstep_stats(x, onehot(lab, K), sh)
    ref = pkg.Clusters(K, x.shape[1])
    ref.avgvar[:K] = cl.avgvar[:K]
    pkg.host_finalize(st, sh, ref, K)
    e = param_errors(cl.N[:K], cl.means[:K], cl.R[:K], ref.N[:K], ref.means[:K], ref.R[:K], sh)
    print(f"\n[seed-kmeans] {what}: N {e['N']:.2e}  mean {e['mean']:.2e}  R {e['R']:.2e}")
    if tensor:
        assert e["worst"] <= 1.0, (what, e)
    else:
        assert max(e["N"], e["mean"], e["R"]) <= 2.4e-7, (what, e)
    np.testing.assert_array_equal(cl.N[:K], ref.N[:K])      # one-hot memberships: the counts are exact on both paths
    return lab


# ---- 1 + 2. k-means++ bit for bit, one-hot M-step -------------------------------------------------------------------------
EXACT = [(D, K) for D in (4, 5, 8, 16, 24, 32) for K in (1, 2, 7, 64, 130)] + [(4, 512)]


@pytest.mark.parametrize("D,K", EXACT)
def test_kmeanspp_exact_and_onehot_mstep(pkg, D, K):
    x = data(pkg, 20_011, D, seed=900 + D)
    seed = 1000 * D + K
    for _ in range(8):                                        # the first seed whose choices and labels are unambiguous
        idx, amb = kmeanspp_ref(x, K, seed)
        if not amb and nearest(x, x[idx])[2] == 0:
            break
        seed += 1
    with engine(pkg, x, K) as eng:
        eng.profile(reset=True)
        cl, cent, it, inertia = eng.seed_kmeans(K, max_iter=0, seed=seed)
        launches = mstep_launches(eng)
    np.testing.assert_array_equal(cent, x[idx])
    assert it == 0
    tensor = D in TENSOR_M_D
    assert launches == ((1, 0) if tensor else (0, 1)), launches
    lab = check_onehot_mstep(pkg, x, cl, cent, K, tensor, f"D={D} K={K}")
    _, dmin, _ = nearest(x, cent)
    assert abs(inertia - dmin.sum()) <= 1e-6 * dmin.sum() + 1e-12, (inertia, dmin.sum())
    assert np.bincount(lab, minlength=K).min() >= 1     # k-means++ centres are events: no cluster is empty


@pytest.mark.parametrize("D", [5, 24])
def test_simt_mstep_forced(pkg, D):
    """mstep_path = SIMT at a D the wgmma M-step covers: the FP64 M-step forms the statistics."""
    K = 9
    x = data(pkg, 20_011, D, seed=950 + D)
    with engine(pkg, x, K, pkg.PATH_SIMT) as eng:
        eng.profile(reset=True)
        cl, cent, _, _ = eng.seed_kmeans(K, max_iter=0, seed=3)
        assert mstep_launches(eng) == (0, 1)
    idx, _ = kmeanspp_ref(x, K, 3)
    np.testing.assert_array_equal(cent, x[idx])
    check_onehot_mstep(pkg, x, cl, cent, K, False, f"SIMT D={D}")


def test_every_event_a_centre(pkg):
    """K = n_global distinct events: every event is chosen exactly once."""
    D, n = 8, 300
    x = np.random.default_rng(5).standard_normal((n, D)).astype(np.float32)
    with engine(pkg, x, n) as eng:
        cl, cent, _, inertia = eng.seed_kmeans(n, max_iter=0, seed=11)
    idx, _ = kmeanspp_ref(x, n, 11)
    np.testing.assert_array_equal(cent, x[idx])
    assert sorted(idx) == list(range(n))
    assert inertia == 0.0
    np.testing.assert_array_equal(cl.N[:n], np.ones(n, np.float32))


def test_fewer_distinct_events_than_k(pkg):
    """3 distinct rows, K = 5: centres 4 and 5 repeat the first; their clusters are empty and follow the N < 0.5 rules."""
    D, K = 8, 5
    rows = np.random.default_rng(6).standard_normal((3, D)).astype(np.float32)
    x = rows[np.random.default_rng(7).integers(0, 3, 3000)]
    with engine(pkg, x, K) as eng:
        cl, cent, _, _ = eng.seed_kmeans(K, max_iter=0, seed=2)
    idx, _ = kmeanspp_ref(x, K, 2)
    np.testing.assert_array_equal(cent, x[idx])
    np.testing.assert_array_equal(cent[3], cent[0])
    np.testing.assert_array_equal(cent[4], cent[0])
    assert len({tuple(r) for r in cent[:3]}) == 3
    for k in (3, 4):
        assert cl.N[k] == 0.0 and cl.pi[k] <= 1e-9              # (the mixing weight's floor)
        np.testing.assert_array_equal(cl.means[k], np.zeros(D, np.float32))
        np.testing.assert_array_equal(cl.R[k], np.eye(D, dtype=np.float32))
    assert cl.N[:3].sum() == 3000


# ---- 3. Lloyd -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", [24, 5])
def test_lloyd_steps(pkg, D):
    """Inertia never rises over max_iter = 0 .. 6, and the run with max_iter = m returns the centroids of the labels that
    the run with max_iter = m - 1 returned centres give."""
    K = 16
    x = data(pkg, 30_011, D, seed=970 + D)
    runs = []
    with engine(pkg, x, K) as eng:
        for m in range(7):
            eng.profile(reset=True)
            cl, cent, it, inertia = eng.seed_kmeans(K, max_iter=m, seed=21)
            t, s = mstep_launches(eng)
            assert (s == 0) if D in TENSOR_M_D else (t == 0), (t, s)
            assert 1 <= t + s <= m + 1
            runs.append((cent, it, inertia))
    for m in range(1, 7):
        assert runs[m][2] <= runs[m - 1][2] * (1 + 1e-6), (m, runs[m][2], runs[m - 1][2])
        if runs[m - 1][1] < m - 1:
            continue                                            # converged earlier: nothing more to compare
        scale = np.abs(x).max()
        errs = []
        for lab in labelings(x, runs[m - 1][0]):                 # an event within FP32 rounding of two centres: either label
            want = centroids(x, lab, runs[m - 1][0])
            errs.append(float((np.abs(runs[m][0] - want) / (np.abs(want) + scale)).max()))
        assert min(errs) <= MSTEP_TOL["mean"], (m, errs)


def test_lloyd_converges_like_sklearn(pkg):
    D, K = 16, 12
    x = data(pkg, 30_011, D, seed=990)
    with engine(pkg, x, K) as eng:
        _, c0, _, _ = eng.seed_kmeans(K, max_iter=0, seed=8)
        _, cent, it, inertia = eng.seed_kmeans(K, max_iter=300, seed=8)
    assert it < 300
    x64 = x.astype(np.float64)
    c = c0.astype(np.float64)
    lab = None
    for _ in range(300):                                       # float64 Lloyd, tol = 0: until no label changes
        new, _, _ = nearest(x64, c)
        if lab is not None and np.array_equal(new, lab):
            break
        lab = new
        c = centroids(x64, lab, c)
    ref_inertia = ((x64 - c[lab]) ** 2).sum()
    np.testing.assert_allclose(cent, c, rtol=1e-5, atol=1e-5 * np.abs(c).max())
    assert abs(inertia - ref_inertia) <= 1e-6 * ref_inertia, (inertia, ref_inertia)
    try:
        from sklearn.cluster import KMeans
    except ImportError:
        return
    km = KMeans(K, init=c0.astype(np.float64), n_init=1, algorithm="lloyd", tol=0, max_iter=300).fit(x64)
    np.testing.assert_allclose(cent, km.cluster_centers_, rtol=1e-5, atol=1e-5 * np.abs(c).max())
    assert abs(inertia - km.inertia_) <= 1e-6 * km.inertia_


# ---- 4. state -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", [24, 12])
def test_state_equals_set_clusters(pkg, D):
    """Seeding then EM equals gmm_set_clusters(host_out) then EM, bit for bit (D = 24: tensor E-step, D = 12: SIMT E-step;
    both run the wgmma M-step, whose sums do not depend on the launch)."""
    K = 10
    x = data(pkg, 20_011, D, seed=1010 + D)
    with engine(pkg, x, K) as eng:
        cl, _, _, _ = eng.seed_kmeans(K, max_iter=5, seed=4)
        with pytest.raises(pkg.GmmError) as ei:
            eng.mstep(K)
        assert ei.value.code == ERR_STATE
        lab, mr, lp, ll = eng.score(K, x[:1000])
        assert np.isfinite(lp).all() and (lab >= 0).all()
        ll_a, it_a = eng.em(K, 10, 10)
        a = eng.get_clusters(K, with_memberships=True)
        eng.set_clusters(K, cl)
        ll_b, it_b = eng.em(K, 10, 10)
        b = eng.get_clusters(K, with_memberships=True)
    assert (ll_a, it_a) == (ll_b, it_b)
    for f in ("N", "pi", "constant", "means", "R", "Rinv", "memberships"):
        np.testing.assert_array_equal(getattr(a, f)[:K], getattr(b, f)[:K], err_msg=f)


# ---- 5. determinism and errors --------------------------------------------------------------------------------------------
def test_deterministic_and_seed_dependent(pkg):
    D, K = 16, 20
    x = data(pkg, 20_011, D, seed=1030)
    with engine(pkg, x, K) as eng:
        a = eng.seed_kmeans(K, max_iter=10, seed=99)
        b = eng.seed_kmeans(K, max_iter=10, seed=99)
        c = eng.seed_kmeans(K, max_iter=0, seed=100)
        d = eng.seed_kmeans(K, max_iter=0, seed=99)
    np.testing.assert_array_equal(a[1], b[1])
    assert a[2:] == b[2:]
    for f in ("N", "pi", "constant", "avgvar", "means", "R", "Rinv"):
        np.testing.assert_array_equal(getattr(a[0], f)[:K], getattr(b[0], f)[:K], err_msg=f)
    assert not np.array_equal(c[1], d[1])


def test_errors(pkg):
    x = data(pkg, 10, 8, seed=1)
    with engine(pkg, x, 16) as eng:
        for K, m in ((0, 0), (17, 0), (11, 0), (4, -1)):
            with pytest.raises(pkg.GmmError) as ei:
                eng.seed_kmeans(K, max_iter=m)
            assert ei.value.code == ERR_ARG, (K, m)
        eng.seed_kmeans(10, max_iter=0)                          # K = n_global is legal


# ---- 6. quality -----------------------------------------------------------------------------------------------------------
def _blobs_missed(means, centres):
    owner = np.argmin(((means[:, None, :] - centres[None]) ** 2).sum(-1), 1)
    return len(centres) - len(set(owner.tolist()))


@pytest.mark.parametrize("order", ["shuffled", "sorted"])
def test_better_than_evenly_spaced_seeds(pkg, order):
    D, K, seed = 16, 16, 7
    x = pkg.synth.make_blobs(50_000, D, K, seed=seed)
    centres = np.random.default_rng(seed).uniform(-10.0, 10.0, size=(K, D))   # make_blobs' first draws
    if order == "sorted":
        own = np.argmin(((x.astype(np.float64)[:, None, :] - centres[None]) ** 2).sum(-1), 1)
        x = np.ascontiguousarray(x[np.argsort(own, kind="stable")])
    with engine(pkg, x, K) as eng:
        eng.seed(K)
        ll_even, _ = eng.em(K, 100, 100)
        m_even = eng.get_clusters(K).means[:K].astype(np.float64)
        eng.seed_kmeans(K, max_iter=300, seed=0)
        ll_km, _ = eng.em(K, 100, 100)
        m_km = eng.get_clusters(K).means[:K].astype(np.float64)
    miss_even, miss_km = _blobs_missed(m_even, centres), _blobs_missed(m_km, centres)
    print(f"\n[seed-kmeans] {order}: loglik evenly spaced {ll_even:.6e} k-means {ll_km:.6e}; blobs missed {miss_even} / {miss_km}")
    assert ll_km > ll_even
    assert miss_km < miss_even


# ---- 7. sharded -----------------------------------------------------------------------------------------------------------
def _sharded(pkg, x, K, G, max_iter, seed):
    N = len(x)
    uid = pkg.nccl_unique_id() if G > 1 else None
    out, errs = [None] * G, [None] * G

    def worker(g):
        try:
            b, n = pkg.shard_range(N, G, g)
            with pkg.Engine(np.ascontiguousarray(x[b:b + n]), K, device=g, n_global=N, offset=b) as eng:
                eng.comm_init(G, g, uid)
                out[g] = eng.seed_kmeans(K, max_iter=max_iter, seed=seed)
        except Exception as ex:  # noqa: BLE001
            errs[g] = ex

    ts = [threading.Thread(target=worker, args=(g,)) for g in range(G)]
    for t in ts:
        t.start()
    for t in ts:
        t.join(timeout=600)
    for g in range(G):
        assert errs[g] is None, f"rank {g}: {errs[g]}"
        assert out[g] is not None, f"rank {g} did not finish"
    return out


@pytest.mark.parametrize("max_iter", [0, 20])
def test_two_ranks_match_one(pkg, max_iter):
    if gpu_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    D, K = 16, 24
    x = data(pkg, 60_001, D, seed=1050)
    one = _sharded(pkg, x, K, 1, max_iter, 5)[0]
    two = _sharded(pkg, x, K, 2, max_iter, 5)
    if max_iter == 0:
        np.testing.assert_array_equal(two[0][1], one[1])
    np.testing.assert_array_equal(two[0][1], two[1][1])
    assert_params_close(two[0][0], one[0], K)
