"""Weighted EM (gmm_set_weights, Engine.set_weights) on the GPU (run with -m gpu on an H100).

Weighted EM is EM over the multiset in which event n appears w_n times: unit weights change no bit, uniform powers of two
scale the statistics and the log-likelihood exactly, integer weights equal replicated rows and zero weights removed rows.
The tensor M-step serves weights with one positive value (tests/test_weights_error_model.py); other weights run the FP64
SIMT M-step."""
import threading

import numpy as np
import pytest

from conftest import RUN_RTOL_N, assert_params_close, fitted_params, gpu_count
from test_gpu_mstep_tc import MSTEP_D, engine
from test_mstep_error_model import param_errors, standardise

pytestmark = pytest.mark.gpu

FIELDS = ("N", "pi", "constant", "means", "R", "Rinv")


@pytest.fixture(scope="module")
def loaded(pkg):
    pkg.load_library()
    return pkg


def same_params(a, b, K, exact=True):
    for f in FIELDS:
        x, y = getattr(a, f)[:K], getattr(b, f)[:K]
        if exact:
            np.testing.assert_array_equal(x, y, err_msg=f)
        else:
            np.testing.assert_allclose(x, y, rtol=1e-6, atol=1e-6 * max(1.0, float(np.abs(y).max())), err_msg=f)


def weighted_stats(ev, memb, w, shift, K):
    """S0 | S1 | S2 (lower triangle) per cluster of sum w g phi(x - shift), float64, then the log-likelihood slot."""
    y = ev.astype(np.float64) - shift
    D = y.shape[1]
    i, j = np.tril_indices(D)
    rows = []
    for k in range(K):
        g = memb[k].astype(np.float64) * w.astype(np.float64)
        S2 = (g[:, None] * y).T @ y
        rows.append(np.concatenate([[g.sum()], g @ y, S2[i, j]]))
    return np.concatenate(rows + [[0.0]])


def run_steps(pkg, ev, K, cl, w, estep, mstep, Kmax=None, dev_fin=1):
    """(E-step log-likelihood, parameters after gmm_mstep, memberships, two em_iterations batches, gmm_em, profile)."""
    with engine(pkg, ev, Kmax or K, estep=estep, mstep=mstep) as eng:
        eng.set_option("finalize", dev_fin)
        if w is not None:
            eng.set_weights(w)
        eng.set_clusters(K, cl)
        ll = eng.estep(K)
        memb = eng.get_clusters(K, with_memberships=True).memberships[:K].copy()
        eng.mstep(K)
        after_m = eng.get_clusters(K)
        eng.set_clusters(K, cl)
        eng.estep(K)
        lli = (eng.em_iterations(K, 2), eng.em_iterations(K, 2))
        batches = eng.get_clusters(K)
        eng.set_clusters(K, cl)
        lle = eng.em(K, 3, 3)
        em = eng.get_clusters(K)
        prof = eng.profile()
    return dict(ll=ll, mstep=after_m, memb=memb, lli=lli, batches=batches, lle=lle, em=em, prof=prof)


UNIT_SHAPES = ([(D, K, "tensor") for D in (8, 16, 24) for K in (7, 33, 64, 100)] +
               [(12, 16, "tensor-m"), (20, 16, "tensor-m"), (32, 8, "simt")])


@pytest.mark.parametrize("D,K,path", UNIT_SHAPES)
def test_unit_weights_equal_no_weights(loaded, oracle64, D, K, path):
    """Unit weights change no bit where the M-step is the wgmma kernel (its addition order is fixed); the FP64 SIMT
    M-step adds with atomics, so there the parameters agree to double rounding."""
    pkg = loaded
    ev = pkg.synth.make_blobs(20_000, D, min(K, 16), seed=800 + D)
    cl = fitted_params(pkg, oracle64, ev, K)
    estep = {"tensor": pkg.PATH_AUTO, "tensor-m": pkg.PATH_AUTO, "simt": pkg.PATH_SIMT}[path]
    mstep = pkg.PATH_SIMT if path == "simt" else pkg.PATH_TENSOR
    a = run_steps(pkg, ev, K, cl, None, estep, mstep)
    b = run_steps(pkg, ev, K, cl, np.ones(len(ev), np.float32), estep, mstep)
    exact = path != "simt"
    if path == "tensor":
        np.testing.assert_array_equal(a["memb"], b["memb"])
    for key in ("ll", "lli", "lle"):
        if path == "tensor":
            assert a[key] == b[key], key
        else:                                    # the SIMT E-step adds its log-likelihood with atomics
            np.testing.assert_allclose(np.ravel(a[key]), np.ravel(b[key]), rtol=1e-6)
    for key in ("mstep", "batches", "em"):
        same_params(a[key], b[key], K, exact=exact)
    if path != "simt":
        assert b["prof"]["mstep_tensor_launches"] > 0 and b["prof"]["mstep_simt_launches"] == 0


def test_unit_weights_fit_equals_no_weights(loaded):
    pkg = loaded
    ev = pkg.synth.make_blobs(20_000, 16, 10, seed=811)
    out = []
    for w in (None, np.ones(len(ev), np.float32)):
        with pkg.Engine(ev, 12) as eng:
            if w is not None:
                eng.set_weights(w)
            out.append(eng.fit(12, 0, 5, 5))
    (ia, ra, sa), (ib, rb, sb) = out
    assert (ia, ra) == (ib, rb)
    same_params(sa, sb, ia)


@pytest.mark.parametrize("j", [-3, 5])
def test_power_of_two_weights_scale_exactly(loaded, oracle64, j):
    pkg = loaded
    D, K = 16, 33
    ev = pkg.synth.make_blobs(20_000, D, 16, seed=820)
    cl = fitted_params(pkg, oracle64, ev, K)
    cl.avgvar[:K] = 0.0                                   # (avgvar is added to the sum before the division by N)
    out = []
    for w in (None, np.full(len(ev), 2.0 ** j, np.float32)):
        with engine(pkg, ev, K, estep=pkg.PATH_AUTO, mstep=pkg.PATH_TENSOR) as eng:
            if w is not None:
                eng.set_weights(w)
            eng.set_clusters(K, cl)
            ll = eng.estep(K)
            eng.mstep(K)
            out.append((ll, eng.get_clusters(K)))
    (la, a), (lb, b) = out
    assert lb == np.float32(la * 2.0 ** j)
    np.testing.assert_array_equal(b.N[:K], a.N[:K] * np.float32(2.0 ** j))
    for f in ("pi", "means", "R"):
        np.testing.assert_array_equal(getattr(b, f)[:K], getattr(a, f)[:K], err_msg=f)


def em_run(pkg, ev, K, cl, w, path, iters=10):
    with pkg.Engine(ev, K) as eng:
        eng.set_option("path", path)
        if w is not None:
            eng.set_weights(w)
        eng.set_clusters(K, cl)
        ll, it = eng.em(K, iters, iters)
        return eng.get_clusters(K), ll


@pytest.mark.parametrize("path", ["simt", "auto"])
def test_integer_weights_equal_replicated_rows(loaded, oracle64, path):
    pkg = loaded
    D, K = 16, 8
    ev = pkg.synth.make_blobs(30_000, D, 8, seed=830)
    w = np.random.default_rng(831).integers(1, 6, len(ev)).astype(np.float32)
    rep = np.repeat(ev, w.astype(np.int64), axis=0)
    cl = fitted_params(pkg, oracle64, ev, K)
    p = {"simt": pkg.PATH_SIMT, "auto": pkg.PATH_AUTO}[path]
    got, ll = em_run(pkg, ev, K, cl, w, p)
    ref_e, ll_e = em_run(pkg, rep, K, cl, None, p)
    assert abs(ll - ll_e) <= 1e-5 * abs(ll_e)
    assert_params_close(got, ref_e, K, rtol_N=RUN_RTOL_N)
    ref = pkg.Clusters(K, D, len(rep))
    for f in FIELDS + ("avgvar",):
        getattr(ref, f)[:K] = getattr(cl, f)[:K]
    ll_o, _ = oracle64.em(oracle64.transpose(rep), ref, K, 10, 10)
    assert abs(ll - ll_o) <= 1e-5 * abs(ll_o)
    assert_params_close(got, ref, K, rtol_N=RUN_RTOL_N)


def test_zero_weights_equal_removed_rows(loaded, oracle64):
    pkg = loaded
    D, K = 24, 12
    ev = pkg.synth.make_blobs(40_000, D, 12, seed=840)
    keep = np.random.default_rng(841).uniform(size=len(ev)) < 0.6
    cl = fitted_params(pkg, oracle64, ev, K)
    with pkg.Engine(ev, K) as eng:
        eng.set_weights(keep.astype(np.float32))
        eng.set_clusters(K, cl)
        ll, _ = eng.em(K, 10, 10)
        got = eng.get_clusters(K)
        assert eng.profile()["mstep_simt_launches"] == 0          # one positive value: the tensor M-step serves it
    ref, ll_r = em_run(pkg, np.ascontiguousarray(ev[keep]), K, cl, None, pkg.PATH_AUTO)
    assert abs(ll - ll_r) <= 1e-5 * abs(ll_r)
    assert_params_close(got, ref, K, rtol_N=RUN_RTOL_N)


FRACTIONAL = ([(D, K, 20_000, law) for D in MSTEP_D for K in (1, 33, 100) for law in ("uniform", "constant")] +
              [(24, 33, n, law) for n in (1, 31, 300_001) for law in ("uniform", "constant")])


@pytest.mark.parametrize("D,K,n,law", FRACTIONAL)
def test_fractional_weights_one_mstep(loaded, oracle64, D, K, n, law):
    """One M-step against sum w g phi in float64 on the read-back memberships, at the per-cluster bar.  "uniform" weights
    in [0.5, 1] run the FP64 SIMT M-step (one event: the wgmma M-step), "constant" 0.7 with 30 % zeros the wgmma M-step."""
    pkg = loaded
    fit = pkg.synth.make_blobs(20_000, D, min(K, 16), seed=850 + D)
    cl = fitted_params(pkg, oracle64, fit, K)
    ev = np.ascontiguousarray(fit[:n]) if n <= len(fit) else pkg.synth.make_blobs(n, D, min(K, 16), seed=850 + D)
    rng = np.random.default_rng(851)
    w = (rng.uniform(0.5, 1.0, n) if law == "uniform" else np.where(rng.uniform(size=n) < 0.7, 0.7, 0.0)).astype(np.float32)
    if not w.any():
        w[0] = 0.7
    check_one_mstep(pkg, ev, cl, K, w, K, law)


def check_one_mstep(pkg, ev, cl, K, w, Kmax, law):
    with engine(pkg, ev, Kmax, estep=pkg.PATH_AUTO) as eng:
        eng.set_weights(w)
        eng.set_clusters(K, cl)
        eng.estep(K)
        memb = eng.get_clusters(K, with_memberships=True).memberships[:K].copy()
        eng.mstep(K)
        got = eng.get_clusters(K)
        prof = eng.profile()
    pos = w[w > 0]
    assert (prof["mstep_tensor_launches"] == 1) == (pos.max() == pos.min())      # one positive value: the wgmma M-step
    shift = standardise(ev)[0]
    ref = pkg.Clusters(K, ev.shape[1])
    ref.avgvar[:K] = got.avgvar[:K]
    pkg.host_finalize(weighted_stats(ev, memb, w, shift, K), shift, ref, K)
    e = param_errors(got.N[:K], got.means[:K], got.R[:K], ref.N[:K], ref.means[:K], ref.R[:K], shift)
    assert e["worst"] <= 1.0, e


def test_fractional_weights_kmax128_at_k64(loaded, oracle64):
    pkg = loaded
    ev = pkg.synth.make_blobs(20_000, 24, 16, seed=860)
    cl = fitted_params(pkg, oracle64, ev, 64)
    w = np.random.default_rng(861).uniform(0.5, 1.0, len(ev)).astype(np.float32)
    check_one_mstep(pkg, ev, cl, 64, w, 128, "uniform")
    check_one_mstep(pkg, ev, cl, 64, np.full(len(ev), 0.7, np.float32), 128, "constant")


@pytest.mark.parametrize("outside", [False, True])
def test_admission_rule(loaded, oracle64, outside):
    """Equal positive weights (and zeros) run the tensor M-step; one weight a float ulp above the others runs SIMT, and is
    an error under GMM_PATH_TENSOR."""
    pkg = loaded
    D, K = 16, 8
    ev = pkg.synth.make_blobs(20_000, D, 8, seed=870)
    cl = fitted_params(pkg, oracle64, ev, K)
    w = np.full(len(ev), 3.0, np.float32)
    w[::5] = 0.0
    if outside:
        w[1] = np.nextafter(np.float32(3.0), np.float32(4.0))
    with pkg.Engine(ev, K) as eng:
        eng.set_weights(w)
        eng.set_clusters(K, cl)
        eng.estep(K)
        eng.mstep(K)
        p = eng.profile()
        assert (p["mstep_tensor_launches"], p["mstep_simt_launches"]) == ((0, 1) if outside else (1, 0))
        eng.set_option("mstep_path", pkg.PATH_TENSOR)
        eng.set_clusters(K, cl)
        eng.estep(K)
        if outside:
            with pytest.raises(pkg.GmmError):
                eng.mstep(K)
        else:
            eng.mstep(K)


def test_device_finalisation_replay_with_weights(loaded, oracle64):
    """A forced host replay (option finalize_fault_iter) of a weighted batch equals the all-host run bit for bit, and so
    does a device batch without one (weights of one positive value: the wgmma M-step, whose sums are reproducible)."""
    pkg = loaded
    D, K = 16, 20
    ev = pkg.synth.make_blobs(20_000, D, 16, seed=880)
    cl = fitted_params(pkg, oracle64, ev, K)
    rng = np.random.default_rng(881)
    w = np.where(rng.uniform(size=len(ev)) < 0.8, 0.5, 0.0).astype(np.float32)
    out = []
    for fin, fault in ((1, 1), (0, -1), (1, -1)):
        with pkg.Engine(ev, K) as eng:
            eng.set_option("finalize", fin)
            eng.set_option("finalize_fault_iter", fault)
            eng.set_weights(w)
            eng.set_clusters(K, cl)
            eng.estep(K)
            ll = eng.em_iterations(K, 4)
            out.append((ll, eng.get_clusters(K, with_memberships=True)))
    (la, a), (lb, b), (lc, c) = out
    assert la == lb
    same_params(a, b, K)
    np.testing.assert_array_equal(a.memberships[:K], b.memberships[:K])
    assert lc == lb
    same_params(c, b, K)


def test_errors_and_state(loaded, oracle64):
    pkg = loaded
    D, K = 16, 8
    ev = pkg.synth.make_blobs(20_000, D, 8, seed=890)
    cl = fitted_params(pkg, oracle64, ev, K)
    n = len(ev)
    w = np.random.default_rng(891).uniform(0.5, 2.0, n).astype(np.float32)
    with pkg.Engine(ev, K) as plain:
        s_plain = plain.seed(K)
        plain.set_clusters(K, cl)
        ll_plain = plain.estep(K)
        m_plain = plain.get_clusters(K, with_memberships=True).memberships[:K].copy()
        plain.mstep(K)
        p_plain = plain.get_clusters(K)
    with pkg.Engine(ev, K) as eng:
        total = eng.set_weights(w)
        assert total == float(np.cumsum(w.astype(np.float64))[-1])   # summed in event order
        s_w = eng.seed(K)                                     # seeding ignores the weights
        same_params(s_w, s_plain, K)
        eng.set_clusters(K, cl)
        ll_w = eng.estep(K)
        m_w = eng.get_clusters(K, with_memberships=True).memberships[:K]
        np.testing.assert_array_equal(m_w, m_plain)          # posteriors do not depend on the weights
        for bad in (np.nan, np.inf, -1.0):
            wb = w.copy()
            wb[7] = bad
            with pytest.raises(pkg.GmmError):
                eng.set_weights(wb)
        with pytest.raises(pkg.GmmError):
            eng.set_weights(np.zeros(n, np.float32))
        assert eng.estep(K) == ll_w                           # the rejected calls left the weights in effect
        eng.set_weights(w)
        with pytest.raises(pkg.GmmError):
            eng.mstep(K)                                      # setting weights marks the memberships stale
        eng.upload_events(ev)                                 # an upload keeps the weights
        eng.set_clusters(K, cl)
        assert eng.estep(K) == ll_w
        assert eng.set_weights(None) == float(n)             # NULL: as if weights had never been set
        eng.set_clusters(K, cl)
        assert eng.estep(K) == ll_plain
        eng.mstep(K)
        same_params(eng.get_clusters(K), p_plain, K)


def _sharded(pkg, ev, w, K, G, iters):
    N = len(ev)
    uid = pkg.nccl_unique_id() if G > 1 else None
    out, errs = [None] * G, [None] * G

    def worker(g):
        try:
            b, n = pkg.shard_range(N, G, g)
            with pkg.Engine(np.ascontiguousarray(ev[b:b + n]), K, device=g, n_global=N, offset=b) as eng:
                if G > 1:
                    eng.comm_init(G, g, uid)
                total = eng.set_weights(np.ascontiguousarray(w[b:b + n]))
                eng.seed(K)
                ll, _ = eng.em(K, iters, iters)
                out[g] = (eng.get_clusters(K), ll, total)
        except Exception as ex:  # noqa: BLE001
            errs[g] = ex

    ts = [threading.Thread(target=worker, args=(g,)) for g in range(G)]
    for t in ts:
        t.start()
    for t in ts:
        t.join(timeout=600)
    assert errs == [None] * G, errs
    return out


def test_two_gpus_weighted_equals_single(loaded):
    if gpu_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    pkg = loaded
    N, D, K, iters = 120_003, 16, 12, 8
    ev = pkg.synth.make_blobs(N, D, K, seed=895)
    w = np.random.default_rng(896).uniform(0.25, 3.0, N).astype(np.float32)
    one = _sharded(pkg, ev, w, K, 1, iters)[0]
    two = _sharded(pkg, ev, w, K, 2, iters)
    for f in FIELDS:
        np.testing.assert_array_equal(getattr(two[1][0], f)[:K], getattr(two[0][0], f)[:K], err_msg=f)
    assert two[0][2] == two[1][2] and two[0][1] == two[1][1]
    assert abs(two[0][2] - one[2]) <= 1e-12 * one[2]
    assert abs(two[0][1] - one[1]) <= 2e-6 * abs(one[1])
    assert_params_close(two[0][0], one[0], K, rtol=2e-6)


@pytest.mark.parametrize("mstep", ["auto", "tensor"])
def test_score_stats_and_condition_stats_ignore_weights(loaded, oracle64, mstep):
    """gmm_score_stats and gmm_condition_stats do not read the shard: with fractional weights set (which send the
    context's own M-step to the FP64 SIMT kernel) they give the same bits and run the same kernels as without, also when
    the M-step is forced to GMM_PATH_TENSOR."""
    pkg = loaded
    D, K = 16, 12
    ev = pkg.synth.make_blobs(20_000, D, 12, seed=900)
    new = pkg.synth.make_blobs(50_000, D, 12, seed=901)
    cl = fitted_params(pkg, oracle64, ev, K)
    obs = [0, 2, 3, 7, 8, 11, 15]
    w = np.random.default_rng(902).uniform(0.5, 2.0, len(ev)).astype(np.float32)
    out = []
    for weights in (None, w):
        with pkg.Engine(ev, K) as eng:
            if mstep == "tensor":
                eng.set_option("mstep_path", pkg.PATH_TENSOR)
            if weights is not None:
                eng.set_weights(weights)
            eng.set_clusters(K, cl)
            ss = eng.score_stats(K, new, stats=True, memberships=True)
            cs = eng.condition_stats(K, obs, np.ascontiguousarray(new[:, obs]), stats=True, memberships=True)
            sp = {k: v for k, v in eng.score_stats_profile().items() if not k.endswith("_ms")}
            cp = {k: v for k, v in eng.condition_stats_profile().items() if not k.endswith("_ms")}
            out.append((ss, cs, sp, cp))
    (ssa, csa, spa, cpa), (ssb, csb, spb, cpb) = out
    for a, b in ((ssa, ssb), (csa, csb)):
        np.testing.assert_array_equal(a[0][:-1], b[0][:-1])                 # statistics
        np.testing.assert_allclose(a[0][-1], b[0][-1], rtol=1e-12)          # log-likelihood slot: added with atomics
        np.testing.assert_array_equal(a[1], b[1])                           # shift
        np.testing.assert_array_equal(a[2], b[2])                           # memberships
    assert spa == spb and cpa == cpb
    assert spb["mstep_tensor_chunks"] > 0 and spb["mstep_simt_chunks"] == 0
    assert cpb["mstep_tensor_chunks"] > 0 and cpb["mstep_simt_chunks"] == 0


def test_seed_kmeans_ignores_weights(loaded):
    """gmm_seed_kmeans runs its Lloyd and final M-steps unweighted: with fractional weights set (which would send a
    weighted M-step to the FP64 SIMT kernel) its outputs and M-step launches are those of a context without weights."""
    pkg = loaded
    D, K = 16, 20
    ev = pkg.synth.make_blobs(30_000, D, 16, seed=910)
    w = np.random.default_rng(911).uniform(0.5, 2.0, len(ev)).astype(np.float32)
    out = []
    for weights in (None, w):
        with pkg.Engine(ev, K) as eng:
            if weights is not None:
                eng.set_weights(weights)
            cl, cent, it, inertia = eng.seed_kmeans(K, max_iter=20, seed=5)
            p = eng.profile()
            out.append((cl, cent, it, inertia, p["mstep_tensor_launches"], p["mstep_simt_launches"]))
    (ca, ea, ia, na, ta, sa), (cb, eb, ib, nb, tb, sb) = out
    same_params(ca, cb, K)
    np.testing.assert_array_equal(ea, eb)
    assert (ia, na, ta, sa) == (ib, nb, tb, sb)
    assert tb > 0 and sb == 0


def test_two_gpus_mixed_null_rejected_on_every_rank(loaded):
    """Weights on one rank and NULL on the other: GMM_ERR_ARG on both (they would disagree on N = sum w)."""
    if gpu_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    pkg = loaded
    N, D, K = 40_001, 8, 4
    ev = pkg.synth.make_blobs(N, D, K, seed=920)
    uid = pkg.nccl_unique_id()
    res = [None, None]

    def worker(g):
        try:
            b, n = pkg.shard_range(N, 2, g)
            with pkg.Engine(np.ascontiguousarray(ev[b:b + n]), K, device=g, n_global=N, offset=b) as eng:
                eng.comm_init(2, g, uid)
                try:
                    eng.set_weights(np.ones(n, np.float32) if g == 0 else None)
                    res[g] = "accepted"
                except pkg.GmmError:
                    res[g] = "rejected"
        except Exception as ex:  # noqa: BLE001
            res[g] = ex

    ts = [threading.Thread(target=worker, args=(g,)) for g in range(2)]
    for t in ts:
        t.start()
    for t in ts:
        t.join(timeout=600)
    assert res == ["rejected", "rejected"], res
