"""Every GPU step at the cluster cap (run with -m gpu on an H100): K from 192 to GMM_MAX_CLUSTERS = 512 against the exact
references of the per-kernel suites, and contexts sized for Kmax = 512 that run a smaller K.

K sits on the structural boundaries of the kernels: 192 and 256 / 257 (32-cluster column blocks and 64-cluster grid rows of
the tensor M-step, 256-centre tiles of the k-means assignment at D = 32), 449 (the 8th 64-cluster E-step pass with one
cluster), 511 / 512 (a partial last and a full last pass).  Each case asserts which kernel ran through the profile
counters.  A large-K0 gmm_fit walks down through every K in one context sized for K0, so the stale passes of the E-step
operand and the stale responsibility rows above K are checked against fresh contexts bit for bit."""
import numpy as np
import pytest

import _combine_ref as cr
import _condition_stats_ref as csr
import _vb_ref as vb
from conftest import RUN_MEMB, assert_params_close
from test_estep_error_model import Emulation, blobs, standardise
from test_gpu_condition import check_ref as check_condition, events as condition_events, model as spd_model
from test_gpu_combine import GAIN_RTOL, _check_against, _fixture, _memberships
from test_gpu_condition_stats import check_stats as check_condition_stats
from test_gpu_estep_tc import ALL_TRIPLES, LANDINGS, TILE, assert_ll_ulp, ring_depth
from test_gpu_finalize import _assert_same, _both, _one_step, _seed_params
from test_gpu_lse_edges import check_memberships, check_score_stats, check_scores, f64_reference, with_zero_pi
from test_gpu_mstep_tc import MSTEP_D, check_bar, dyadic_events, edge_n, estep_mstep, n_sms, reference
from test_gpu_sample import check_restatement
from test_gpu_score import mixture, new_batches, top_two_gap
from test_gpu_score_stats import finalise
from test_gpu_seed_kmeans import AMBIG, kmeanspp_ref
from test_gpu_vb import _prior_of as vb_prior_of, _ref_params as vb_ref_params, _start as vb_start
from test_gpu_simt import dyadic, dyadic_params, mstep_tier, resp_ratio
from test_mstep_error_model import cta_ranges, emulate as mstep_emulate, exact_mstep_stats, param_errors
from test_simt_error_model import blobs as simt_blobs, epack, logits, param_set as simt_param_set, simt_bar

pytestmark = pytest.mark.gpu

KMAX = 512
TENSOR_D = (8, 16, 24)


def engine(pkg, ev, Kmax, estep=None, mstep=None):
    eng = pkg.Engine(ev, Kmax)
    eng.set_option("estep_path", pkg.PATH_TENSOR if estep is None else estep)
    eng.set_option("mstep_path", pkg.PATH_TENSOR if mstep is None else mstep)
    return eng


_blobs = {}


def data(D):
    """The events of tests/test_estep_error_model.py at this D (N_DATA of them), made once per module."""
    if D not in _blobs:
        _blobs[D] = blobs(D)
    return _blobs[D]


# ---- 1. tensor E-step and gmm_score ----------------------------------------------------------------------------------------
def ring_n(sms, slot, wg, tiles=12, rem=37):
    """At least `tiles` 64-event tiles per CTA (every (slot, use parity, wait parity) of the ring), and a last partial
    tile (rem events) on the given slot and warpgroup."""
    nt = tiles * sms
    while True:
        n = TILE * (nt - 1) + rem
        if ring_depth(n, sms)["last"] == (slot, wg):
            return n
        nt += 1


def last_tiles(n, sms):
    """The events of the last tile of each warpgroup of every CTA: the deepest use of the slot ring."""
    rd = ring_depth(n, sms)
    g, nt = rd["grid"], rd["ntiles"]
    tiles = {list(range(2 * b + h, nt, 2 * g))[-1] for b in range(g) for h in range(2) if 2 * b + h < nt}
    return np.concatenate([np.arange(t * TILE, min(n, t * TILE + TILE)) for t in sorted(tiles)])


def emulate(held, K, x, shift, scale, memb=None, lp=None, labels=None, mr=None, chunk=1024):
    """Worst error / bar of the responsibilities and log-densities (E-step), or of gmm_score's outputs, over x."""
    w = [0.0, 0.0]
    for s in range(0, len(x), chunk):
        sel = slice(s, s + chunk)
        em = Emulation(held, K, x[sel], shift, scale)
        if labels is None:
            w[0] = max(w[0], em.ratio(memb[:, sel]))
            w[1] = max(w[1], em.lse_ratio(lp[sel]))
        else:
            r_mr, r_lp, bad = em.score_check(labels[sel], mr[sel], lp[sel])
            assert bad == 0, bad
            w = [max(w[0], r_mr), max(w[1], r_lp)]
    return w


ESTEP_K = (257, 449, 512)


@pytest.mark.parametrize("K", ESTEP_K)
@pytest.mark.parametrize("D", TENSOR_D)
def test_tensor_estep_at_the_cap(pkg, D, K):
    """12+ tiles per CTA, the last partial tile on each slot and warpgroup in turn: the responsibilities of the last tile of
    every warpgroup and of 2 048 random events, and every gmm_score output of new events, within the Emulation bars;
    max_resp the stored responsibility of the label bit for bit; the log-likelihood within 1 ulp of gmm_score's."""
    sms = n_sms()
    slot, wg = LANDINGS[(D + K) % len(LANDINGS)]
    n = ring_n(sms, slot, wg)
    rd = ring_depth(n, sms)
    assert rd["grid"] == sms and rd["min_tiles"] >= 10 and rd["triples"] == ALL_TRIPLES and rd["last"] == (slot, wg), rd
    ev_all = data(D)
    ev = np.ascontiguousarray(ev_all[:n])
    with engine(pkg, ev, K) as eng:
        eng.set_clusters(K, mixture(pkg, ev, K))
        ll = eng.estep(K)
        memb = eng.get_clusters(K, with_memberships=True).memberships[:K].copy()
        held = eng.get_clusters(K)
        eng.score_profile(reset=True)
        lab, mr, lp, _ = eng.score(K, ev)
        np.testing.assert_array_equal(mr, memb[lab, np.arange(n)])
        differ = top_two_gap(memb, 0) > 0
        np.testing.assert_array_equal(lab[differ], memb.argmax(0)[differ])
        rng = np.random.default_rng(D * 1000 + K)
        batches = {name: x[:2048] for name, x in new_batches(ev_all[:n + 20_000], n, rng).items()}
        scored = {name: eng.score(K, x)[:3] for name, x in batches.items()}
        assert eng.score_profile()["tensor_chunks"] > 0 and eng.score_profile()["simt_chunks"] == 0
        eng.score_stats_profile(reset=True)
        shift = eng.score_stats(K, ev[:1], stats=False, memberships=True)[1]
        prof = eng.score_stats_profile()
        assert prof["estep_tensor_chunks"] == 1 and prof["estep_simt_chunks"] == 0, prof
    assert_ll_ulp(ll, lp, "estep vs score")
    scale = standardise(ev)[1]
    idx = np.unique(np.r_[last_tiles(n, sms), rng.choice(n, 2048, replace=False)])
    worst = emulate(held, K, ev[idx], shift, scale, memb=memb[:, idx], lp=lp[idx])
    worst_new = [0.0, 0.0]
    for name, x in batches.items():
        l2, m2, p2 = scored[name]
        r = emulate(held, K, x, shift, scale, labels=l2, mr=m2, lp=p2)
        worst_new = [max(worst_new[0], r[0]), max(worst_new[1], r[1])]
    print(f"\n[cap estep-tc] D={D} K={K} n={n}, {len(idx)} events: responsibilities {worst[0]:.3g}, logp {worst[1]:.3g}; "
          f"new events max_resp {worst_new[0]:.3g}, logp {worst_new[1]:.3g} of the bar")
    assert max(worst + worst_new) <= 1.0, (worst, worst_new)


ZERO = {"pass8": (512, list(range(448, 512))), "lone448": (449, [448])}


@pytest.mark.parametrize("case", list(ZERO))
@pytest.mark.parametrize("D", TENSOR_D)
def test_tensor_zero_pi_last_pass(pkg, D, case):
    """pi = 0 on the whole 8th pass (no finite logit in it) or on its lone cluster: those responsibilities exactly 0, the
    others against the float64 log-sum-exp, gmm_score and gmm_score_stats as in tests/test_gpu_lse_edges.py."""
    K, zero = ZERO[case]
    ev = np.ascontiguousarray(data(D)[:20_011])
    with engine(pkg, ev, K, mstep=pkg.PATH_AUTO) as eng:
        eng.set_clusters(K, with_zero_pi(mixture(pkg, ev, K), zero))
        held = eng.get_clusters(K)
        ll = eng.estep(K)
        memb = eng.get_clusters(K, with_memberships=True).memberships[:K].copy()
        L, gamma, lse = f64_reference(held, K, ev)
        w = check_memberships(memb, L, gamma, lse, zero, f"D={D} {case}")
        assert np.isfinite(ll) and abs(ll - lse.sum()) <= 1e-5 * abs(lse.sum()), (ll, lse.sum())
        eng.score_profile(reset=True)
        check_scores(pkg, eng, K, ev, held, zero, memb, ll, f"D={D} {case}")
        assert eng.score_profile()["simt_chunks"] == 0
        eng.score_stats_profile(reset=True)
        check_score_stats(eng, K, ev, zero, memb, f"score_stats D={D} {case}")
        prof = eng.score_stats_profile()
        assert prof["estep_tensor_chunks"] > 0 and prof["estep_simt_chunks"] == 0, prof
    print(f"\n[cap pi=0] D={D} {case}: memberships worst/bar {w:.3g}")


# ---- 2. tensor M-step ------------------------------------------------------------------------------------------------------
MSTEP_K = (192, 257, 449, 512)


@pytest.mark.parametrize("K", MSTEP_K)
@pytest.mark.parametrize("D", MSTEP_D)
def test_tensor_mstep_at_the_cap(pkg, D, K):
    """Grid rows 3 .. 7 and column blocks up to 15: the per-cluster MSTEP_TOL bar against the exact M-step on the
    responsibilities the kernel read."""
    ev = pkg.synth.make_blobs(40_000, D, 16, seed=800 + D)
    with engine(pkg, ev, K, estep=pkg.PATH_SIMT) as eng:
        got, memb = estep_mstep(pkg, eng, K, mixture(pkg, ev, K))
        assert eng.profile()["mstep_tensor_launches"] == 1
    check_bar(pkg, ev, memb, got, K, f"D={D} K={K} N=40000")


@pytest.mark.parametrize("D", MSTEP_D)
def test_tensor_mstep_exact_at_the_cap(pkg, oracle64, D):
    """The dyadic data of test_mstep_tc_exact_on_dyadic_data with its four clusters in column blocks 0, 8, 14 and 15 (grid
    rows 0, 4 and 7) of K = 512; the others sit far from every event and take responsibility exactly 0.  Bit for bit."""
    K = KMAX
    sms = n_sms()
    ev, centres, scale = dyadic_events(D, 4, sms)
    N = len(ev)
    shift, sc, z, zb = standardise(ev)
    assert not shift.any() and np.array_equal(sc, scale) and zb == 2.0
    per, gx = cta_ranges(N, sms)
    assert per == 128
    live = [0, 8 * 32 + 31, 14 * 32, 15 * 32 + 31]
    assert [k // 32 for k in live] == [0, 8, 14, 15] and live[-1] // 64 == 7
    cl = pkg.Clusters(K, D)
    for k in range(K):
        cl.means[k] = 64.0 * (1.0 + k / K) * scale
    cl.means[live] = centres
    cl.R[:K] = np.diag((0.05 * scale) ** 2)
    cl.N[:K] = N / K
    oracle64.constants(cl, K)
    with engine(pkg, ev, K, estep=pkg.PATH_SIMT) as eng:
        got, memb = estep_mstep(pkg, eng, K, cl)
        assert eng.profile()["mstep_tensor_launches"] == 1
    assert np.isin(memb[:K], (0.0, 1.0)).all() and (memb[:K].sum(0) == 1.0).all()
    assert (memb[live].sum(1) > 0).all() and memb[:K].sum() == memb[live].sum()
    ref, _ = reference(pkg, ev, memb, got, K)
    for f in ("N", "means", "R"):
        np.testing.assert_array_equal(getattr(got, f)[:K], getattr(ref, f)[:K], err_msg=f)


@pytest.mark.parametrize("D", [12, 24])
def test_tensor_mstep_one_event_at_the_cap(pkg, D):
    """A shard of one event: one CTA, one live column of the 16 column blocks."""
    N = edge_n("1", n_sms())
    per, gx = cta_ranges(N, n_sms())
    big = pkg.synth.make_blobs(20_000, D, 16, seed=840 + D)
    ev = np.ascontiguousarray(big[:N])
    with engine(pkg, ev, KMAX, estep=pkg.PATH_SIMT) as eng:
        got, memb = estep_mstep(pkg, eng, KMAX, mixture(pkg, big, KMAX))
        assert eng.profile()["mstep_tensor_launches"] == 1
    check_bar(pkg, ev, memb, got, KMAX, f"D={D} K={KMAX} N={N} (1: per {per}, gx {gx})")


@pytest.mark.parametrize("D", [12, 24])
def test_tensor_mstep_full_plus_one_at_the_cap(pkg, D):
    """Full CTAs and a last CTA of one event (4 225 events on 132 SMs), K = 512: about 8 events per cluster.

    MSTEP_TOL does not hold for the kernel's arithmetic at this shape: the faithful emulation of the scheme
    (tests/test_mstep_error_model.py emulate) on the same responsibilities reaches 1.15 of the bar on N at D = 12 (a cluster
    of mass ~1 made mostly of events with small g, where the FP16 rounding of g_l dominates), see
    tests/test_cluster_cap_models.py.  So the kernel is held to that emulation (within a quarter of MSTEP_TOL: it
    differs only by the truncating accumulation of the remainder chains), and its error against the exact M-step to at
    most 1.25 times the emulation's."""
    sms = n_sms()
    N = edge_n("full+1", sms)
    per, gx = cta_ranges(N, sms)
    assert N - (gx - 1) * per == 1
    big = pkg.synth.make_blobs(20_000, D, 16, seed=840 + D)
    ev = np.ascontiguousarray(big[:N])
    with engine(pkg, ev, KMAX, estep=pkg.PATH_SIMT) as eng:
        got, memb = estep_mstep(pkg, eng, KMAX, mixture(pkg, big, KMAX))
        assert eng.profile()["mstep_tensor_launches"] == 1
    ref, shift = reference(pkg, ev, memb, got, KMAX)
    emu_stats = np.r_[mstep_emulate(ev, memb[:KMAX], n_sms=sms, variants=("faithful",))[0]["faithful"].ravel(), 0.0]
    emu = pkg.Clusters(KMAX, D)
    emu.avgvar[:KMAX] = got.avgvar[:KMAX]
    pkg.host_finalize(emu_stats, shift, emu, KMAX)
    K = KMAX
    e_gpu = param_errors(got.N[:K], got.means[:K], got.R[:K], ref.N[:K], ref.means[:K], ref.R[:K], shift)
    e_emu = param_errors(emu.N[:K], emu.means[:K], emu.R[:K], ref.N[:K], ref.means[:K], ref.R[:K], shift)
    e_same = param_errors(got.N[:K], got.means[:K], got.R[:K], emu.N[:K], emu.means[:K], emu.R[:K], shift)
    print(f"\n[cap mstep-tc] D={D} K={K} N={N} (full+1: per {per}, gx {gx}): kernel vs exact {e_gpu['worst']:.3f}, "
          f"emulated scheme vs exact {e_emu['worst']:.3f}, kernel vs emulated scheme {e_same['worst']:.3f} of MSTEP_TOL")
    assert e_same["worst"] <= 0.25, e_same
    assert e_gpu["worst"] <= max(1.0, 1.25 * e_emu["worst"]), (e_gpu, e_emu)


# ---- 3. Kmax = 512 at smaller K ------------------------------------------------------------------------------------------------
SMALLER_K = (449, 448, 385, 257, 256, 65)


def one_of_each(pkg, eng, K, cl, ev):
    """E-step memberships, M-step parameters, one device-finalised iteration and gmm_score, from cl (the E-step through
    gmm_score_stats asserted to be the tensor one)."""
    eng.set_clusters(K, cl)
    eng.score_stats_profile(reset=True)
    eng.score_stats(K, ev[:64], stats=False, memberships=True)
    p = eng.score_stats_profile()
    assert p["estep_tensor_chunks"] == 1 and p["estep_simt_chunks"] == 0, p
    eng.estep(K)
    memb = eng.get_clusters(K, with_memberships=True).memberships[:K].copy()
    eng.mstep(K)
    after_m = eng.get_clusters(K)
    eng.set_clusters(K, cl)
    eng.estep(K)
    ll = eng.em_iterations(K, 1)
    after_em = eng.get_clusters(K, with_memberships=True)
    return memb, after_m, ll, after_em, eng.score(K, ev)


@pytest.mark.parametrize("D", [16, 24])
def test_kmax_512_runs_smaller_k(pkg, D):
    """After a K = 512 iteration, each smaller K equals a fresh Kmax = K context bit for bit."""
    ev = pkg.synth.make_blobs(20_000, D, 16, seed=860 + D)
    with engine(pkg, ev, KMAX) as eng:
        eng.set_option("finalize", 1)
        one_of_each(pkg, eng, KMAX, mixture(pkg, ev, KMAX), ev)
        big = {K: one_of_each(pkg, eng, K, mixture(pkg, ev, K, seed=K), ev) for K in SMALLER_K}
        fp = eng.fit_profile()
        assert eng.profile()["mstep_tensor_launches"] == 2 * (1 + len(SMALLER_K))
        assert fp["device_finalize_launches"] == 1 + len(SMALLER_K) and fp["host_replays"] == 0, fp
    for K in SMALLER_K:
        with engine(pkg, ev, K) as eng:
            eng.set_option("finalize", 1)
            fresh = one_of_each(pkg, eng, K, mixture(pkg, ev, K, seed=K), ev)
        got = big[K]
        np.testing.assert_array_equal(got[0], fresh[0], err_msg=f"K={K} E-step")
        _assert_same(got[1], fresh[1], K, f"K={K} M-step")
        assert got[2] == fresh[2], (K, got[2], fresh[2])
        _assert_same(got[3], fresh[3], K, f"K={K} finalised iteration")
        for a, b, what in zip(got[4][:3], fresh[4][:3], ("labels", "max_resp", "logp")):
            np.testing.assert_array_equal(a, b, err_msg=f"K={K} score {what}")


# ---- 4. device finalisation against the host ----------------------------------------------------------------------------------
@pytest.mark.parametrize("D,K", [(16, 512), (24, 449), (24, 512)])
def test_finalisation_bit_identical_at_the_cap(pkg, D, K):
    """One step, em_iterations(K, 3) and gmm_em(K, 2, 3) with the device finalisation equal the host finalisation's."""
    N = 8 * K
    ev = pkg.synth.make_blobs(N, D, 12, seed=880 + D + K)
    P0 = _seed_params(pkg, ev, K)
    (((dev, ll_d), fp_d), ((host, ll_h), fp_h)) = _both(pkg, ev, K, _one_step(P0, K))
    assert fp_d["device_finalize_launches"] == 1 and fp_d["host_replays"] == 0 and fp_h["device_finalize_launches"] == 0
    _assert_same(dev, host, K, f"D={D} K={K} one step")
    assert ll_d == ll_h

    def drivers(eng):
        eng.seed(K)
        eng.estep(K)
        ll1 = eng.em_iterations(K, 3)
        a = eng.get_clusters(K, with_memberships=True)
        ll2, it = eng.em(K, 2, 3)
        return a, ll1, eng.get_clusters(K, with_memberships=True), ll2, it

    ((d, fp_d), (h, fp_h)) = _both(pkg, ev, K, drivers)
    assert fp_d["device_finalize_launches"] >= 5 and fp_d["host_replays"] == 0 and fp_h["device_finalize_launches"] == 0
    _assert_same(d[0], h[0], K, "em_iterations")
    _assert_same(d[2], h[2], K, "gmm_em")
    assert d[1] == h[1] and d[3] == h[3] and d[4] == h[4]


def test_replay_at_the_cap(pkg):
    """A forced replay (finalize_fault_iter = 1) in a 3-iteration batch at K = 512 equals the all-host run bit for bit."""
    D, K = 24, KMAX
    ev = pkg.synth.make_blobs(8 * K, D, 12, seed=890)

    def run(eng, fault):
        eng.seed(K)
        eng.estep(K)
        if fault:
            eng.set_option("finalize_fault_iter", 1)
        ll = eng.em_iterations(K, 3)
        return eng.get_clusters(K, with_memberships=True), ll

    with pkg.Engine(ev, K) as eng:
        eng.set_option("finalize", 1)
        rep, ll_r = run(eng, True)
        fp = eng.fit_profile()
    with pkg.Engine(ev, K) as eng:
        eng.set_option("finalize", 0)
        host, ll_h = run(eng, False)
        assert eng.fit_profile()["device_finalize_launches"] == 0
    print(f"\n[cap replay] fit_profile {fp}")
    assert fp["host_replays"] == 1 and fp["device_finalize_launches"] >= 2, fp
    _assert_same(rep, host, K)
    assert ll_r == ll_h


# ---- 5. SIMT E- and M-step ------------------------------------------------------------------------------------------------------
SIMT_D = (5, 13, 21, 28)              # one D per JMAX tier of mstep_simt_kernel (3, 10, 21, 36)


@pytest.mark.parametrize("K", [257, 512])
@pytest.mark.parametrize("D", SIMT_D)
def test_simt_estep_at_the_cap(pkg, oracle64, D, K):
    n = 4_097
    ev = simt_blobs(n, D, K)
    cl = simt_param_set(pkg, oracle64, "fitted", D, K, ev)
    with engine(pkg, ev, K, estep=pkg.PATH_SIMT, mstep=pkg.PATH_SIMT) as eng:
        eng.set_clusters(K, cl)
        eng.estep(K)
        memb = eng.get_clusters(K, with_memberships=True).memberships[:K].copy()
        eng.score_profile(reset=True)
        lab, mr, lp, _ = eng.score(K, ev)
        sp = eng.score_profile()
        assert sp["tensor_chunks"] == 0 and sp["simt_chunks"] > 0, sp
    l = logits(ev, epack(cl, K))
    gamma, lse, gbar, lbar = simt_bar(l)
    worst = resp_ratio(memb, gamma, gbar)
    lw = float((np.abs(lp.astype(np.float64) - lse) / lbar).max())
    print(f"\n[cap simt-estep] D={D} K={K} n={n}: resp {worst:.3f}  logp {lw:.3f} of the bar")
    assert worst <= 1.0 and lw <= 1.0, (worst, lw)
    np.testing.assert_array_equal(lab, l.argmax(1))
    np.testing.assert_array_equal(mr, memb[lab, np.arange(n)])


@pytest.mark.parametrize("K", [257, 512])
@pytest.mark.parametrize("D", SIMT_D)
def test_simt_mstep_exact_at_the_cap(pkg, oracle64, D, K):
    ev, cen, _ = dyadic(D, K, 8)
    n = len(ev)
    tier = mstep_tier(D, K, n, n_sms())
    cl = dyadic_params(pkg, oracle64, cen, n)
    with engine(pkg, ev, K, estep=pkg.PATH_SIMT, mstep=pkg.PATH_SIMT) as eng:
        eng.set_clusters(K, cl)
        eng.estep(K)
        memb = eng.get_clusters(K, with_memberships=True).memberships[:K].copy()
        eng.mstep(K)
        assert eng.profile()["mstep_simt_launches"] == 1
        got = eng.get_clusters(K)
    assert np.isin(memb, (0.0, 1.0)).all() and (memb.sum(0) == 1.0).all()
    sh = np.zeros(D)
    ref = exact_mstep_stats(ev, memb, sh)
    fin = pkg.Clusters(K, D)
    fin.avgvar[:K] = got.avgvar[:K]
    pkg.host_finalize(ref, sh, fin, K)
    for f in ("N", "means", "R"):
        np.testing.assert_array_equal(getattr(got, f)[:K], getattr(fin, f)[:K], err_msg=f)
    print(f"\n[cap simt-mstep] dyadic D={D} K={K} n={n} (JMAX, CPT, KT, rows, per, gx) = {tier}: bit-exact")


# ---- 6. chunked calls -----------------------------------------------------------------------------------------------------------
def test_score_stats_shard_at_the_cap(pkg):
    """gmm_score_stats on the training shard: the resident E-step's memberships bit for bit, and the statistics finalise
    to the resident tensor M-step's parameters bit for bit (D = 24, K = 512)."""
    D, K = 24, KMAX
    ev = pkg.synth.make_blobs(20_011, D, 16, seed=900)
    with engine(pkg, ev, K) as eng:
        eng.set_clusters(K, mixture(pkg, ev, K))
        ll = eng.estep(K)
        eng.score_stats_profile(reset=True)
        st, sh, mb = eng.score_stats(K, ev, memberships=True)
        prof = eng.score_stats_profile()
        assert (prof["estep_tensor_chunks"], prof["estep_simt_chunks"], prof["mstep_tensor_chunks"], prof["mstep_simt_chunks"]) \
            == (1, 0, 1, 0), prof
        before = eng.get_clusters(K, with_memberships=True)
        np.testing.assert_array_equal(mb, before.memberships[:K])
        assert abs(st[-1] - ll) <= 1e-6 * abs(ll), (st[-1], ll)
        eng.mstep(K)
        eng.constants(K)
        res = eng.get_clusters(K)
    got = finalise(pkg, st, sh, K, D, before.avgvar)
    for f in ("N", "pi", "constant", "means", "R", "Rinv"):
        np.testing.assert_array_equal(getattr(got, f)[:K], getattr(res, f)[:K], err_msg=f)


@pytest.mark.parametrize("D", [24, 32])
def test_condition_at_the_cap(pkg, D):
    """gmm_condition and gmm_condition_stats on half of the dimensions against their restatements, K = 512."""
    K = KMAX
    cl = spd_model(pkg, K, D, seed=910 + D)
    obs = np.arange(0, D, 2)
    ev = condition_events(cl, K, 6_000, seed=D, far=0.0)
    with pkg.Engine(ev, K) as eng:
        eng.set_clusters(K, cl)
        x = condition_events(cl, K, 3_000, seed=D + 1)
        eng.condition_profile(reset=True)
        out = eng.condition(K, obs, np.ascontiguousarray(x[:, obs]), mean=True, var=True)
        assert eng.condition_profile()["kernel_ms"] > 0
        check_condition(cl, K, obs, np.ascontiguousarray(x[:, obs]), out, f"condition D={D} K={K}")
        xo = np.ascontiguousarray(ev[:, obs])
        eng.condition_stats_profile(reset=True)
        st, sh, mb = eng.condition_stats(K, obs, xo, memberships=True)
        p = eng.condition_stats_profile()
        assert p["mstep_tensor_chunks"] + p["mstep_simt_chunks"] == 1, p
        check_condition_stats(st, cl, K, obs, xo, mb, sh, p["mstep_tensor_chunks"] == 0, f"condition_stats D={D} K={K}")
        post, lp = csr.marginal_posterior(cl, K, obs, xo)
        np.testing.assert_allclose(mb, post, **RUN_MEMB)


@pytest.mark.parametrize("D,K", [(24, 512), (32, 300), (32, 512)])
def test_sample_at_the_cap(pkg, D, K):
    cl = spd_model(pkg, K, D, seed=920 + D + K)
    cl.pi[1] = 0.0
    n, seed = 5_003, 0x9E3779B97F4A7C15 ^ (D * K)
    with pkg.Engine(pkg.synth.make_blobs(4096, D, 4, seed=5), K) as eng:
        eng.set_clusters(K, cl)
        for first in (0, (1 << 32) + 5):
            eng.sample_profile(reset=True)
            x, lab = eng.sample(K, n, seed=seed, first=first)
            assert eng.sample_profile()["kernel_ms"] > 0
            check_restatement(cl, K, seed, first, x, lab, f"D={D} K={K} first={first}")
            assert not np.any(lab == 1) and lab.min() >= 0 and lab.max() < K


# ---- 7. gmm_combine -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [257, 512])
@pytest.mark.parametrize("D", [8, 24])
def test_combine_at_the_cap(pkg, D, K):
    """Merges, gains, entropy and masses against tests/_combine_ref.py (pair pass with 9 and 16 tiles per side, step pass
    with hundreds of live groups); labels at three levels of the kernel's hierarchy bit for bit.

    Over 511 steps some step's two largest gains lie within 10x the gain bar of each other at every fixture seed (relative
    gaps down to 1.7e-6 against GAIN_RTOL = 2e-6), and past such a near tie either merge is legal.  At K = 512 the merges,
    gains and masses are compared up to the first near tie (the whole hierarchy when there is none), the entropy of the
    K-cluster level and the labels in full."""
    n = 8 * K + 2000
    for attempt in range(3 if K < 512 else 1):
        ev, cl = _fixture(pkg, D, K, n, 1000 * attempt + 10 * D + K)
        with pkg.Engine(ev, K) as eng:
            eng.set_clusters(K, cl)
            eng.estep(K)
            tau = _memberships(eng, K)
            ref = cr.combine(tau)
            near = np.nonzero(ref["gap"] < 10 * GAIN_RTOL)[0]
            if K < 512 and near.size:
                continue
            eng.combine_profile(reset=True)
            got = eng.combine(K)
            assert eng.combine_profile()["kernel_ms"] > 0
            steps = int(near[0]) if near.size else None
            print(f"\n[cap combine] D={D} K={K} n={len(ev)}: {len(near)} near-tied steps, compared "
                  f"{K - 1 if steps is None else steps} of {K - 1} steps")
            assert steps is None or steps >= 64, steps
            _check_against(got, ref, K, len(ev), nsteps=steps)
            for L in (1, K // 2 + 1, K - 1):
                grp = pkg.host_combine_groups(got["merges"], K, L)
                lab, mx = eng.combine_labels(K, grp)
                rl, rm = cr.labels(tau, grp, L)
                np.testing.assert_array_equal(lab, rl, err_msg=f"L={L}")
                np.testing.assert_array_equal(mx.view(np.int32), rm.view(np.int32), err_msg=f"L={L}")
        return
    pytest.fail("no fixture seed gave every step a top-two gap of 10x the gain bar")


# ---- 8. gmm_seed_kmeans with several centre tiles ----------------------------------------------------------------------------
def nearest_chunked(x, centres, chunk=512):
    """float64 labels and the number of events whose two nearest centres are within FP32 rounding of each other."""
    c64 = centres.astype(np.float64)
    lab, amb = np.empty(len(x), np.int64), 0
    for s in range(0, len(x), chunk):
        d = ((x[s:s + chunk, None, :].astype(np.float64) - c64[None]) ** 2).sum(-1)
        lab[s:s + chunk] = d.argmin(1)
        two = np.partition(d, 1, axis=1)[:, :2]
        amb += int(((two[:, 1] - two[:, 0]) <= AMBIG * np.maximum(two[:, 1], 1e-30)).sum())
    return lab, amb


@pytest.mark.parametrize("D,K", [(32, 257), (32, 512), (24, 342), (24, 512)])
def test_seed_kmeans_several_centre_tiles(pkg, D, K):
    """k-means++ bit for bit against kmeanspp_ref (L = 8 candidates at K >= 404); the counts of the one-hot M-step are
    those of the float64 nearest centre (TILE = 8192 / D centres per tile of kmeans_assign_kernel: 2 tiles at (32, 257)
    and (24, 342), where centre 341 is alone in the second one, 3 and 2 at K = 512); one Lloyd step moves the centres to
    the float64 centroids of those labels."""
    tile = 8192 // D
    assert K > tile
    if (D, K) == (24, 342):
        assert K - tile == 1                                    # one centre alone in the second tile
    assert (2 + int(np.floor(np.log(K))) == 8) == (K >= 404)
    x = pkg.synth.make_blobs(8_011, D, 12, seed=930 + D)
    seed = 1000 * D + K
    for _ in range(8):                                          # the first seed whose choices and labels are unambiguous
        idx, amb = kmeanspp_ref(x, K, seed)
        amb_lab = nearest_chunked(x, x[idx])[1]
        if not amb and amb_lab == 0:
            break
        seed += 1
    assert not amb and amb_lab == 0, "no unambiguous seed in 8: pick other data"
    with pkg.Engine(x, K) as eng:
        eng.profile(reset=True)
        cl, cent, it, _ = eng.seed_kmeans(K, max_iter=0, seed=seed)
        p = eng.profile()
        assert (p["mstep_tensor_launches"], p["mstep_simt_launches"]) == ((1, 0) if D <= 24 else (0, 1)), p
        cl1, cent1, it1, _ = eng.seed_kmeans(K, max_iter=1, seed=seed)
    np.testing.assert_array_equal(cent, x[idx])
    lab, _ = nearest_chunked(x, cent)
    np.testing.assert_array_equal(cl.N[:K], np.bincount(lab, minlength=K).astype(np.float32))
    assert lab.max() >= tile                                    # some event's nearest centre is in a later tile
    assert it1 == 1                                             # k-means++ centres are events: the first assignment moves them
    want = cent.astype(np.float64).copy()
    for k in np.unique(lab):
        want[k] = x[lab == k].astype(np.float64).mean(0)
    scale = np.abs(x).max()
    assert float((np.abs(cent1 - want) / (np.abs(want) + scale)).max()) <= 1e-5


def test_seed_kmeans_tie_across_tiles(pkg):
    """3 distinct rows, K = 400, D = 32: centres 3 .. 399 repeat centre 0 (include/gmm.h), so every copy of that row ties
    with centres in the second 256-centre tile.  The lowest k wins: label 0, and clusters 3 .. 399 stay empty."""
    D, K = 32, 400
    rows = np.random.default_rng(16).standard_normal((3, D)).astype(np.float32)
    x = rows[np.random.default_rng(17).integers(0, 3, 3000)]
    with pkg.Engine(x, K) as eng:
        eng.profile(reset=True)
        cl, cent, _, _ = eng.seed_kmeans(K, max_iter=0, seed=2)
        assert eng.profile()["mstep_simt_launches"] == 1
    idx, _ = kmeanspp_ref(x, K, 2)
    np.testing.assert_array_equal(cent, x[idx])
    assert len({tuple(r) for r in cent[:3]}) == 3
    np.testing.assert_array_equal(cent[3:], np.repeat(cent[:1], K - 3, 0))
    counts = [int((x == cent[k]).all(1).sum()) for k in range(3)]
    np.testing.assert_array_equal(cl.N[:3], np.array(counts, np.float32))
    assert np.all(cl.N[3:K] == 0.0)


# ---- 9. drivers ---------------------------------------------------------------------------------------------------------------
def test_fit_across_the_last_pass(pkg, oracle64):
    """gmm_fit from K0 = 452 to 446 (across 449 -> 448, where the 8th E-step pass goes), 3 iterations per order, D = 24,
    against the CPU oracle at the run-level bars."""
    N, D, K0, Kt = 3_000, 24, 452, 446
    ev = pkg.synth.make_blobs(N, D, 16, seed=940)
    with pkg.Engine(ev, K0) as eng:
        eng.set_option("path", pkg.PATH_TENSOR)
        eng.profile(reset=True)
        ideal, mr, got = eng.fit(K0, Kt, 3, 3, with_memberships=True)
        assert eng.profile()["mstep_tensor_launches"] > 0 and eng.profile()["mstep_simt_launches"] == 0
    ref = pkg.Clusters(K0, D, N)
    ideal_ref, mr_ref = oracle64.fit(ev, K0, Kt, 3, 3, pkg.Clusters(K0, D, N), ref)
    assert ideal == ideal_ref == Kt
    assert abs(mr - mr_ref) <= 1e-4 * abs(mr_ref), (mr, mr_ref)
    # about 7 events per cluster: a cluster of one event has R = avgvar I in exact arithmetic, where S2 / N - mu mu^T
    # cancels to 0; the tensor M-step leaves its error relative to the raw second moment about the centre there (the unit
    # of MSTEP_TOL), which the run-level bar, scaled to the cluster's own R, cannot absorb.  N and the means of every
    # cluster are compared, R, Rinv and the constant of the clusters of mass 1.5 or more
    np.testing.assert_allclose(got.N[:ideal], ref.N[:ideal], rtol=5e-4, atol=1e-3)
    mscale = max(1.0, float(np.abs(ref.means[:ideal]).max()))
    np.testing.assert_allclose(got.means[:ideal], ref.means[:ideal], rtol=5e-4, atol=5e-4 * mscale)
    live = np.nonzero(ref.N[:ideal] >= 1.5)[0]
    assert len(live) >= ideal // 2, len(live)
    sub = [pkg.Clusters(len(live), D) for _ in range(2)]
    for a, b in zip(sub, (got, ref)):
        for f in ("N", "pi", "constant", "means", "R", "Rinv", "avgvar"):
            getattr(a, f)[...] = getattr(b, f)[live]
    print(f"\n[cap fit] {len(live)} of {ideal} clusters with N >= 1.5")
    assert_params_close(sub[0], sub[1], len(live), rtol=5e-4)
    np.testing.assert_allclose(got.memberships[:ideal], ref.memberships[:ideal], **RUN_MEMB)


def test_vb_one_step_at_the_cap(pkg):
    """gmm_vb_em with max_iters = 0 at D = 24, K = 512: posterior 0 from the engine's responsibilities against
    tests/_vb_ref.py at the per-operator bar."""
    D, K, N = 24, KMAX, 6_000
    ev = pkg.synth.make_blobs(N, D, 12, seed=950)
    with pkg.Engine(ev, K) as eng:
        g0 = vb_start(eng, K)
        cl, post, lb, _, it, conv = eng.vb_em(K, 0, 0, prior_type=vb.DP)
        assert it == 0 and not conv and lb == -np.inf
        p = vb.m_step(vb.stats_from_resp(ev, g0, np.zeros(D)), np.zeros(D), K, D, vb_prior_of(post, K, D, vb.DP))
        assert_params_close(cl, vb_ref_params(pkg, p, K, D), K)
        np.testing.assert_allclose(post["weights"], p["weights"], rtol=1e-4, atol=1e-7)
        np.testing.assert_allclose(post["dof"], p["nu"], rtol=1e-4)
        got = eng.get_clusters(K, with_memberships=True).memberships[:K].T
        lr, _ = vb.e_step(ev, p)
        np.testing.assert_allclose(got, np.exp(lr), **RUN_MEMB)
