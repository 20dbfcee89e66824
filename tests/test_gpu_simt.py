"""The SIMT E-step, scoring and M-step kernels (`estep_simt_kernel<D, WT>`, `score_simt_kernel<D>`,
`mstep_simt_kernel<JMAX, CPT, WT>`, csrc/kernels_simt.cuh) against exact references (run with -m gpu on an H100).

E-step: every responsibility, log-density and log-likelihood is held to the bar of tests/test_simt_error_model.py, which
restates the kernel's logits bit for bit and bounds what follows them (expf, logf, the FP32 sums).  The cases cover all 32
compiled D, K on both sides of the 16-cluster staging chunk up to GMM_MAX_CLUSTERS, event counts with a partial last
128-event block, and the two GMM_PATH_AUTO fallbacks from the tensor E-step.  The scoring kernel's max_resp must be the
E-step's stored responsibility bit for bit, at every D.

M-step: on dyadic data (integer coordinates, mirrored events so that the centre is exactly 0, responsibilities exactly 0
or 1) every statistic is an integer below 2^53, so the statistics must equal the integer reference bit for bit, and
gmm_mstep's parameters must equal the host finalisation of them.  On realistic data every packed statistic is held to
    |S_gpu - S_ref| <= (gamma_m + gamma_r) sum_n |g_n phi_f(x_n - s)|,   gamma_j = j 2^-53 / (1 - j 2^-53),
m = per + gx + 4 (the kernel's fma chain over a block's events, the atomics of the gx blocks, the roundings of x - s and of
the product), r = ceil(log2 n) + 20 (the reference's elementwise terms and numpy's pairwise sum, whose blocks of 128 are
summed by 8 sequential accumulators).  The cases cover all 11 (JMAX, CPT) instances, weighted and not, and the shard
edges of the launch.  Every case asserts which kernels ran."""
import math

import numpy as np
import pytest

from test_mstep_error_model import cta_ranges, exact_mstep_stats
from test_simt_error_model import blobs, epack, estep_cases, logits, param_set, simt_bar

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
INSTANCES = {(3, 1), (3, 2), (3, 4), (10, 1), (10, 2), (10, 4), (21, 1), (21, 2), (21, 4), (36, 1), (36, 2)}


def n_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def gam(j):
    return j * 2.0 ** -53 / (1 - j * 2.0 ** -53)


def mstep_tier(D, K, n, sms):
    """launch_mstep_simt_on / launch_mstep_simt_t: (JMAX, CPT, KT, grid rows, per, gx)."""
    F = 1 + D + D * (D + 1) // 2
    cpt = 1 if K <= 16 else (2 if K <= 32 else 4)
    jmax = 3 if F <= 48 else 10 if F <= 160 else 21 if F <= 336 else 36
    if jmax == 36:
        cpt = min(cpt, 2)
    per, gx = cta_ranges(n, sms)
    return jmax, cpt, 16 * cpt, -(-K // (16 * cpt)), per, gx


def engine(pkg, ev, K, estep=None, mstep=None):
    eng = pkg.Engine(ev, K)
    eng.set_option("estep_path", pkg.PATH_SIMT if estep is None else estep)
    eng.set_option("mstep_path", pkg.PATH_SIMT if mstep is None else mstep)
    return eng


def chunks(p):
    return p["estep_tensor_chunks"], p["estep_simt_chunks"], p["mstep_tensor_chunks"], p["mstep_simt_chunks"]


# ---- E-step ---------------------------------------------------------------------------------------------------------------
def resp_ratio(memb, gamma, gbar):
    """Worst |gamma_gpu - gamma| / bar; memb is [K][n]."""
    return float((np.abs(np.asarray(memb, np.float64).T - gamma) / gbar).max())


def ll_bound(lse, lbar, n, w=None):
    """Bound on the double log-likelihood slot: the per-event bars plus the double sum (warp shuffles, 4 warps, one atomic
    per 128-event block)."""
    w = np.ones_like(lse) if w is None else np.asarray(w, np.float64)
    return float((w * lbar).sum() + gam(9 + -(-n // 128)) * (w * (np.abs(lse) + lbar)).sum())


ESTEP = estep_cases()


def test_estep_cases_cover_every_instance():
    assert {D for _, D, _, _ in ESTEP} == set(range(1, 33))
    assert {K for _, _, K, _ in ESTEP} == {1, 15, 16, 17, 33, 130, 512}


@pytest.mark.parametrize("kind,D,K,n", ESTEP)
def test_estep_every_responsibility(pkg, oracle64, kind, D, K, n):
    """Resident E-step, gmm_score_stats on the shard and on 1, 127 and 129 events, gmm_score: responsibilities, log-densities
    and the log-likelihood to the bar; max_resp and labels against the E-step and the emulated logits, bit for bit."""
    ev = blobs(n, D, K)
    cl = param_set(pkg, oracle64, kind, D, K, ev)
    with engine(pkg, ev, K) as eng:
        eng.set_clusters(K, cl)
        eng.estep(K)
        memb = eng.get_clusters(K, with_memberships=True).memberships[:K].copy()
        eng.score_stats_profile(reset=True)
        st, _, mb = eng.score_stats(K, ev, memberships=True)
        assert chunks(eng.score_stats_profile()) == (0, 1, 0, 1)
        small = {m: eng.score_stats(K, ev[:m], stats=False, memberships=True)[2] for m in (1, 127, 129)}
        eng.score_profile(reset=True)
        lab, mr, lp, _ = eng.score(K, ev)
        sp = eng.score_profile()
        assert sp["tensor_chunks"] == 0 and sp["simt_chunks"] > 0, sp
    np.testing.assert_array_equal(mb, memb)
    l = logits(ev, epack(cl, K))
    gamma, lse, gbar, lbar = simt_bar(l)
    worst = resp_ratio(memb, gamma, gbar)
    for m, g in small.items():
        worst = max(worst, resp_ratio(g, gamma[:m], gbar[:m]))
    if K == 1:
        assert (memb == 1.0).all()
    lw = float((np.abs(lp.astype(np.float64) - lse) / lbar).max())
    dll = abs(st[-1] - lse.sum()) / ll_bound(lse, lbar, n)
    print(f"\n[simt-estep] {kind} D={D} K={K} n={n}: resp {worst:.3f}  logp {lw:.3f}  loglik {dll:.3f} of the bar")
    assert worst <= 1.0 and lw <= 1.0 and dll <= 1.0, (worst, lw, dll)
    # score_simt_kernel: the arg-max of the logits (lowest k on ties) and the E-step's stored responsibility there
    np.testing.assert_array_equal(lab, l.argmax(1))
    np.testing.assert_array_equal(mr, memb[lab, np.arange(n)])


def check_against_forced_simt(pkg, ev, cl, K, x, resident, what):
    """GMM_PATH_AUTO's E-step on the events x through gmm_score_stats (and, with resident, on the shard) against the forced
    SIMT E-step, bit for bit, and the bar."""
    out = {}
    for name, path in (("auto", pkg.PATH_AUTO), ("simt", pkg.PATH_SIMT)):
        with engine(pkg, ev, K, estep=path) as eng:
            eng.set_clusters(K, cl)
            if resident:
                eng.estep(K)
                out[name + "_res"] = eng.get_clusters(K, with_memberships=True).memberships[:K].copy()
            eng.score_stats_profile(reset=True)
            out[name] = eng.score_stats(K, x, stats=False, memberships=True)[2]
            assert chunks(eng.score_stats_profile())[:2] == (0, 1)
    np.testing.assert_array_equal(out["auto"], out["simt"])
    gamma, _, gbar, _ = simt_bar(logits(x, epack(cl, K)))
    r = resp_ratio(out["auto"], gamma, gbar)
    if resident:
        np.testing.assert_array_equal(out["auto_res"], out["simt_res"])
        r = max(r, resp_ratio(out["auto_res"], gamma, gbar))
    print(f"\n[simt-estep] {what}: resp {r:.3f} of the bar")
    assert r <= 1.0


def test_fallback_event_beyond_fp16(pkg, oracle64):
    """D = 24: an event 2^15 training standard deviations out puts gmm_score_stats' chunk on the SIMT E-step under
    GMM_PATH_AUTO.  (A resident shard cannot hold one: no event of n lies more than sqrt(n - 1) standard deviations of the
    shard from its mean, so the resident range test trips only past 2^28 events.)"""
    D, K, n = 24, 17, 4_097
    ev = blobs(n, D, K)
    cl = param_set(pkg, oracle64, "fitted", D, K, ev)
    x = ev[:1000].copy()
    e64 = ev.astype(np.float64)
    x[500, 3] = np.float32(e64[:, 3].mean() + 2.0 ** 15 * e64[:, 3].std())
    check_against_forced_simt(pkg, ev, cl, K, x, False, "D=24 K=17, one event 2^15 sigma out (AUTO)")


def test_fallback_not_positive_definite(pkg, oracle64):
    """D = 16: one cluster with an indefinite R and its LU inverse (not symmetric) puts the parameter set on the SIMT E-step
    under GMM_PATH_AUTO; the kernel's combined coefficients Rinv_ij + Rinv_ji matter here."""
    D, K, n = 16, 17, 4_097
    ev = blobs(n, D, K)
    cl = param_set(pkg, oracle64, "fitted", D, K, ev)
    rng = np.random.default_rng(16)
    Q = np.linalg.qr(rng.standard_normal((D, D)))[0]
    lam = np.r_[-0.3, rng.uniform(0.5, 2.0, D - 1)]
    R = (Q * lam) @ Q.T + 0.05 * np.triu(rng.standard_normal((D, D)), 1)
    cl.R[5] = R.astype(np.float32)
    cl.Rinv[5] = pkg.host_invert(cl.R[5])[0]
    Ri = cl.Rinv[5].astype(np.float64)
    assert np.abs(Ri - Ri.T).max() > 1e-3 and np.linalg.eigvalsh(0.5 * (Ri + Ri.T)).min() < 0
    check_against_forced_simt(pkg, ev, cl, K, ev, True, "D=16 K=17, one indefinite cluster (AUTO)")


WEIGHTED_D = (5, 13, 21, 28)          # one D per JMAX tier


@pytest.mark.parametrize("K", [16, 17, 33])
@pytest.mark.parametrize("D", WEIGHTED_D)
def test_weighted_estep(pkg, oracle64, D, K):
    """estep_simt_kernel<D, true>: the responsibilities of the unweighted run bit for bit; the log-likelihood is
    sum w denom within the bar (and the float of gmm_estep)."""
    n = 4_097
    ev = blobs(n, D, K)
    cl = param_set(pkg, oracle64, "fitted", D, K, ev)
    w = np.random.default_rng(D + K).uniform(0.0, 3.0, n).astype(np.float32)
    with engine(pkg, ev, K) as eng:
        eng.set_clusters(K, cl)
        eng.estep(K)
        plain = eng.get_clusters(K, with_memberships=True).memberships[:K].copy()
        eng.set_weights(w)
        ll = eng.estep(K)
        weighted = eng.get_clusters(K, with_memberships=True).memberships[:K]
    np.testing.assert_array_equal(weighted, plain)
    _, lse, _, lbar = simt_bar(logits(ev, epack(cl, K)))
    ref = float((w.astype(np.float64) * lse).sum())
    bound = ll_bound(lse, lbar, n, w) + U * (abs(ref) + ll_bound(lse, lbar, n, w))
    print(f"\n[simt-estep] weighted D={D} K={K}: loglik {abs(ll - ref) / bound:.3f} of the bar")
    assert abs(ll - ref) <= bound


# ---- M-step: bit for bit on dyadic data -------------------------------------------------------------------------------------
def dyadic(D, K, m, w=False):
    """Events on which the FP64 SIMT M-step is exact: cluster centres (2k - K + 1) * 10 * (1, .., 1), events the centre plus
    integer offsets in [-2, 2], cluster K - 1 - k the mirror image of cluster k (the middle cluster of an odd K mirrors
    itself), so every column sum and the centre are exactly 0.  Neighbouring centres are 20 sqrt(D) apart under R = I: every
    other logit lies at least 160 below the event's own, so expf gives 0 and the responsibilities are exactly 0 or 1.
    Returns (events [K m][D], centres, weights: integers 1..4, mirrored, or None)."""
    rng = np.random.default_rng(D * 1000 + K)
    cen = ((2 * np.arange(K) - K + 1) * 10.0)[:, None] * np.ones(D)
    off = np.empty((K, m, D))
    wt = np.empty((K, m))
    for k in range(K // 2):
        off[k] = rng.integers(-2, 3, (m, D))
        off[K - 1 - k] = -off[k]
        wt[k] = wt[K - 1 - k] = rng.integers(1, 5, m)
    if K % 2:
        h = rng.integers(-2, 3, (m // 2, D))
        off[K // 2] = np.concatenate([h, -h])
        hw = rng.integers(1, 5, m // 2)
        wt[K // 2] = np.concatenate([hw, hw])
    ev = (cen[:, None, :] + off).reshape(-1, D).astype(np.float32)
    return ev, cen, (wt.reshape(-1).astype(np.float32) if w else None)


def dyadic_params(pkg, oracle64, cen, n):
    K, D = cen.shape
    cl = pkg.Clusters(K, D)
    cl.means[:K] = cen
    cl.R[:K] = np.eye(D, dtype=np.float32)
    cl.N[:K] = n / K
    oracle64.constants(cl, K)
    return cl


DYADIC_K = (1, 16, 17, 32, 33, 64, 65, 130)
DYADIC = [(D, K) for D in range(1, 33) for K in DYADIC_K]
WEIGHTED_M = [(D, K) for D in WEIGHTED_D for K in (16, 17, 33)]


def test_mstep_cases_cover_every_instance():
    assert {mstep_tier(D, K, 1, 132)[:2] for D, K in DYADIC} == INSTANCES
    assert {mstep_tier(D, K, 1, 132)[:2] for D, K in WEIGHTED_M} == INSTANCES
    assert {mstep_tier(D, K, 1, 132)[:2] for D, K in REALISTIC} == INSTANCES


def finalise_ref(pkg, stats, shift, got, K, D):
    ref = pkg.Clusters(K, D)
    ref.avgvar[:K] = got.avgvar[:K]
    pkg.host_finalize(stats, shift, ref, K)
    return ref


@pytest.mark.parametrize("D,K", DYADIC)
def test_mstep_exact_on_dyadic_data(pkg, oracle64, D, K):
    ev, cen, _ = dyadic(D, K, 64 if K == 1 else 8)
    n = len(ev)
    tier = mstep_tier(D, K, n, n_sms())
    cl = dyadic_params(pkg, oracle64, cen, n)
    with engine(pkg, ev, K) as eng:
        eng.set_clusters(K, cl)
        eng.estep(K)
        memb = eng.get_clusters(K, with_memberships=True).memberships[:K].copy()
        eng.score_stats_profile(reset=True)
        st, sh, mb = eng.score_stats(K, ev, memberships=True)
        assert chunks(eng.score_stats_profile()) == (0, 1, 0, 1)
        eng.mstep(K)
        assert eng.profile()["mstep_simt_launches"] == 1
        got = eng.get_clusters(K)
    assert np.isin(memb, (0.0, 1.0)).all() and (memb.sum(0) == 1.0).all()
    assert not sh.any()
    np.testing.assert_array_equal(mb, memb)
    ref = exact_mstep_stats(ev, memb, sh)
    np.testing.assert_array_equal(st[:-1], ref[:-1])
    fin = finalise_ref(pkg, ref, sh, got, K, D)
    for f in ("N", "means", "R"):
        np.testing.assert_array_equal(getattr(got, f)[:K], getattr(fin, f)[:K], err_msg=f)
    print(f"\n[simt-mstep] dyadic D={D} K={K} n={n} (JMAX, CPT, KT, rows, per, gx) = {tier}: bit-exact")


@pytest.mark.parametrize("D,K", WEIGHTED_M)
def test_weighted_mstep_exact_on_dyadic_data(pkg, oracle64, D, K):
    """mstep_simt_kernel<JMAX, CPT, true> with integer weights 1..4: gmm_mstep's parameters equal the host finalisation
    of the exact weighted statistics bit for bit."""
    ev, cen, w = dyadic(D, K, 8, w=True)
    n = len(ev)
    tier = mstep_tier(D, K, n, n_sms())
    cl = dyadic_params(pkg, oracle64, cen, n)
    with engine(pkg, ev, K) as eng:
        eng.set_weights(w)
        eng.set_clusters(K, cl)
        eng.estep(K)
        memb = eng.get_clusters(K, with_memberships=True).memberships[:K].copy()
        eng.mstep(K)
        assert eng.profile()["mstep_simt_launches"] == 1
        got = eng.get_clusters(K)
    assert np.isin(memb, (0.0, 1.0)).all()
    ref = exact_mstep_stats(ev, memb * w[None], np.zeros(D))
    fin = finalise_ref(pkg, ref, np.zeros(D), got, K, D)
    for f in ("N", "means", "R"):
        np.testing.assert_array_equal(getattr(got, f)[:K], getattr(fin, f)[:K], err_msg=f)
    print(f"\n[simt-mstep] weighted dyadic D={D} K={K} {tier}: bit-exact")


# ---- M-step: the rigorous bar on realistic data -----------------------------------------------------------------------------
def stats_ratio(st, x, g, shift, per, gx):
    """Worst |S_gpu - S_ref| / ((gamma_m + gamma_r) sum |g phi|) over the packed statistics, one cluster at a time."""
    n, D = x.shape
    y = np.asarray(x, np.float32).astype(np.float64) - np.asarray(shift, np.float64)
    i, j = np.tril_indices(D)
    phi = np.ascontiguousarray(np.concatenate([np.ones((1, n)), y.T, (y[:, i] * y[:, j]).T]))       # [F][n]
    F = phi.shape[0]
    aphi = np.abs(phi)
    g64 = np.asarray(g, np.float64)
    tol = gam(per + gx + 4) + gam(math.ceil(math.log2(max(n, 2))) + 20)
    worst = 0.0
    for k in range(g64.shape[0]):
        ref = (phi * g64[k]).sum(axis=1)
        bound = tol * (aphi @ np.abs(g64[k])) * (1 + 1e-12)
        d = np.abs(st[k * F:(k + 1) * F] - ref)
        worst = max(worst, float(np.max(np.where(bound > 0, d / np.where(bound > 0, bound, 1.0), np.where(d > 0, np.inf, 0.0)))))
    return worst


REALISTIC = [(D, K) for D in (8, 9, 16, 17, 24, 25, 32) for K in (16, 17, 32, 33, 64, 65)]


def edge_ns(sms):
    """Shard edges of launch_mstep_simt_t (cta_ranges): tiny shards, a partial first tile, fewer blocks than SMs (each of
    one 32-event tile), full blocks then a last block of one event."""
    return {"1": 1, "31": 31, "32": 32, "33": 33, "gx<sms": 32 * (sms - 4) - 1, "full+1": 64 * (sms // 2) + 1}


@pytest.mark.parametrize("D,K", REALISTIC)
def test_mstep_bar_on_realistic_data(pkg, oracle64, D, K):
    sms = n_sms()
    n = 6_007
    ev = blobs(n, D, K)
    cl = param_set(pkg, oracle64, "fitted", D, K, ev)
    edges = edge_ns(sms)
    per, gx = cta_ranges(edges["gx<sms"], sms)
    assert per == 32 and gx < sms
    per, gx = cta_ranges(edges["full+1"], sms)
    assert edges["full+1"] - (gx - 1) * per == 1
    runs = [("shard", n)] + ([(k, v) for k, v in edges.items()] if D in (9, 17, 25, 32) else [])
    worst = 0.0
    with engine(pkg, ev, K) as eng:
        eng.set_clusters(K, cl)
        for name, m in runs:
            x = np.ascontiguousarray(ev[:m])
            eng.score_stats_profile(reset=True)
            st, sh, mb = eng.score_stats(K, x, memberships=True)
            assert chunks(eng.score_stats_profile()) == (0, 1, 0, 1)
            jmax, cpt, kt, rows, per, gx = mstep_tier(D, K, m, sms)
            r = stats_ratio(st, x, mb, sh, per, gx)
            print(f"\n[simt-mstep] D={D} K={K} {name} n={m} (JMAX {jmax}, CPT {cpt}, KT {kt}, rows {rows}, per {per}, gx {gx}): "
                  f"{r:.3g} of the bar")
            worst = max(worst, r)
    assert worst <= 1.0, worst
