"""The log-sum-exp epilogues where they branch (run with -m gpu on an H100): the fused D = 8 tensor E-step against the
exact emulation, score_tc_kernel's running state across the K > 64 passes (exact ties, the pass offset of the label, the
two max_resp branches), and mixtures with components at pi = 0.

pi = 0 is a valid parameter (gmm_set_clusters accepts it, gmm_sample never draws such a component): its logit constant
constant + ln pi is -inf.  The reference (estep2) takes the maximum over all clusters first, so such a component gets a
responsibility of exactly 0 and every event a finite density.  The kernels keep a running or per-pass maximum instead; it
starts at -FLT_MAX so that a -inf logit ahead of every finite one, or a whole pass of them, adds exp(-inf) = 0 rather
than exp(-inf - -inf) = NaN.  Every case here compares with a float64 log-sum-exp over the same parameter set."""
import numpy as np
import pytest
from scipy.special import logsumexp

from test_estep_error_model import KINDS, N_DATA, Emulation, blobs, param_set, standardise
from test_gpu_condition import check_ref as check_condition
from test_gpu_estep_tc import LANDINGS, check_deep, deep_n, emulated_events, assert_ll_ulp
from conftest import fitted_params
from test_gpu_mstep_tc import n_sms
from test_gpu_score_stats import TENSOR_M_D
from test_mstep_error_model import exact_mstep_stats, mstep_errors
from test_gpu_score import check_f64, new_batches, ref_logits, top_two_gap

pytestmark = pytest.mark.gpu

TENSOR_D = (8, 16, 24)
SIMT_D = (5, 24, 32)


# ---- helpers -----------------------------------------------------------------------------------------------------------
def engine(pkg, ev, K, path):
    eng = pkg.Engine(ev, K)
    eng.set_option("estep_path", path)
    eng.set_option("mstep_path", pkg.PATH_AUTO)           # the wgmma M-step at the D it covers (TENSOR_M_D), else FP64
    return eng


def events(pkg, n, D, seed=11):
    return pkg.synth.make_blobs(n, D, 6, seed=seed)


_fitted = {}


def fitted(pkg, oracle, ev, K):
    """The CPU oracle's seeding and 2 EM iterations on the first 20 000 events (cached per shape)."""
    key = (ev.shape[1], K, float(ev[0, 0]))
    if key not in _fitted:
        _fitted[key] = fitted_params(pkg, oracle, np.ascontiguousarray(ev[:20_000]), K)
    cl = _fitted[key]
    out = pkg.Clusters(K, ev.shape[1])
    for f in ("means", "R", "Rinv", "constant", "pi", "N", "avgvar"):
        getattr(out, f)[...] = getattr(cl, f)[:K]
    return out


def with_zero_pi(cl, zero):
    """The parameter set with pi = 0 on the components `zero` (the others keep theirs: sum pi < 1 is allowed)."""
    cl.pi[list(zero)] = 0.0
    return cl


def f64_reference(cl, K, x):
    """float64 logits [n][K], responsibilities [K][n] and log-densities [n]."""
    L = ref_logits(cl, K, x)
    lse = logsumexp(L, axis=1)
    return L, np.exp(L - lse[:, None]).T, lse


def check_memberships(memb, L, gamma, lse, zero, what):
    """Zero-weight rows exactly 0, every value finite, the others within 1e-6 + (1e-4 + 2e-6 (|l_k| + |lse|)) gamma of
    the float64 responsibilities (the parity bar of 1e-4 / 1e-6, widened by the float32 rounding of large logits)."""
    assert np.all(np.isfinite(memb)), (what, int((~np.isfinite(memb)).sum()))
    if len(zero):
        assert np.all(memb[list(zero)] == 0.0), what
    mag = np.where(np.isfinite(L), np.abs(L), 0.0).T + np.abs(lse)[None, :]
    d = np.abs(memb.astype(np.float64) - gamma) / (1e-6 + (1e-4 + 2e-6 * mag) * gamma)
    assert d.max() <= 1.0, (what, float(d.max()))
    return float(d.max())


def check_score_stats(eng, K, ev, zero, memb, what):
    """gmm_score_stats: memberships bit-identical to the E-step's, the statistics of zero-weight components exactly 0 and
    the others against the exact float64 M-step on those memberships (test_gpu_score_stats' bars: 1e-10 for the FP64
    M-step, MSTEP_TOL for the wgmma one)."""
    st, sh, mb = eng.score_stats(K, ev, stats=True, memberships=True)
    np.testing.assert_array_equal(mb, memb, err_msg=what)
    D = ev.shape[1]
    F = 1 + D + D * (D + 1) // 2
    rows, ref = st[:K * F].reshape(K, F), exact_mstep_stats(ev, mb, sh)[:K * F].reshape(K, F)
    assert np.all(np.isfinite(st)) and np.all(rows[list(zero)] == 0.0), what
    keep = np.setdiff1d(np.arange(K), zero)
    e = mstep_errors(np.r_[rows[keep].ravel(), st[-1]], np.r_[ref[keep].ravel(), 0.0], sh, len(keep))
    if D in TENSOR_M_D:
        assert e["worst"] <= 1.0, (what, e)
    else:
        assert max(e["N"], e["mean"], e["R"]) <= 1e-10, (what, e)


def check_scores(pkg, eng, K, ev, cl, zero, memb, ll, what):
    """gmm_score on the training shard and on new events: finite, never a zero-weight label, within check_f64's bars;
    on the shard max_resp is the stored responsibility of the label, bit for bit."""
    lab, mr, lp, sll = eng.score(K, ev)
    assert np.all(np.isfinite(lp)) and np.all(np.isfinite(mr)), what
    assert not np.isin(lab, list(zero)).any(), what
    check_f64(cl, K, ev, lab, mr, lp, what + " shard")
    top = memb[lab, np.arange(len(ev))]
    np.testing.assert_array_equal(mr, top, err_msg=what)
    assert abs(sll - ll) <= 1e-5 * abs(ll), (what, sll, ll)
    rng = np.random.default_rng(len(ev))
    ev_all = np.concatenate([ev, events(pkg, 4000, ev.shape[1], seed=99)])
    for name, x in new_batches(ev_all, len(ev), rng).items():
        lab, mr, lp, _ = eng.score(K, x)
        assert not np.isin(lab, list(zero)).any(), (what, name)
        check_f64(cl, K, x, lab, mr, lp, f"{what} {name}")


# ---- 1. pi = 0: tensor E-step and gmm_score ----------------------------------------------------------------------------------
# Padding clusters past K (to a multiple of 16) carry the finite constant -1e30 (tc_params_begin), so a pass has no finite
# logit only when it is 16 n clusters that all have pi = 0.
TENSOR_ZERO = {
    "first": (17, [0]),                                   # K <= 64, ahead of every finite logit
    "pass0": (70, [0, 5, 63]),                            # in pass 0 of two
    "last": (129, [128]),                                 # alone in the last pass, beside 15 padding clusters (S > 0)
    "k64": (65, [64]),                                    # idem, two passes
    "whole-last16": (80, list(range(64, 80))),            # the last pass (mode 2) has no finite logit: S = 0, scale 0
    "whole-last64": (128, list(range(64, 128))),          # idem, a full last pass of 4 supergroups
    "whole-pass0": (129, list(range(64))),                # pass 0 has no finite logit (modes 1, 3)
    "whole-pass1": (130, list(range(64, 128))),           # a middle pass has none (the join of mode 1)
}


@pytest.mark.parametrize("case", list(TENSOR_ZERO))
@pytest.mark.parametrize("D", TENSOR_D)
def test_zero_pi_tensor(pkg, oracle64, D, case):
    K, zero = TENSOR_ZERO[case]
    ev = events(pkg, 20_011, D)
    cl = with_zero_pi(fitted(pkg, oracle64, ev, K), zero)
    with engine(pkg, ev, K, pkg.PATH_TENSOR) as eng:
        eng.set_clusters(K, cl)
        held = eng.get_clusters(K)
        ll = eng.estep(K)
        memb = eng.get_clusters(K, with_memberships=True).memberships[:K].copy()
        L, gamma, lse = f64_reference(held, K, ev)
        w = check_memberships(memb, L, gamma, lse, zero, f"tensor D={D} {case}")
        assert np.isfinite(ll) and abs(ll - lse.sum()) <= 1e-5 * abs(lse.sum()), (ll, lse.sum())
        check_scores(pkg, eng, K, ev, held, zero, memb, ll, f"tensor D={D} {case}")
        # gmm_score_stats runs the same E-step per chunk
        check_score_stats(eng, K, ev, zero, memb, f"score_stats tensor D={D} {case}")
        prof = eng.score_stats_profile()
        assert prof["estep_tensor_chunks"] > 0 and prof["estep_simt_chunks"] == 0, prof
    print(f"\n[pi=0 tensor] D={D} {case}: memberships worst/bar {w:.3g}")


# ---- 2. pi = 0: SIMT E-step, gmm_score and gmm_condition ------------------------------------------------------------------
SIMT_ZERO = {
    "first": (7, [0]),
    "last": (7, [6]),
    "chunk1": (40, list(range(16, 32))),                  # a whole 16-cluster chunk
    "chunk0": (40, list(range(16))),                      # the first chunk: run_max stays at its start for 16 clusters
}


@pytest.mark.parametrize("case", list(SIMT_ZERO))
@pytest.mark.parametrize("D", SIMT_D)
def test_zero_pi_simt(pkg, oracle64, D, case):
    K, zero = SIMT_ZERO[case]
    ev = events(pkg, 20_011, D)
    cl = with_zero_pi(fitted(pkg, oracle64, ev, K), zero)
    with engine(pkg, ev, K, pkg.PATH_SIMT) as eng:
        eng.set_clusters(K, cl)
        held = eng.get_clusters(K)
        ll = eng.estep(K)
        memb = eng.get_clusters(K, with_memberships=True).memberships[:K].copy()
        L, gamma, lse = f64_reference(held, K, ev)
        w = check_memberships(memb, L, gamma, lse, zero, f"simt D={D} {case}")
        assert np.isfinite(ll) and abs(ll - lse.sum()) <= 1e-5 * abs(lse.sum()), (ll, lse.sum())
        check_scores(pkg, eng, K, ev, held, zero, memb, ll, f"simt D={D} {case}")
        eng.score_stats_profile(reset=True)
        check_score_stats(eng, K, ev, zero, memb, f"score_stats simt D={D} {case}")
        assert eng.score_stats_profile()["estep_simt_chunks"] > 0
        # gmm_condition on half of the dimensions: the marginal mixture has the same zero weights
        obs = np.arange(0, D, 2)
        x = ev[:5000]
        out = eng.condition(K, obs, x[:, obs], mean=D > 1, var=D > 1)
        for a in out[:5]:
            assert a is None or np.all(np.isfinite(a)), case
        assert not np.isin(out[0], zero).any()
        check_condition(held, K, obs, x[:, obs], out, f"condition D={D} {case}")
        # gmm_condition_stats: the marginal posteriors of the zero-weight components are 0
        st, _, mb = eng.condition_stats(K, obs, x[:, obs], stats=True, memberships=True)
        assert np.all(np.isfinite(st)) and np.all(np.isfinite(mb)) and np.all(mb[zero] == 0.0), case
    print(f"\n[pi=0 simt] D={D} {case}: memberships worst/bar {w:.3g}")


# ---- 3. pi = 0 through EM, gmm_combine and weights ---------------------------------------------------------------------------
@pytest.mark.parametrize("path,D,K,zero", [("tensor", 24, 65, [64]), ("tensor", 16, 17, [0]), ("simt", 5, 20, list(range(16)))])
def test_zero_pi_em_step_and_combine(pkg, oracle64, path, D, K, zero):
    ev = events(pkg, 20_011, D)
    cl = with_zero_pi(fitted(pkg, oracle64, ev, K), zero)
    ref = pkg.Clusters(K, D, len(ev))
    with engine(pkg, ev, K, pkg.PATH_TENSOR if path == "tensor" else pkg.PATH_SIMT) as eng:
        eng.seed(K)                                       # the global moments the M-step shifts by
        eng.set_clusters(K, cl)
        held = eng.get_clusters(K, out=ref)
        ll = eng.estep(K)
        got = eng.get_clusters(K, with_memberships=True)
        assert np.all(got.memberships[zero] == 0.0)
        comb = eng.combine(K)
        assert np.all(np.isfinite(comb["gain"])) and np.all(np.isfinite(comb["entropy"])) and np.all(np.isfinite(comb["mass"])), comb
        ll1 = eng.em_iterations(K, 1)
        after = eng.get_clusters(K, with_memberships=True)
    ll_ref = oracle64.estep(oracle64.transpose(ev), held, K)
    assert abs(ll - ll_ref) <= 1e-5 * abs(ll_ref), (ll, ll_ref)
    np.testing.assert_allclose(got.memberships[:K], held.memberships[:K], rtol=1e-4, atol=1e-5)
    # the M-step sees N_k = 0 and the reference's N < 0.5 rule sets pi = 1e-10: the next E-step stays finite
    assert np.isfinite(ll1)
    assert np.all(np.isfinite(after.pi[:K])) and np.all(np.isfinite(after.constant[:K]))
    assert np.all(np.isfinite(after.memberships[:K]))
    assert np.all(after.pi[zero] > 0) and np.all(after.pi[zero] < 1e-6), after.pi[zero]


@pytest.mark.parametrize("path,D,K,zero", [("tensor", 24, 129, list(range(64))), ("simt", 24, 7, [0])])
def test_zero_pi_weighted(pkg, oracle64, path, D, K, zero):
    ev = events(pkg, 20_011, D)
    cl = with_zero_pi(fitted(pkg, oracle64, ev, K), zero)
    rng = np.random.default_rng(3)
    w = rng.uniform(0.0, 3.0, len(ev)).astype(np.float32)
    with engine(pkg, ev, K, pkg.PATH_TENSOR if path == "tensor" else pkg.PATH_SIMT) as eng:
        eng.set_clusters(K, cl)
        held = eng.get_clusters(K)
        eng.estep(K)
        memb = eng.get_clusters(K, with_memberships=True).memberships[:K].copy()
        eng.set_weights(w)
        llw = eng.estep(K)
        membw = eng.get_clusters(K, with_memberships=True).memberships[:K]
    np.testing.assert_array_equal(membw, memb)
    lse = f64_reference(held, K, ev)[2]
    ref = float(np.dot(w.astype(np.float64), lse))
    assert np.isfinite(llw) and abs(llw - ref) <= 1e-5 * abs(ref), (llw, ref)


# ---- 4. score_tc_kernel exactly, at every K ---------------------------------------------------------------------------------
SCORE_K = (7, 64, 65, 129, 209)


@pytest.mark.parametrize("K", SCORE_K)
@pytest.mark.parametrize("D", TENSOR_D)
def test_score_tc_exact(pkg, oracle64, D, K):
    """max_resp is the stored responsibility of the label bit for bit on the training shard at every K (the E-step's mode
    0, 2 or 3 operations); logp, max_resp and the labels of new events, up to 2^13 standard deviations out, within the
    bars of the exact emulation (Emulation.score_check: max_resp against the emulated responsibility of the label, logp
    against the emulated log-sum-exp, the label wherever the emulated top-two gap clears both logits' bars), and within
    the float64 bars."""
    n_train = 20_000
    ev_all = events(pkg, n_train + 10_000, D, seed=21)
    ev = np.ascontiguousarray(ev_all[:n_train])
    cl = fitted(pkg, oracle64, ev, K)
    with engine(pkg, ev, K, pkg.PATH_TENSOR) as eng:
        eng.set_clusters(K, cl)
        held = eng.get_clusters(K)
        ll = eng.estep(K)
        memb = eng.get_clusters(K, with_memberships=True).memberships[:K].copy()
        eng.score_profile(reset=True)
        lab, mr, lp, sll = eng.score(K, ev)
        np.testing.assert_array_equal(mr, memb[lab, np.arange(n_train)])
        differ = top_two_gap(memb, 0) > 0
        np.testing.assert_array_equal(lab[differ], memb.argmax(0)[differ])
        rng = np.random.default_rng(K)
        batches = new_batches(ev_all, n_train, rng)
        mu, sd = ev.mean(0), ev.std(0)
        dirs = rng.standard_normal((2000, D))
        dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
        batches["very far"] = (mu + dirs * sd * 2.0 ** rng.uniform(6, 13, (2000, 1))).astype(np.float32)
        shift = eng.score_stats(K, ev[:1], stats=False, memberships=True)[1]
        scale = standardise(ev)[1]
        for name, x in batches.items():
            lab, mr, lp, _ = eng.score(K, x)
            if name == "very far":                        # logits of -1e8: the float64 bars scale with |l|
                L = ref_logits(held, K, x)
                rl = logsumexp(L, axis=1)
                assert np.all(np.abs(lp - rl) <= 1e-5 * np.abs(rl)), name
                sure = top_two_gap(L, 1) > 1e-5 * np.abs(L.max(1))
                np.testing.assert_array_equal(lab[sure], L.argmax(1)[sure])
            else:
                check_f64(held, K, x, lab, mr, lp, f"D={D} K={K} {name}")
            worst = (0.0, 0.0)
            for s in range(0, len(x), 4096):
                sel = slice(s, s + 4096)
                r_mr, r_lp, bad = Emulation(held, K, x[sel], shift, scale).score_check(lab[sel], mr[sel], lp[sel])
                assert bad == 0, (name, bad)
                worst = (max(worst[0], r_mr), max(worst[1], r_lp))
            print(f"\n[score-tc emulation] D={D} K={K} {name}: max_resp worst/bar {worst[0]:.3g}, logp worst/bar {worst[1]:.3g}")
            assert worst[0] <= 1.0 and worst[1] <= 1.0, (name, worst)
        assert eng.score_profile()["simt_chunks"] == 0


# ---- 5. exact ties ----------------------------------------------------------------------------------------------------------
def duplicate(cl, dst, src):
    for f in ("means", "R", "Rinv", "constant", "pi", "N", "avgvar"):
        getattr(cl, f)[dst] = getattr(cl, f)[src]


@pytest.mark.parametrize("D", TENSOR_D)
def test_ties_across_passes(pkg, oracle64, D):
    """Cluster k + 64 a copy of cluster k (same position in its pass): identical rows, and the label is never k + 64:
    an earlier pass wins ties."""
    K = 129
    ev = events(pkg, 20_011, D)
    cl = fitted(pkg, oracle64, ev, K)
    for k in range(64):
        duplicate(cl, k + 64, k)
    with engine(pkg, ev, K, pkg.PATH_TENSOR) as eng:
        eng.set_clusters(K, cl)
        eng.estep(K)
        memb = eng.get_clusters(K, with_memberships=True).memberships[:K]
        np.testing.assert_array_equal(memb[64:128], memb[:64])
        lab, mr, _, _ = eng.score(K, ev)
        assert not ((lab >= 64) & (lab < 128)).any()
        np.testing.assert_array_equal(mr, memb[lab, np.arange(len(ev))])
        # where the top of pass 0 is the overall top and unique within the pass, the label is pass 0's arg-max
        tied = (memb[:64].max(0) == memb.max(0)) & (top_two_gap(memb[:64], 0) > 0)
        assert tied.mean() > 0.5
        np.testing.assert_array_equal(lab[tied], memb[:64].argmax(0)[tied])


WITHIN = [(1, 0), (2, 0), (8, 3), (4, 1), (20, 3), (40, 7), (63, 2)]   # (copy, source): quad lanes, chunks, supergroups


@pytest.mark.parametrize("path,D", [("tensor", D) for D in TENSOR_D] + [("simt", D) for D in SIMT_D])
def test_ties_within_a_pass(pkg, oracle64, path, D):
    """Copies of a cluster in other quad lanes, 4-cluster chunks and supergroups of one pass: the lowest k wins wherever
    the copies' stored responsibilities are equal."""
    K = 64
    ev = events(pkg, 20_011, D)
    cl = fitted(pkg, oracle64, ev, K)
    for dst, src in WITHIN:
        duplicate(cl, dst, src)
    with engine(pkg, ev, K, pkg.PATH_TENSOR if path == "tensor" else pkg.PATH_SIMT) as eng:
        eng.set_clusters(K, cl)
        eng.estep(K)
        memb = eng.get_clusters(K, with_memberships=True).memberships[:K]
        lab, mr, _, _ = eng.score(K, ev)
    np.testing.assert_array_equal(mr, memb[lab, np.arange(len(ev))])
    equal_rows = 0
    for dst, src in WITHIN:
        same = memb[dst] == memb[src]
        equal_rows += int(same.all())
        assert not (same & (lab == dst)).any(), (dst, src)
    # a unique top responsibility is the label (the kernels' arg-max is over the logits, which equal stored values may hide)
    differ = top_two_gap(memb, 0) > 0
    np.testing.assert_array_equal(lab[differ], memb.argmax(0)[differ])
    print(f"\n[ties] {path} D={D}: {equal_rows} of {len(WITHIN)} copies give bit-identical rows")


# ---- 6. the fused D = 8 E-step against the exact emulation ----------------------------------------------------------------------
D8_SHAPES = [(kind, K) for kind in KINDS for K in (1, 16, 17, 33, 49, 64, 65, 129, 209)
             if not (kind == "needle" and K == 1)]         # (the needle set places its special clusters at 0, 1 and K - 1)


@pytest.mark.parametrize("kind,K", D8_SHAPES)
def test_d8_deep_against_emulation(pkg, oracle64, kind, K):
    D = 8
    sms = n_sms()
    slot, wg = LANDINGS[(KINDS.index(kind) + K) % len(LANDINGS)]
    n = deep_n(sms, slot, wg)
    check_deep(n, sms, slot, wg)
    ev_all = blobs(D)
    assert n <= N_DATA
    ev = np.ascontiguousarray(ev_all[:n])
    cl = param_set(pkg, oracle64, kind, D, K, ev_all)
    with engine(pkg, ev, K, pkg.PATH_TENSOR) as eng:
        eng.set_clusters(K, cl)
        ll = eng.estep(K)
        memb = eng.get_clusters(K, with_memberships=True).memberships[:K].copy()
        held = eng.get_clusters(K)
        eng.score_profile(reset=True)
        lp = eng.score(K, ev)[2]
        assert eng.score_profile()["tensor_chunks"] > 0 and eng.score_profile()["simt_chunks"] == 0
        eng.score_stats_profile(reset=True)
        shift = eng.score_stats(K, ev[:1], stats=False, memberships=True)[1]
        prof = eng.score_stats_profile()
        assert prof["estep_tensor_chunks"] == 1 and prof["estep_simt_chunks"] == 0, prof
    assert_ll_ulp(ll, lp, "estep vs score")
    scale = standardise(ev)[1]
    idx = emulated_events(n, sms, np.random.default_rng(D + K))
    worst = worst_lp = 0.0
    for s in range(0, len(idx), 4096):
        sel = idx[s:s + 4096]
        em = Emulation(held, K, ev[sel], shift, scale)
        worst = max(worst, em.ratio(memb[:, sel]))
        worst_lp = max(worst_lp, em.lse_ratio(lp[sel]))
    print(f"\n[estep-tc emulation] {kind} D=8 K={K} n={n}, {len(idx)} events: responsibilities worst/bar {worst:.3g}, "
          f"logp worst/bar {worst_lp:.3g}")
    assert worst <= 1.0 and worst_lp <= 1.0, (worst, worst_lp)
