"""The device-side M-step finalisation (finalize_params_kernel, option "finalize" = 1) against the host finalisation
(option "finalize" = 0), bit for bit.

DESIGN §5.4: the kernel evaluates the host's operations in the host's order, so N, pi, constant, means, R, Rinv and the
resident E-step operand it writes are the host's to the last bit.  EM amplifies a last-bit difference by about 3x per
iteration, so these tests compare with assert_array_equal / ==, never with a tolerance: two contexts run the same calls
from identical inputs, one per finalisation, and must agree exactly, one step at a time, at every branch of the
kernel, over whole drivers, and when a cluster sends the device path back to the host (the host replay).  One test
anchors the step to an independent float64 reference (the only tolerances of this file, each with its reason).
Every case asserts which path ran (fit_profile: device_finalize_launches, host_replays).
"""
import numpy as np
import pytest

from conftest import random_spd_params

pytestmark = pytest.mark.gpu

FIELDS = ("N", "pi", "constant", "means", "R", "Rinv")
LN2PI = float(np.log(2.0 * np.pi))


@pytest.fixture(scope="module")
def loaded(pkg):
    pkg.load_library()
    return pkg


def _assert_same(a, b, K, what=""):
    """Bit equality of two parameter sets (and their memberships, when both carry them)."""
    for f in FIELDS:
        np.testing.assert_array_equal(getattr(a, f)[:K], getattr(b, f)[:K], err_msg=f"{what} {f}")
    if a.memberships is not None and b.memberships is not None and a.memberships.size and b.memberships.size:
        np.testing.assert_array_equal(a.memberships[:K], b.memberships[:K], err_msg=f"{what} memberships")


def _consistent(cl, K):
    """Rinv and constant of cl made consistent with its R (float64), as a user of gmm_set_clusters supplies them."""
    D = cl.R.shape[1]
    for k in range(K):
        R = cl.R[k].astype(np.float64)
        cl.Rinv[k] = np.linalg.inv(R).astype(np.float32)
        cl.constant[k] = np.float32(-0.5 * D * LN2PI - 0.5 * np.linalg.slogdet(R)[1])
    return cl


def _both(pkg, ev, Kmax, body, Kmax_host=None):
    """body(eng) in a context with the device finalisation and in one with the host finalisation, from identical inputs.
    Returns ((result, fit_profile) device, (result, fit_profile) host)."""
    out = []
    for fin, km in ((1, Kmax), (0, Kmax_host or Kmax)):
        with pkg.Engine(ev, km) as eng:
            eng.set_option("finalize", fin)
            r = body(eng)
            out.append((r, eng.fit_profile()))
    return out


def _one_step(P0, K):
    def body(eng):
        eng.set_clusters(K, P0)
        eng.estep(K)
        ll = eng.em_iterations(K, 1)
        return eng.get_clusters(K, with_memberships=True), ll
    return body


def _seed_params(pkg, ev, K):
    with pkg.Engine(ev, K) as eng:
        return eng.seed(K)


# ---- 1. one finalisation, bit for bit -------------------------------------------------------------------------------
@pytest.mark.parametrize("D,K", [(D, K) for D in (8, 16, 24) for K in (1, 15, 16, 17, 63, 64, 65, 130)] + [(8, 512)])
def test_one_finalisation_bit_identical(loaded, D, K):
    """set_clusters(P0), estep, em_iterations(K, 1): the parameter set and the responsibilities of the E-step after the
    step (the operand image the kernel wrote, padding clusters of K % 16 != 0 and of a second 64-cluster pass included)
    equal the host finalisation's."""
    pkg = loaded
    N = max(6_000, 8 * K)
    ev = pkg.synth.make_blobs(N, D, max(2, min(K, 12)), seed=300 + D + K)
    P0 = _seed_params(pkg, ev, K)
    (((dev, ll_d), fp_d), ((host, ll_h), fp_h)) = _both(pkg, ev, K, _one_step(P0, K))
    assert fp_d["device_finalize_launches"] == 1 and fp_d["host_replays"] == 0
    assert fp_h["device_finalize_launches"] == 0 and fp_h["host_replays"] == 0
    _assert_same(dev, host, K, f"D={D} K={K}")
    assert ll_d == ll_h


def test_one_finalisation_kmax_above_k(loaded):
    """A context sized for Kmax = 200 running K = 65 (parameter-set stride Kmax, operand passes for K only) equals a
    Kmax = K context with the host finalisation."""
    pkg = loaded
    D, K, N = 16, 65, 8_000
    ev = pkg.synth.make_blobs(N, D, 10, seed=311)
    P0 = _seed_params(pkg, ev, K)
    (((dev, ll_d), fp_d), ((host, ll_h), fp_h)) = _both(pkg, ev, 200, _one_step(P0, K), Kmax_host=K)
    assert fp_d["device_finalize_launches"] == 1 and fp_d["host_replays"] == 0 and fp_h["device_finalize_launches"] == 0
    _assert_same(dev, host, K)
    assert ll_d == ll_h


# ---- 2. the step against an independent float64 reference ---------------------------------------------------------
@pytest.mark.parametrize("D,K", [(8, 17), (16, 65), (24, 64)])
def test_one_finalisation_against_float64(loaded, oracle64, D, K):
    """The device-finalised set from the statistics gmm_score_stats returns for the training shard in one chunk (the
    wgmma M-step's own statistics, gmm.h), against plain float64 numpy."""
    pkg = loaded
    N = 12_000
    ev = pkg.synth.make_blobs(N, D, 8, seed=320 + D)
    P0 = _seed_params(pkg, ev, K)
    with pkg.Engine(ev, K) as eng:
        eng.set_option("finalize", 1)
        eng.set_option("score_chunk", N)
        eng.set_clusters(K, P0)
        st, shift, _ = eng.score_stats(K, ev)
        eng.estep(K)
        eng.em_iterations(K, 1)
        got = eng.get_clusters(K, with_memberships=True)
        fp = eng.fit_profile()
    assert fp["device_finalize_launches"] == 1 and fp["host_replays"] == 0
    F = 1 + D + D * (D + 1) // 2
    S = st[:K * F].reshape(K, F)
    S0, S1 = S[:, 0], S[:, 1:1 + D]
    Nf = S0.astype(np.float32)
    np.testing.assert_array_equal(got.N[:K], Nf)
    m = np.where(S0[:, None] != 0, S1 / np.where(S0 != 0, S0, 1.0)[:, None], 0.0)
    mu = np.where((Nf > 0.5)[:, None], (m + shift).astype(np.float32), np.float32(0))
    np.testing.assert_array_equal(got.means[:K], mu)
    il = np.tril_indices(D)
    for k in range(K):
        if not Nf[k] > 0.5:
            np.testing.assert_array_equal(got.R[k], np.eye(D, dtype=np.float32))
            continue
        S2 = np.zeros((D, D))
        S2[il] = S[k, 1 + D:]
        S2 = np.tril(S2) + np.tril(S2, -1).T
        cov = S2 - np.outer(m[k], S1[k]) if Nf[k] >= 1 else np.zeros((D, D))
        cov = np.tril(cov) + np.tril(cov, -1).T            # the lower triangle is what the finalisation forms
        cov[np.diag_indices(D)] += float(P0.avgvar[k])
        R = (cov * (1.0 / float(Nf[k]))).astype(np.float32)
        # numpy rounds m_i * S1_j before subtracting it (no fused multiply-add on this Python), the library fuses the
        # two: the results may differ by one float ulp where the subtraction cancels
        ulp = np.spacing(np.abs(R))
        assert np.all(np.abs(got.R[k].astype(np.float64) - R) <= ulp), f"R[{k}] beyond one ulp"
    ref = pkg.Clusters(K, D, N)
    for f in FIELDS + ("avgvar",):
        getattr(ref, f)[...] = getattr(got, f)
    _consistent(ref, K)
    tot = 0.0
    for x in Nf:                                           # the reference's order (compute_pi): k = 0, 1, ...
        tot += float(x)
    ref.pi[:K] = np.where(Nf < 0.5, np.float32(1e-10), (Nf.astype(np.float64) / tot).astype(np.float32))
    np.testing.assert_array_equal(got.pi[:K], ref.pi[:K])
    for k in range(K):
        # Rinv and ln det from a float64 inverse of the float R: an inverse moves a relative change of R by up to
        # cond(R), so these are held to the parity bars of assert_params_close, not to equality
        cond = float(np.linalg.cond(got.R[k].astype(np.float64)))
        tol = 1e-4 * max(10.0, cond)
        np.testing.assert_allclose(got.Rinv[k], ref.Rinv[k], rtol=tol, atol=tol * float(np.abs(ref.Rinv[k]).max()))
        assert abs(float(got.constant[k]) - float(ref.constant[k])) <= max(2e-3, 0.5 * D * 1e-4 * cond) + 1e-4 * abs(float(ref.constant[k]))
    # the E-step after the step, on the device-produced set, against the float64 E-step: the per-operator bar of 1e-4
    # (the tensor E-step evaluates the quadratic forms in FP16 hi/lo products with FP32 accumulation)
    chk = pkg.Clusters(K, D, N)
    for f in FIELDS + ("avgvar",):
        getattr(chk, f)[...] = getattr(got, f)
    oracle64.estep(oracle64.transpose(ev), chk, K)
    np.testing.assert_allclose(got.memberships[:K], chk.memberships[:K], rtol=1e-4, atol=1e-6)


# ---- 3. statistics at every branch of the kernel --------------------------------------------------------------------
def _branch_scene(pkg, D, rank_events=3, needle_avgvar=3e-10):
    """Blob data with isolated events about 20 global standard deviations out (inside the tensor M-step's 64-sigma range),
    and a parameter set P0 whose next finalisation meets every branch of the kernel.  Returns (events, P0, roles)."""
    rng = np.random.default_rng(400 + D)
    nb = 3
    centres = rng.standard_normal((nb, D)) * 4.0
    blobs = [c + rng.standard_normal((5_000, D)) for c in centres]
    base = np.concatenate(blobs)
    centre = base.mean(0)
    gs = float(base.std(0).mean())
    far = 20.0 * gs
    ax = np.eye(D)
    e_pair = centre + far * ax[0]                                   # shared by the 0.7 : 0.3 pair
    rank_pts = centre + far * ax[1] + rng.standard_normal((rank_events, D))   # rank_events - 1 <= D - 1
    wide_pts = np.stack([centre - far * ax[0], centre - far * ax[1]])      # owned by the wide cluster only
    off_pts = centre + far * ax[2] + 0.5 * rng.standard_normal((D + 4, D))  # full rank, far from the centre
    extra = [e_pair[None], rank_pts, wide_pts, off_pts, np.repeat(centre[None], 3, 0)]
    ev = np.concatenate([base] + extra).astype(np.float32)
    # the needle's three identical events sit on the centre the statistics are taken about (the float-rounded mean of
    # all events): their moments are exactly zero, so the needle keeps its width through the step
    for _ in range(3):
        ev[-3:] = ev.astype(np.float64).mean(0).astype(np.float32)
    needle_pt = ev[-1].copy()
    ev = ev[rng.permutation(ev.shape[0])]

    # the E-step flushes responsibilities far below the largest to zero: the 1e-34 probe has S0 = 0 exactly, the others
    # N from ~1e-5 up, many ulps of the double sum below the sum's last bit
    probes = [1e-34, 2e-9, 7e-9, 3e-8, 1e-7, 4e-7, 2e-6, 1e-5, 1e-3, 1e-1]
    roles = {}
    rows = []                                                      # (name, mean, sigma, pi, avgvar)
    for b in range(nb):
        rows.append((f"blob{b}", centres[b], 1.0, 0.3, 0.01))
    rows.append(("far", centre + 40.0 * gs * ax[3 % D] + 30.0 * gs * ax[4 % D], 1.0, 0.01, 0.01))
    rows.append(("pair7", e_pair, 1.0, 0.007, 0.01))
    rows.append(("pair3", e_pair, 1.0, 0.003, 0.01))
    rows.append(("rank", rank_pts.mean(0), 3.0, 0.01, 0.1))
    rows.append(("needle", needle_pt, 1e-5, 0.01, needle_avgvar))
    rows.append(("wide", centre, 400.0 * gs, 1e-3, 2.0 * (400.0 * gs) ** 2))
    rows.append(("offset", off_pts.mean(0), 0.5, 0.01, 0.01))
    for i, eps in enumerate(probes):                                # N = (5000 events) x eps: 0, 1e-5 .. 500
        rows.append((f"probe{i}", centres[0], 1.0, 0.3 * eps, 0.01))
    K = len(rows)
    P0 = pkg.Clusters(K, D)
    for k, (name, mean, sig, pi, av) in enumerate(rows):
        roles[name] = k
        P0.means[k] = mean
        P0.R[k] = np.eye(D) * sig * sig
        P0.pi[k] = pi
        P0.N[k] = pi * ev.shape[0]
        P0.avgvar[k] = av
    _consistent(P0, K)
    return ev, P0, roles, gs


@pytest.mark.parametrize("D", [8, 16, 24])
def test_finalisation_branches_bit_identical(loaded, D):
    """S0 = 0, 0 < N < 0.5 (mu = 0, R = I, pi = 1e-10), 0.5 < N < 1 (R = diag(avgvar) / N), a rank-deficient cluster
    positive definite through avgvar only, a needle (sigma ~ 1e-5) and a cluster 400x wider than the data (power-of-two
    operand scales far from 0 both ways), an offset v larger than every factor entry, and N from 1e-5 to 5e3 (the
    double sum behind pi depends on its order): the branch the reference rules give, and device == host bit for bit."""
    pkg = loaded
    ev, P0, ro, gs = _branch_scene(pkg, D)
    K = P0.N.shape[0]
    (((dev, ll_d), fp_d), ((host, ll_h), fp_h)) = _both(pkg, ev, K, _one_step(P0, K))
    assert fp_d["device_finalize_launches"] == 1 and fp_d["host_replays"] == 0
    assert fp_h["device_finalize_launches"] == 0
    I = np.eye(D, dtype=np.float32)
    # S0 underflows to exactly 0
    k = ro["far"]
    assert dev.N[k] == 0.0 and dev.pi[k] == np.float32(1e-10)
    np.testing.assert_array_equal(dev.means[k], 0.0)
    np.testing.assert_array_equal(dev.R[k], I)
    # 0 < N < 0.5: mu = 0, R = I, pi = 1e-10
    k = ro["pair3"]
    assert 0.25 < dev.N[k] < 0.35 and dev.pi[k] == np.float32(1e-10)
    np.testing.assert_array_equal(dev.means[k], 0.0)
    np.testing.assert_array_equal(dev.R[k], I)
    # 0.5 < N < 1: the covariance is zeroed, R = diag(avgvar) / N
    k = ro["pair7"]
    assert 0.65 < dev.N[k] < 0.75 and dev.pi[k] != np.float32(1e-10)
    rdiag = np.float32(float(P0.avgvar[k]) * (1.0 / float(dev.N[k])))
    np.testing.assert_array_equal(dev.R[k], I * rdiag)
    # rank-deficient: N = its events, positive definite only through avgvar
    k = ro["rank"]
    assert abs(float(dev.N[k]) - 3.0) < 1e-3
    reg = np.eye(D) * float(P0.avgvar[k]) / float(dev.N[k])
    assert np.linalg.matrix_rank(dev.R[k].astype(np.float64) - reg, tol=0.1 * reg[0, 0]) <= 2
    # needle and wide cluster: R at 1e-10 and at (400 sigma)^2
    k = ro["needle"]
    assert abs(float(dev.N[k]) - 3.0) < 1e-3 and 0 < float(np.diag(dev.R[k]).max()) < 1e-9
    k = ro["wide"]
    assert float(np.diag(dev.R[k]).min()) > (100.0 * gs) ** 2
    # probes: N = 0 and 1e-5 .. 500, the small ones take the N < 0.5 branch
    Np = np.array([dev.N[ro[f"probe{i}"]] for i in range(10)], np.float64)
    assert Np[0] == 0.0 and np.all(Np[1:] > 0) and Np[1] < 1e-4 and Np[-1] > 100
    for i in range(10):
        if Np[i] < 0.5:
            assert dev.pi[ro[f"probe{i}"]] == np.float32(1e-10)
    _assert_same(dev, host, K, f"D={D}")
    assert ll_d == ll_h


# ---- 4. whole drivers ------------------------------------------------------------------------------------------------
def test_em_iterations_two_batches_bit_identical(loaded):
    """em_iterations(K, 6), then a second batch of 2 in the same context."""
    pkg = loaded
    N, D, K = 20_000, 24, 40
    ev = pkg.synth.make_blobs(N, D, 12, seed=501)

    def body(eng):
        eng.seed(K)
        eng.estep(K)
        ll1 = eng.em_iterations(K, 6)
        a = eng.get_clusters(K, with_memberships=True)
        ll2 = eng.em_iterations(K, 2)
        return a, ll1, eng.get_clusters(K, with_memberships=True), ll2

    (((d1, dl1, d2, dl2), fp_d), ((h1, hl1, h2, hl2), fp_h)) = _both(pkg, ev, K, body)
    assert fp_d["device_finalize_launches"] == 8 and fp_d["host_replays"] == 0 and fp_h["device_finalize_launches"] == 0
    _assert_same(d1, h1, K, "batch 1")
    _assert_same(d2, h2, K, "batch 2")
    assert dl1 == hl1 and dl2 == hl2


def test_em_driver_bit_identical(loaded):
    """gmm_em(K, 4, 20): the first 4 iterations on the device path, then the host path of the convergence test."""
    pkg = loaded
    N, D, K = 20_000, 16, 24
    ev = pkg.synth.make_blobs(N, D, 8, seed=502)

    def body(eng):
        eng.seed(K)
        ll, it = eng.em(K, 4, 20)
        return eng.get_clusters(K, with_memberships=True), ll, it

    (((d, dll, dit), fp_d), ((h, hll, hit), fp_h)) = _both(pkg, ev, K, body)
    assert fp_d["device_finalize_launches"] == 4 and fp_d["host_replays"] == 0 and fp_h["device_finalize_launches"] == 0
    assert dit == hit and dit >= 4
    _assert_same(d, h, K)
    assert dll == hll


def test_fit_driver_bit_identical(loaded):
    """gmm_fit(K0 = 72, target = 60) at D = 24: K shrinks inside one context, each K starts on the device path."""
    pkg = loaded
    N, D = 30_000, 24
    ev = pkg.synth.make_blobs(N, D, 16, seed=503)

    def body(eng):
        ideal, mr, saved = eng.fit(72, 60, 2, 2, with_memberships=True)
        return ideal, mr, saved

    (((di, dmr, ds), fp_d), ((hi, hmr, hs), fp_h)) = _both(pkg, ev, 72, body)
    assert fp_d["device_finalize_launches"] == 2 * 13 and fp_d["host_replays"] == 0 and fp_h["device_finalize_launches"] == 0
    assert di == hi == 60 and dmr == hmr
    _assert_same(ds, hs, di)


# ---- 5. real host replays ----------------------------------------------------------------------------------------------
def test_replay_negative_definite_cluster(loaded):
    """A strongly negative avgvar (gmm_set_clusters does not validate it) makes a cluster's R negative definite: the device
    factorisation fails at its first pivot, the host takes the no-pivot LU path and the SIMT E-step, and the result is the
    all-host run's bit for bit."""
    pkg = loaded
    N, D, K = 15_000, 16, 12
    ev = pkg.synth.make_blobs(N, D, 6, seed=511)
    P0 = _seed_params(pkg, ev, K)
    P0.avgvar[5] = -1e6

    def body(eng):
        eng.set_clusters(K, P0)
        eng.estep(K)
        ll = eng.em_iterations(K, 1)
        return eng.get_clusters(K, with_memberships=True), ll

    (((d, dll), fp_d), ((h, hll), fp_h)) = _both(pkg, ev, K, body)
    assert fp_d["device_finalize_launches"] == 1 and fp_d["host_replays"] == 1
    assert fp_h["device_finalize_launches"] == 0 and fp_h["host_replays"] == 0
    assert np.all(np.linalg.eigvalsh(d.R[5].astype(np.float64)) < 0)
    _assert_same(d, h, K)
    np.testing.assert_equal(dll, hll)


@pytest.mark.parametrize("D", [8, 24])
def test_replay_zero_avgvar_on_repeated_events(loaded, D):
    """avgvar = 0 on a cluster that owns only identical events (the raw covariance score_stats' users ask for): its R is
    zero up to rounding, and whichever way the rounding goes (device path or host replay), device == host bit for bit."""
    pkg = loaded
    ev, P0, ro, _ = _branch_scene(pkg, D, needle_avgvar=0.0)
    K = P0.N.shape[0]
    (((d, dll), fp_d), ((h, hll), fp_h)) = _both(pkg, ev, K, _one_step(P0, K))
    assert fp_d["device_finalize_launches"] == 1 and fp_d["host_replays"] in (0, 1)
    assert fp_h["device_finalize_launches"] == 0 and fp_h["host_replays"] == 0
    assert abs(float(d.N[ro["needle"]]) - 3.0) < 1e-3
    _assert_same(d, h, K)
    np.testing.assert_equal(dll, hll)


@pytest.mark.parametrize("batch", [1, 2])
@pytest.mark.parametrize("start", ["seed", "set_clusters"])
def test_replay_at_first_iteration_of_a_batch(loaded, batch, start):
    """A replay at the first iteration of a batch (finalize_fault_iter = 0) of the first batch, or of a second batch after
    a good device batch: the host rebuilds the responsibilities that batch started from exactly as the all-host run
    built them (from R's factor after a finalisation, from the given Rinv after a seed or gmm_set_clusters)."""
    pkg = loaded
    N, D, K = 20_000, 24, 32
    ev = pkg.synth.make_blobs(N, D, 10, seed=520)
    P0 = random_spd_params(pkg, K, D, np.random.default_rng(521), spread=8.0) if start == "set_clusters" else None
    if P0 is not None:
        P0.pi[:] = P0.N / P0.N.sum()
        _consistent(P0, K)

    def body(fault):
        def run(eng):
            if P0 is None:
                eng.seed(K)
            else:
                eng.set_clusters(K, P0)
            eng.estep(K)
            if batch == 1 and fault:
                eng.set_option("finalize_fault_iter", 0)
            ll1 = eng.em_iterations(K, 3)
            a = eng.get_clusters(K, with_memberships=True)
            p1 = eng.fit_profile()
            if batch == 2 and fault:
                eng.set_option("finalize_fault_iter", 0)
            ll2 = eng.em_iterations(K, 2)
            return a, ll1, p1, eng.get_clusters(K, with_memberships=True), ll2
        return run

    with pkg.Engine(ev, K) as eng:
        eng.set_option("finalize", 1)
        rep = body(True)(eng)
        fp = eng.fit_profile()
    with pkg.Engine(ev, K) as eng:
        eng.set_option("finalize", 0)
        host = body(False)(eng)
        fp_h = eng.fit_profile()
    assert fp_h["device_finalize_launches"] == 0 and fp_h["host_replays"] == 0
    if batch == 1:
        assert rep[2]["host_replays"] == 1 and rep[2]["device_finalize_launches"] == 3
        assert fp["host_replays"] == 1 and fp["device_finalize_launches"] == 3      # the context stays on the host path
    else:
        assert rep[2]["host_replays"] == 0 and rep[2]["device_finalize_launches"] == 3
        assert fp["host_replays"] == 1 and fp["device_finalize_launches"] == 5
    _assert_same(rep[0], host[0], K, "batch 1")
    _assert_same(rep[3], host[3], K, "batch 2")
    assert rep[1] == host[1] and rep[4] == host[4]
