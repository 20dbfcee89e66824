"""The tensor M-step (`mstep_tc_kernel<D>`) against an exact M-step on the responsibilities it actually read
(run with -m gpu on an H100).

The reference isolates the M-step from the E-step: the engine's E-step writes the responsibilities, they are read back,
the packed statistics are formed from them and the float32 events in float64 (exact_mstep_stats) about the
engine's centre, and the library's own host finalisation turns them into N, means and R.  The only difference left is the
statistics the tensor kernels produce.  Every case asserts which M-step kernel ran, and holds the per-cluster bar of
MSTEP_TOL, which tests/test_mstep_error_model.py derives from the kernel's operand arithmetic and shows to fail
for dropped or wrong operand products and a lost drain.  On data built so that the whole kernel is exact, the parameters
must be bit-identical to the reference."""
import numpy as np
import pytest

from conftest import fitted_params
from test_mstep_error_model import cta_ranges, exact_mstep_stats, outlier_blobs, param_errors, standardise

pytestmark = pytest.mark.gpu

MSTEP_D = (4, 8, 12, 16, 20, 24)


def n_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def loaded(pkg):
    pkg.load_library()
    return pkg


def estep_mstep(pkg, eng, K, cl):
    """set_clusters + E-step + tensor M-step on an open engine: (parameters, responsibilities the M-step read)."""
    eng.set_clusters(K, cl)
    eng.estep(K)
    memb = eng.get_clusters(K, with_memberships=True).memberships.copy()
    eng.mstep(K)
    return eng.get_clusters(K), memb


def engine(pkg, ev, Kmax, estep=None, mstep=None):
    eng = pkg.Engine(ev, Kmax)
    eng.set_option("estep_path", pkg.PATH_SIMT if estep is None else estep)
    if mstep is not None:
        eng.set_option("mstep_path", mstep)
    return eng


def reference(pkg, ev, memb, got, K):
    """The exact M-step on the engine's responsibilities, finalised by the library's host code."""
    shift = standardise(ev)[0]
    ref = pkg.Clusters(K, ev.shape[1])
    ref.avgvar[:K] = got.avgvar[:K]
    pkg.host_finalize(exact_mstep_stats(ev, memb[:K], shift), shift, ref, K)
    return ref, shift


def check_bar(pkg, ev, memb, got, K, label):
    ref, shift = reference(pkg, ev, memb, got, K)
    e = param_errors(got.N[:K], got.means[:K], got.R[:K], ref.N[:K], ref.means[:K], ref.R[:K], shift)
    print(f"\n[mstep-tc] {label}: N {e['N']:.2e}  mean {e['mean']:.2e}  R {e['R']:.2e}  worst/bar {e['worst']:.3f}")
    assert e["worst"] <= 1.0, e
    return ref


def run_tensor_mstep(pkg, ev, cl, K, label):
    with engine(pkg, ev, K, mstep=pkg.PATH_TENSOR) as eng:
        got, memb = estep_mstep(pkg, eng, K, cl)
        assert eng.profile()["mstep_tensor_launches"] == 1
    check_bar(pkg, ev, memb, got, K, label)


@pytest.mark.parametrize("K", [7, 33, 100])
@pytest.mark.parametrize("D", MSTEP_D)
def test_mstep_tc_every_D(loaded, oracle64, D, K):
    """Every compiled width, one and several 32-cluster grid rows (33: one live column in the second row)."""
    ev = loaded.synth.make_blobs(20_000, D, min(K, 16), seed=600 + D)
    run_tensor_mstep(loaded, ev, fitted_params(loaded, oracle64, ev, K), K, f"D={D} K={K} N=20000")


@pytest.mark.parametrize("D", MSTEP_D)
def test_mstep_tc_one_cluster(loaded, oracle64, D):
    """K = 1: every responsibility is 1 and only column 0 of the grid row is live."""
    ev = loaded.synth.make_blobs(20_000, D, 4, seed=610 + D)
    run_tensor_mstep(loaded, ev, fitted_params(loaded, oracle64, ev, 1), 1, f"D={D} K=1 N=20000")


def edge_n(name, sms):
    """Event counts at the M-step's tile and launch edges, from launch_mstep_d()'s per / gx arithmetic."""
    return {"gx<sms": 32 * (sms - 4) - 1,           # per = 32 (one sub-tile per CTA), fewer CTAs than SMs
            "full+1": 64 * (sms // 2) + 1,          # full CTAs, then a last CTA that holds one event
            "partial-chain": 160 * sms - 17,        # per = 160: a 128-event chain and a partial one, a partial last sub-tile
            }.get(name) or int(name)


EDGES = ["1", "31", "32", "33", "127", "129", "gx<sms", "full+1", "partial-chain", "300001"]


@pytest.mark.parametrize("name", EDGES)
@pytest.mark.parametrize("D", [12, 24])
def test_mstep_tc_shard_edges(loaded, oracle64, D, name):
    """Tiny shards, CTAs that end in a partial sub-tile or a partial chain, fewer CTAs than SMs, one full CTA plus one
    event, and many 512-event remainder chains per CTA.  Parameters are fitted on 20 000 events; the data is their
    first N."""
    sms = n_sms()
    N = edge_n(name, sms)
    per, gx = cta_ranges(N, sms)
    if name == "gx<sms":
        assert per == 32 and gx < sms
    elif name == "full+1":
        assert N - (gx - 1) * per == 1
    elif name == "partial-chain":
        assert per % 128 and N % 32
    K = 8
    big = loaded.synth.make_blobs(max(N, 20_000), D, 8, seed=620 + D)
    cl = fitted_params(loaded, oracle64, big[:20_000], K)
    run_tensor_mstep(loaded, np.ascontiguousarray(big[:N]), cl, K, f"D={D} K={K} N={N} ({name}: per {per}, gx {gx})")


@pytest.mark.parametrize("estep", ["simt", "tensor"])
def test_mstep_tc_stale_rows_above_K(loaded, oracle64, estep):
    """A context sized for Kmax = 100 after a K = 100 iteration runs K = 40: the second grid row's TMA box reads stale
    responsibility rows 40..63.  The K = 40 results must be those of a fresh Kmax = 40 context, bit for bit."""
    pkg = loaded
    D, N = 24, 20_000
    ev = pkg.synth.make_blobs(N, D, 16, seed=630)
    p100 = fitted_params(pkg, oracle64, ev, 100)
    p40 = fitted_params(pkg, oracle64, ev, 40)
    path = pkg.PATH_SIMT if estep == "simt" else pkg.PATH_TENSOR
    with engine(pkg, ev, 100, estep=path, mstep=pkg.PATH_TENSOR) as eng:
        estep_mstep(pkg, eng, 100, p100)
        got, memb = estep_mstep(pkg, eng, 40, p40)
        assert eng.profile()["mstep_tensor_launches"] == 2
    with engine(pkg, ev, 40, estep=path, mstep=pkg.PATH_TENSOR) as eng:
        fresh, memb_fresh = estep_mstep(pkg, eng, 40, p40)
        assert eng.profile()["mstep_tensor_launches"] == 1
    np.testing.assert_array_equal(memb[:40], memb_fresh[:40])
    for f in ("N", "means", "R"):
        np.testing.assert_array_equal(getattr(got, f)[:40], getattr(fresh, f)[:40], err_msg=f)
    check_bar(pkg, ev, memb, got, 40, f"D={D} K=40 of Kmax=100, {estep} E-step")


# ---- exactness on dyadic data -------------------------------------------------------------------------------------
def dyadic_events(D, K, sms):
    """Events on which the whole tensor M-step is exact.  In standardised units each coordinate is a cluster centre
    +-c plus an offset from {+-A, +-B}, every multiset balanced per cluster and dimension, so that every column mean is 0
    and every variance is exactly 1 (c^2 + E[o^2] = 1); dimension d is scaled by 2^((d mod 3) - 1), a power-of-two
    standard deviation.  The largest |z| is 1.75 (K = 1) or 1.6875 (|o| < c: every coordinate lies on its cluster's
    side), so zb = 2 and every z (multiple of 2^-4) and z_i z_j (of 2^-8) is a multiple of its quantum (2^-10, 2^-9).
    Each cluster's events are sorted by their dimension-0 offset, so that whole 128-event chains repeat the largest
    square.  N is the largest multiple of the balanced unit with at most 128 events per CTA."""
    if K == 1:
        c, A, B, big, small = 0.0, 1.75, 0.25, 5, 11              # (5 * 1.75^2 + 11 * 0.25^2) / 16 = 1
    else:
        c, A, B, big, small = 0.9375, 0.75, 0.125, 27, 113        # 0.9375^2 + (27 * 0.75^2 + 113 * 0.125^2) / 140 = 1
    unit = 2 * (big + small)
    u = 128 * sms // (K * unit)
    m = unit * u                                                   # events per cluster
    if K == 1:
        sign = np.ones((1, D))
    elif K == 2:
        sign = np.array([[1 - 2 * ((k + d) % 2) for d in range(D)] for k in range(2)], np.float64)
    else:
        sign = np.array([[1 - 2 * ((k >> (d % 2)) & 1) for d in range(D)] for k in range(4)], np.float64)
    rng = np.random.default_rng(640 + D * 8 + K)
    base = np.repeat([A, -A, B, -B], [big * u, big * u, small * u, small * u])
    blocks = []
    for k in range(K):
        o = np.stack([rng.permutation(base) for _ in range(D)], axis=1)
        o = o[np.argsort(-o[:, 0] * sign[k, 0], kind="stable")]
        blocks.append(sign[k] * c + o)
    z = np.concatenate(blocks)
    scale = 2.0 ** (np.arange(D) % 3 - 1)
    return (z * scale).astype(np.float32), sign * c * scale, scale


@pytest.mark.parametrize("K", [1, 2, 4])
@pytest.mark.parametrize("D", MSTEP_D)
def test_mstep_tc_exact_on_dyadic_data(loaded, oracle64, D, K):
    """Responsibilities exactly 0 or 1, exact centre and scale, no remainder (p_l = 0, g_l = 0), one exact chain per
    CTA and tile at up to 77 % of the 2^24-quanta budget: a wrong row map, scale, drain, lost chain or budget overflow
    changes the parameters.  They must equal the float64 reference bit for bit."""
    pkg = loaded
    sms = n_sms()
    ev, centres, scale = dyadic_events(D, K, sms)
    N = len(ev)
    shift, sc, z, zb = standardise(ev)
    assert not shift.any() and np.array_equal(sc, scale) and zb == 2.0
    per, gx = cta_ranges(N, sms)
    assert per == 128
    cl = pkg.Clusters(K, D)
    cl.means[:K] = centres
    cl.R[:K] = np.diag((0.05 * scale) ** 2)                       # 0/1 responsibilities: log-odds of several hundred
    cl.N[:K] = N / K
    oracle64.constants(cl, K)
    with engine(pkg, ev, K, mstep=pkg.PATH_TENSOR) as eng:
        got, memb = estep_mstep(pkg, eng, K, cl)
        assert eng.profile()["mstep_tensor_launches"] == 1
    assert np.isin(memb, (0.0, 1.0)).all() and (memb.sum(0) == 1.0).all()
    # the fullest chain: the diagonal statistic of dimension 0 over one CTA's 128 events of one cluster
    pad = gx * per - N
    zz = np.pad(z[:, 0] ** 2, (0, pad)).reshape(gx, per)
    g = np.pad(memb[:K], ((0, 0), (0, pad))).reshape(K, gx, per)
    budget = float((g * zz).sum(2).max()) / (128 * zb * zb)
    assert budget >= 0.7, budget
    ref, _ = reference(pkg, ev, memb, got, K)
    print(f"\n[mstep-tc] dyadic D={D} K={K} N={N}: fullest chain {budget:.1%} of the budget")
    np.testing.assert_array_equal(got.N[:K], ref.N[:K])
    np.testing.assert_array_equal(got.means[:K], ref.means[:K])
    np.testing.assert_array_equal(got.R[:K], ref.R[:K])


# ---- the fixed-point range boundary (tc_mstep_ready: zb <= 64) ----------------------------------------------------
@pytest.mark.parametrize("ztarget,tensor", [(63.0, True), (65.0, False)])
def test_mstep_range_boundary(loaded, oracle64, ztarget, tensor):
    """One event just under 64 standard deviations (zb = 64, the fewest bits above the quantum for the bulk): GMM_PATH_AUTO
    runs the tensor M-step and it holds the bar (test_mstep_error_model: no widening is needed at zb = 64).  Just over 64
    (zb = 128): GMM_PATH_AUTO runs the FP64 SIMT M-step."""
    pkg = loaded
    K = 8
    ev = outlier_blobs(200_000, 12, ztarget, seed=611)
    assert standardise(ev)[3] == (64.0 if tensor else 128.0)
    cl = fitted_params(pkg, oracle64, ev, K)
    with pkg.Engine(ev, K) as eng:
        got, memb = estep_mstep(pkg, eng, K, cl)
        p = eng.profile()
    assert (p["mstep_tensor_launches"], p["mstep_simt_launches"]) == ((1, 0) if tensor else (0, 1))
    check_bar(pkg, ev, memb, got, K, f"D=12 K={K} N=200000, largest |z| {ztarget:g} ({'tensor' if tensor else 'SIMT'})")


# ---- tensor E-step: fewer events than one tile, and a second / third pass of 64 clusters ---------------------------
@pytest.mark.parametrize("N,K", [(1, 5), (63, 5), (64, 5), (65, 5), (3_000, 1), (3_000, 65), (3_000, 129)])
@pytest.mark.parametrize("D", [8, 16, 24])
def test_estep_tc_small_edges(loaded, oracle64, D, N, K):
    """The wgmma E-step against the f64 oracle at the per-operator bar.  Parameters are fitted on 20 000 events; the
    data is their first N."""
    pkg = loaded
    big = pkg.synth.make_blobs(20_000, D, min(K, 16), seed=650 + D)
    fit = fitted_params(pkg, oracle64, big, K)
    ev = np.ascontiguousarray(big[:N])
    ref = pkg.Clusters(K, D, N)
    for f in pkg.Clusters.FIELDS:
        getattr(ref, f)[...] = getattr(fit, f)
    with pkg.Engine(ev, K) as eng:
        eng.set_option("path", pkg.PATH_TENSOR)
        eng.set_clusters(K, ref)
        ll = eng.estep(K)
        got = eng.get_clusters(K, with_memberships=True)
    ll_ref = oracle64.estep(oracle64.transpose(ev), ref, K)
    np.testing.assert_allclose(got.memberships, ref.memberships, rtol=1e-4, atol=1e-6)
    np.testing.assert_allclose(got.memberships.sum(0), 1.0, atol=1e-5)
    assert abs(ll - ll_ref) <= 1e-5 * abs(ll_ref)
