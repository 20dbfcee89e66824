"""The tensor M-step's schedule for K > 32 (`mstep_tc_kernel<D, 64>`: two CTAs per event range, each with half of the
feature rows and 64 clusters) against an exact M-step on the responsibilities it read (run with -m gpu on an H100).

The bars are those of tests/test_gpu_mstep_tc.py: the per-cluster bar of MSTEP_TOL against the FP64 statistics of the
engine's own responsibilities, and bit-identity with the float64 reference on dyadic data with 0/1 responsibilities."""
import numpy as np
import pytest

from conftest import fitted_params
from test_gpu_mstep_tc import (MSTEP_D, check_bar, dyadic_events, edge_n, engine, estep_mstep, n_sms, reference,
                               run_tensor_mstep)
from test_mstep_error_model import cta_ranges, standardise

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def loaded(pkg):
    pkg.load_library()
    return pkg


@pytest.mark.parametrize("K", [33, 40, 64, 65, 100, 128])
@pytest.mark.parametrize("D", MSTEP_D)
def test_mstep_pair_every_D(loaded, oracle64, D, K):
    """One and two 64-cluster grid rows; 33 / 65: one live cluster in the last 32-cluster block (65: its second box is
    not loaded)."""
    ev = loaded.synth.make_blobs(20_000, D, 16, seed=700 + D)
    run_tensor_mstep(loaded, ev, fitted_params(loaded, oracle64, ev, K), K, f"D={D} K={K} N=20000")


@pytest.mark.parametrize("K", [40, 64, 128])
@pytest.mark.parametrize("D", MSTEP_D)
def test_mstep_pair_exact_on_dyadic_data(loaded, oracle64, D, K):
    """The dyadic data of test_mstep_tc_exact_on_dyadic_data (4 clusters, every step of the kernel exact), its clusters
    placed in both 32-cluster blocks of a CTA and, at K = 128, in the second grid row; the other clusters sit far from
    every event and take responsibility exactly 0.  The parameters must equal the float64 reference bit for bit."""
    pkg = loaded
    sms = n_sms()
    ev, centres, scale = dyadic_events(D, 4, sms)
    N = len(ev)
    shift, sc, z, zb = standardise(ev)
    assert not shift.any() and np.array_equal(sc, scale) and zb == 2.0
    per, gx = cta_ranges(N, sms)
    assert per == 128
    live = [0, 31, 32, K - 1]
    cl = pkg.Clusters(K, D)
    for k in range(K):
        cl.means[k] = 64.0 * (1.0 + k / K) * scale
    cl.means[live] = centres
    cl.R[:K] = np.diag((0.05 * scale) ** 2)
    cl.N[:K] = N / K
    oracle64.constants(cl, K)
    with engine(pkg, ev, K, mstep=pkg.PATH_TENSOR) as eng:
        got, memb = estep_mstep(pkg, eng, K, cl)
        assert eng.profile()["mstep_tensor_launches"] == 1
    assert np.isin(memb, (0.0, 1.0)).all() and (memb.sum(0) == 1.0).all()
    assert (memb[live].sum(1) > 0).all() and memb.sum() == memb[live].sum()
    pad = gx * per - N
    zz = np.pad(z[:, 0] ** 2, (0, pad)).reshape(gx, per)
    g = np.pad(memb[:K], ((0, 0), (0, pad))).reshape(K, gx, per)
    budget = float((g * zz).sum(2).max()) / (128 * zb * zb)
    assert budget >= 0.7, budget
    ref, _ = reference(pkg, ev, memb, got, K)
    print(f"\n[mstep-pair] dyadic D={D} K={K} N={N}: fullest chain {budget:.1%} of the budget")
    np.testing.assert_array_equal(got.N[:K], ref.N[:K])
    np.testing.assert_array_equal(got.means[:K], ref.means[:K])
    np.testing.assert_array_equal(got.R[:K], ref.R[:K])


def test_mstep_pair_kmax128_at_k64(loaded, oracle64):
    """A context sized for Kmax = 128 after a K = 128 iteration runs K = 64: the results must be those of a fresh
    Kmax = 64 context, bit for bit."""
    pkg = loaded
    D, N = 24, 20_000
    ev = pkg.synth.make_blobs(N, D, 16, seed=730)
    p128 = fitted_params(pkg, oracle64, ev, 128)
    p64 = fitted_params(pkg, oracle64, ev, 64)
    with engine(pkg, ev, 128, mstep=pkg.PATH_TENSOR) as eng:
        estep_mstep(pkg, eng, 128, p128)
        got, memb = estep_mstep(pkg, eng, 64, p64)
        assert eng.profile()["mstep_tensor_launches"] == 2
    with engine(pkg, ev, 64, mstep=pkg.PATH_TENSOR) as eng:
        fresh, memb_fresh = estep_mstep(pkg, eng, 64, p64)
        assert eng.profile()["mstep_tensor_launches"] == 1
    np.testing.assert_array_equal(memb[:64], memb_fresh[:64])
    for f in ("N", "means", "R"):
        np.testing.assert_array_equal(getattr(got, f)[:64], getattr(fresh, f)[:64], err_msg=f)
    check_bar(pkg, ev, memb, got, 64, f"D={D} K=64 of Kmax=128")


@pytest.mark.parametrize("name", ["1", "33", "gx<sms", "full+1", "partial-chain"])
@pytest.mark.parametrize("D", [12, 24])
def test_mstep_pair_shard_edges(loaded, oracle64, D, name):
    """One event, fewer ranges than SMs, a last range of one event, and ranges that end in a partial chain and a partial
    sub-tile, at K = 65 (two grid rows).  Parameters are fitted on 20 000 events; the data is their first N."""
    sms = n_sms()
    N = edge_n(name, sms)
    per, gx = cta_ranges(N, sms)
    if name == "gx<sms":
        assert per == 32 and gx < sms
    elif name == "full+1":
        assert N - (gx - 1) * per == 1
    elif name == "partial-chain":
        assert per % 128 and N % 32
    K = 65
    big = loaded.synth.make_blobs(max(N, 20_000), D, 16, seed=740 + D)
    cl = fitted_params(loaded, oracle64, big[:20_000], K)
    run_tensor_mstep(loaded, np.ascontiguousarray(big[:N]), cl, K, f"D={D} K={K} N={N} ({name}: per {per}, gx {gx})")
