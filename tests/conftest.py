import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as entry  # noqa: E402


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu on a GPU machine)")


@pytest.fixture(scope="session")
def pkg():
    p = entry.load_package()
    if not os.path.exists(p.library_path()):
        entry.build()
    p.load_library()
    return p


@pytest.fixture(scope="session")
def oracle64(pkg):
    return entry.load_oracle("f64")


@pytest.fixture(scope="session")
def oracle32(pkg):
    return entry.load_oracle("f32")


def have_gpu():
    try:
        import ctypes
        rt = ctypes.CDLL("libcudart.so.12")
        n = ctypes.c_int(0)
        return rt.cudaGetDeviceCount(ctypes.byref(n)) == 0 and n.value > 0
    except OSError:
        try:
            import torch
            return torch.cuda.is_available()
        except Exception:
            return False


def gpu_count():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


def random_spd_params(pkg, K, D, rng, spread=4.0):
    """Random, well-conditioned mixture parameters with consistent Rinv/constant."""
    cl = pkg.Clusters(K, D)
    cl.means[...] = rng.uniform(-spread, spread, size=(K, D)).astype(np.float32)
    for k in range(K):
        A = rng.standard_normal((D, D))
        R = A @ A.T / D + 0.5 * np.eye(D)
        cl.R[k] = R.astype(np.float32)
    w = rng.dirichlet(np.full(K, 5.0))
    cl.N[...] = (w * 1000).astype(np.float32)
    cl.avgvar[...] = 0.01
    return cl


def fitted_params(pkg, oracle, ev, K, iters=2):
    """Realistic parameters: the oracle's seeding followed by `iters` EM iterations
    (so that every event has at least one cluster at a moderate Mahalanobis distance,
    as in any real EM state)."""
    N, D = ev.shape
    cl = pkg.Clusters(K, D, N)
    oracle.seed(ev, K, cl)
    if iters:
        oracle.em(oracle.transpose(ev), cl, K, iters, iters)
    return cl


# Run-level tolerances.  Per-operator parity (one E-step / one M-step from identical inputs) is
# held to the 1e-4 bar of BASELINE.json.  After many EM iterations the comparison is against the
# exact-arithmetic oracle (ORACLE_REAL=double), and the reference's OWN FP32 arithmetic (the
# ORACLE_REAL=float build, pinned to the reference binary) already deviates from it by up to
# 4e-4 relative on responsibilities and 1e-5 on N_k (N=100k, D=16, K=32, 10 iterations; measured,
# see DESIGN.md "parity").  The run-level bar is therefore 1e-3 on responsibilities / 5e-4 on N_k,
# and still 1e-4 (scaled) on means and covariances.
RUN_RTOL_N = 5e-4
RUN_MEMB = dict(rtol=1e-3, atol=1e-5)


def assert_params_close(got, ref, K, rtol=1e-4, rtol_N=None):
    """The parity bar of BASELINE.json: 1e-4 relative on means / covariances
    (absolute floor scaled to each cluster's largest covariance entry)."""
    np.testing.assert_allclose(got.N[:K], ref.N[:K], rtol=rtol_N or rtol, atol=1e-3)
    np.testing.assert_allclose(got.pi[:K], ref.pi[:K], rtol=rtol, atol=1e-7)
    mscale = max(1.0, float(np.abs(ref.means[:K]).max()))
    np.testing.assert_allclose(got.means[:K], ref.means[:K], rtol=rtol, atol=rtol * mscale)
    for k in range(K):
        s = float(np.abs(ref.R[k]).max())
        np.testing.assert_allclose(got.R[k], ref.R[k], rtol=rtol, atol=rtol * s, err_msg=f"R[{k}]")
        # the inverse amplifies a relative perturbation of R by up to cond(R)
        si = float(np.abs(ref.Rinv[k]).max())
        cond = float(np.linalg.cond(ref.R[k].astype(np.float64)))
        tol_inv = rtol * max(10.0, cond)
        np.testing.assert_allclose(got.Rinv[k], ref.Rinv[k], rtol=tol_inv, atol=tol_inv * si, err_msg=f"Rinv[{k}] cond={cond:.3g}")
    for k in range(K):
        # d(ln det R) = tr(R^-1 dR) <= D * cond(R) * |dR|/|R|
        cond = float(np.linalg.cond(ref.R[k].astype(np.float64)))
        tol_c = max(2e-3, 0.5 * ref.R.shape[1] * rtol * cond)
        assert abs(float(got.constant[k]) - float(ref.constant[k])) <= tol_c + rtol * abs(float(ref.constant[k])), \
            (k, got.constant[k], ref.constant[k], cond)
