"""Checks of gmm_condition_stats that need no GPU:
  * the float64 restatement's expansion (tests/_condition_stats_ref.py) equals a per-event brute force that completes every
    event per cluster and adds the conditional covariance, on random mixtures and observed sets;
  * condition_stats_prep_kernel, the one kernel the call adds, is built for sm_90a without a register spill or other local
    memory.  The E- and M-step kernels it launches are the resident steps' own, unchanged."""
import os
import re
import subprocess

import numpy as np
import pytest

import _condition_stats_ref as ref
from conftest import ROOT, random_spd_params
from test_mstep_codegen import _nvcc

CSRC = os.path.join(ROOT, "cuda-gmm-mpi_b200", "csrc")


def _mixture(pkg, K, D, seed):
    rng = np.random.default_rng(seed)
    cl = random_spd_params(pkg, K, D, rng)
    for k in range(K):
        cl.Rinv[k] = np.linalg.inv(cl.R[k].astype(np.float64)).astype(np.float32)
    return cl, rng


@pytest.mark.parametrize("D,K,obs", [(2, 1, (0,)), (3, 3, (1,)), (5, 2, (0, 2, 4)), (8, 3, (0, 1, 2, 3, 7)),
                                     (8, 4, tuple(range(7))), (12, 3, (0, 1, 2, 3, 4, 5, 8, 9)), (6, 2, tuple(range(6)))])
def test_expansion_equals_brute_force(pkg, D, K, obs):
    cl, rng = _mixture(pkg, K, D, seed=D * 100 + K)
    n = 60
    xo = (rng.standard_normal((n, len(obs))) * 3.0 + rng.uniform(-4, 4, len(obs))).astype(np.float32)
    memb = rng.dirichlet(np.ones(K), size=n).T.astype(np.float32)
    shift = rng.uniform(-2, 2, D)
    got = ref.expected_stats(cl, K, obs, xo, memb, shift)
    want = ref.brute_force_stats(cl, K, obs, xo, memb, shift)
    F = 1 + D + D * (D + 1) // 2
    scale = np.abs(want[:-1]).reshape(K, F).max(1).repeat(F)
    np.testing.assert_array_less(np.abs(got[:-1] - want[:-1]), 1e-12 * scale + 1e-300)


def test_expansion_with_every_dimension_observed_is_the_moments(pkg):
    D, K = 5, 3
    cl, rng = _mixture(pkg, K, D, seed=9)
    x = rng.standard_normal((40, D)).astype(np.float32)
    memb = rng.dirichlet(np.ones(K), size=40).T.astype(np.float32)
    shift = rng.uniform(-1, 1, D)
    y = x.astype(np.float64) - shift
    i, j = np.tril_indices(D)
    want = np.concatenate([np.concatenate([[g.sum()], g @ y, ((g[:, None] * y).T @ y)[i, j]]) for g in memb.astype(np.float64)]
                          + [[0.0]])
    np.testing.assert_allclose(ref.expected_stats(cl, K, tuple(range(D)), x, memb, shift), want, rtol=1e-13, atol=1e-13)


def test_prep_kernel_built_without_local_memory(tmp_path):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-I/usr/include", "-Xptxas", "-v",
           "-c", "-o", str(tmp_path / "gmm_api.o"), os.path.join(CSRC, "gmm_api.cu")]
    res = subprocess.run(cmd, cwd=CSRC, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-4000:]
    current, frame = False, None
    for ln in (res.stdout + res.stderr).splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", ln)
        if m:
            current = "condition_stats_prep_kernel" in m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", ln)
        if m and current:
            frame = sum(int(v) for v in m.groups())
            current = False
    assert frame is not None, "condition_stats_prep_kernel was not compiled"
    assert frame == 0, frame
