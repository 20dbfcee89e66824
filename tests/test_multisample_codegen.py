"""Code-generation guard for gmm_em_multisample (no GPU needed): every instance of the kernels of kernels_multisample.cuh
(the reweight pass with and without weights, in full and masses-only mode, and the finishing kernel) is built for sm_90a
without a register spill or a stack frame."""
import os
import re
import subprocess

import pytest

from conftest import ROOT
from test_mstep_codegen import _nvcc

CSRC = os.path.join(ROOT, "cuda-gmm-mpi_b200", "csrc")

_SRC = """#include "kernels_multisample.cuh"
void launch_all(float* m, size_t pitch, int K, const float* w, const float* rho, const gmm::MsUnit* u, const int* idx,
                double* part, double* out) {
    gmm::ms_reweight_kernel<true, false><<<1, gmm::kMsThreads>>>(m, pitch, K, w, rho, u, idx, 32, part);
    gmm::ms_reweight_kernel<false, false><<<1, gmm::kMsThreads>>>(m, pitch, K, nullptr, rho, u, idx, 32, part);
    gmm::ms_reweight_kernel<true, true><<<1, gmm::kMsThreads>>>(m, pitch, K, w, rho, u, idx, 32, part);
    gmm::ms_reweight_kernel<false, true><<<1, gmm::kMsThreads>>>(m, pitch, K, nullptr, rho, u, idx, 32, part);
    gmm::ms_finish_kernel<<<1, gmm::kMsFinishThreads>>>(part, idx, 1, K, out, out);
}
"""


def test_multisample_kernels_built_without_spills(tmp_path):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    src = tmp_path / "multisample_codegen.cu"
    src.write_text(_SRC)
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-I", CSRC, "-Xptxas", "-v", "-c", "-o",
           str(tmp_path / "multisample.o"), str(src)]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-4000:]
    current, seen = None, {}
    for ln in (res.stdout + res.stderr).splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", ln)
        if m:
            current = m.group(1) if "ms_" in m.group(1) else None
            continue
        if current is None:
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", ln)
        if m:
            seen[current] = tuple(int(g) for g in m.groups())
    assert len(seen) == 5, seen
    bad = {k: v for k, v in seen.items() if any(v)}
    assert not bad, bad

