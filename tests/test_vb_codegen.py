"""Code-generation guard for gmm_vb_em (no GPU needed): both instances of resp_entropy_kernel (with and without weights) are
built for sm_90a without a register spill or local memory."""
import os
import re
import subprocess

import pytest

from conftest import ROOT
from test_mstep_codegen import _nvcc

CSRC = os.path.join(ROOT, "cuda-gmm-mpi_b200", "csrc")

_SRC = """#include "kernels_vb.cuh"
void launch_both(const float* m, size_t pitch, int n, int K, const float* w, double* part) {
    gmm::resp_entropy_kernel<true><<<1, gmm::kEntropyThreads>>>(m, pitch, n, K, w, part);
    gmm::resp_entropy_kernel<false><<<1, gmm::kEntropyThreads>>>(m, pitch, n, K, nullptr, part);
}
"""


def test_entropy_kernel_built_without_spills(tmp_path):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    src = tmp_path / "vb_codegen.cu"
    src.write_text(_SRC)
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-I", CSRC, "-Xptxas", "-v", "-c", "-o",
           str(tmp_path / "vb.o"), str(src)]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-4000:]
    current, seen = None, {}
    for ln in (res.stdout + res.stderr).splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", ln)
        if m:
            current = m.group(1) if "resp_entropy_kernel" in m.group(1) else None
            continue
        if current is None:
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", ln)
        if m:
            seen[current] = tuple(int(g) for g in m.groups())
    assert len(seen) == 2, seen
    bad = {k: v for k, v in seen.items() if any(v)}
    assert not bad, bad
