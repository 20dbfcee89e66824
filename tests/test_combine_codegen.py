"""Code-generation guard for gmm_combine (no GPU needed): every instance of the kernels of kernels_combine.cuh (the all-pairs
pass, the step pass with and without weights, the range sums and the labels) is built for sm_90a without a register spill or
a stack frame."""
import os
import re
import subprocess

import pytest

from conftest import ROOT
from test_mstep_codegen import _nvcc

CSRC = os.path.join(ROOT, "cuda-gmm-mpi_b200", "csrc")

_SRC = """#include "kernels_combine.cuh"
void launch_all(const float* m, size_t pitch, int n, int K, const float* w, double* part, const int* mem, const int* off,
                int* lab, float* mx) {
    gmm::combine_pairs_kernel<true><<<1, gmm::kCombPairThreads>>>(m, pitch, n, K, w, 64, part, 1);
    gmm::combine_pairs_kernel<false><<<1, gmm::kCombPairThreads>>>(m, pitch, n, K, nullptr, 64, part, 1);
    gmm::combine_sum_ranges_kernel<<<1, gmm::kCombSumThreads>>>(part, 1, 1, part);
    gmm::combine_step_kernel<true><<<1, gmm::kCombStepThreads>>>(m, pitch, n, w, mem, off, 2, 0, part);
    gmm::combine_step_kernel<false><<<1, gmm::kCombStepThreads>>>(m, pitch, n, nullptr, mem, off, 2, 0, part);
    gmm::combine_labels_kernel<<<1, gmm::kCombLabelThreads>>>(m, pitch, n, mem, off, 2, lab, mx);
}
"""


def test_combine_kernels_built_without_spills(tmp_path):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    src = tmp_path / "combine_codegen.cu"
    src.write_text(_SRC)
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-I", CSRC, "-Xptxas", "-v", "-c", "-o",
           str(tmp_path / "combine.o"), str(src)]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-4000:]
    current, seen = None, {}
    for ln in (res.stdout + res.stderr).splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", ln)
        if m:
            current = m.group(1) if "combine_" in m.group(1) else None
            continue
        if current is None:
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", ln)
        if m:
            seen[current] = tuple(int(g) for g in m.groups())
    assert len(seen) == 6, seen
    bad = {k: v for k, v in seen.items() if any(v)}
    assert not bad, bad
