"""Code-generation guard for gmm_modes / gmm_mode_labels (no GPU needed): every instance of the kernels of kernels_modes.cuh
(the iteration and the labels at the 8 padded dimensions, the start and the compaction) is built for sm_90a without a
register spill or a stack frame."""
import os
import re
import subprocess

import pytest

from conftest import ROOT
from test_mstep_codegen import _nvcc

CSRC = os.path.join(ROOT, "cuda-gmm-mpi_b200", "csrc")

_SRC = """#include "kernels_modes.cuh"
template <int DP> void one(const float* r, const float* s, const int* a, float* x, int* it, int* st, int* lab, float* ep, float* lp) {
    gmm::mode_iter_kernel<DP><<<1, gmm::kModeThreads, gmm::mode_iter_smem(DP)>>>(DP, 8, r, s, a, 1, x, it, st, 10, 1e-5f, 16);
    gmm::mode_label_kernel<DP><<<1, gmm::kModeLabelThreads>>>(1, DP, 8, r, s, r, 1, 1e-2f, x, st, s, lab, ep, lp);
}
void launch_all(const float* r, const float* s, const int* a, float* x, int* it, int* st, int* lab, float* ep, float* lp, int* b) {
    one<4>(r, s, a, x, it, st, lab, ep, lp); one<8>(r, s, a, x, it, st, lab, ep, lp); one<12>(r, s, a, x, it, st, lab, ep, lp);
    one<16>(r, s, a, x, it, st, lab, ep, lp); one<20>(r, s, a, x, it, st, lab, ep, lp); one<24>(r, s, a, x, it, st, lab, ep, lp);
    one<28>(r, s, a, x, it, st, lab, ep, lp); one<32>(r, s, a, x, it, st, lab, ep, lp);
    gmm::mode_init_kernel<<<1, 256>>>(r, 4, 1, 1, 4, 4, s, x, it, st);
    gmm::mode_count_kernel<<<1, gmm::kModeScanThreads>>>(a, 1, st, b);
    gmm::mode_scan_kernel<<<1, gmm::kModeScanThreads>>>(b, 1, b);
    gmm::mode_scatter_kernel<<<1, gmm::kModeScanThreads>>>(a, 1, st, b, b);
}
"""


def test_modes_kernels_built_without_spills(tmp_path):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    src = tmp_path / "modes_codegen.cu"
    src.write_text(_SRC)
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-I", CSRC, "-Xptxas", "-v", "-c", "-o",
           str(tmp_path / "modes.o"), str(src)]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-4000:]
    current, seen = None, {}
    for ln in (res.stdout + res.stderr).splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", ln)
        if m:
            current = m.group(1) if "mode_" in m.group(1) else None
            continue
        if current is None:
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", ln)
        if m:
            seen[current] = tuple(int(g) for g in m.groups())
    assert len(seen) == 20, seen
    bad = {k: v for k, v in seen.items() if any(v)}
    assert not bad, bad
