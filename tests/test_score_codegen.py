"""Code-generation guard for the scoring kernel (no GPU needed): every score_tc_kernel<D> is built for sm_90a, and
none of them has a register spill or a ptxas C75xx performance line that estep_tc_kernel<D> of the same D does not
already have in the same compile.  The two kernels share the operand path and the per-tile logits
(tc_tile_logits), so a scoring epilogue that costs more registers than the E-step's would show here first."""
import os
import re
import subprocess

import pytest

from conftest import ROOT
from test_mstep_codegen import _nvcc

CSRC = os.path.join(ROOT, "cuda-gmm-mpi_b200", "csrc")
SCORE_DIMS = (8, 16, 24)


def test_score_kernels_built_without_new_spills_or_serialisation(tmp_path):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
           "-c", "-o", str(tmp_path / "kernels_tc.o"), os.path.join(CSRC, "kernels_tc.cu")]
    res = subprocess.run(cmd, cwd=CSRC, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-4000:]
    log = (res.stdout + res.stderr).splitlines()

    def kernel_of(name):
        m = re.search(r"(estep|score)_tc_kernelILi(\d+)E", name)
        return (m.group(1), int(m.group(2))) if m else None

    perf = {}                      # (kernel, D) -> set of C75xx codes
    spill = {}                     # (kernel, D) -> spill stores + loads
    current = None
    for ln in log:
        m = re.search(r"\((C75\d\d)\).*function '([^']+)'", ln)
        if m and kernel_of(m.group(2)):
            perf.setdefault(kernel_of(m.group(2)), set()).add(m.group(1))
        m = re.search(r"Compiling entry function '([^']+)'", ln)
        if m:
            current = kernel_of(m.group(1))
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", ln)
        if m and current:
            spill[current] = int(m.group(1)) + int(m.group(2))
            current = None
    assert {d for (k, d) in spill if k == "score"} == set(SCORE_DIMS), sorted(spill)
    for d in SCORE_DIMS:
        new_codes = perf.get(("score", d), set()) - perf.get(("estep", d), set())
        assert not new_codes, (d, new_codes)
        if spill[("estep", d)] == 0:
            assert spill[("score", d)] == 0, (d, spill[("score", d)])
