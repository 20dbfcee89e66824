"""Code-generation guard for gmm_score_stats' chunk prep kernel (no GPU needed): score_stats_prep_kernel is built for
sm_90a without a register spill.  It is the one kernel the statistics pipeline adds; the E- and M-step kernels it
launches are the resident steps' own, unchanged."""
import os
import re
import subprocess

import pytest

from conftest import ROOT
from test_mstep_codegen import _nvcc

CSRC = os.path.join(ROOT, "cuda-gmm-mpi_b200", "csrc")


def test_prep_kernel_built_without_spills(tmp_path):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-I/usr/include", "-Xptxas", "-v",
           "-c", "-o", str(tmp_path / "gmm_api.o"), os.path.join(CSRC, "gmm_api.cu")]
    res = subprocess.run(cmd, cwd=CSRC, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-4000:]
    log = (res.stdout + res.stderr).splitlines()
    current, spills = False, None
    for ln in log:
        m = re.search(r"Compiling entry function '([^']+)'", ln)
        if m:
            current = "score_stats_prep_kernel" in m.group(1)
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", ln)
        if m and current:
            spills = int(m.group(1)) + int(m.group(2))
            current = False
    assert spills is not None, "score_stats_prep_kernel was not compiled"
    assert spills == 0, spills
