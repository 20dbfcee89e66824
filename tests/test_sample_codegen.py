"""Code-generation guard for gmm_sample (no GPU needed): every instance of sample_kernel (D = 1 .. 32) is built for sm_90a
without a register spill."""
import os
import re
import subprocess

import pytest

from conftest import ROOT
from test_mstep_codegen import _nvcc

CSRC = os.path.join(ROOT, "cuda-gmm-mpi_b200", "csrc")


def test_sample_kernels_built_without_spills(tmp_path):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-I/usr/include", "-Xptxas", "-v",
           "-c", "-o", str(tmp_path / "gmm_api.o"), os.path.join(CSRC, "gmm_api.cu")]
    res = subprocess.run(cmd, cwd=CSRC, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-4000:]
    current, spills = None, {}
    for ln in (res.stdout + res.stderr).splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", ln)
        if m:
            current = m.group(1) if "sample_kernel" in m.group(1) else None
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", ln)
        if m and current:
            spills[current] = int(m.group(1)) + int(m.group(2))
            current = None
    assert len(spills) == 32, sorted(spills)
    bad = {n: s for n, s in spills.items() if s}
    assert not bad, bad
